"""GPU: the training step's data-gradient, normalisation and loss-scaling kernels, one C entry point at a time, against
float64 torch on the CPU computed on the same fp16-rounded operands.

Every entry point is driven in the sequence the training trunk uses (csrc/trunk_train.cu::conv_backward /
bn_backward), and every output buffer starts as NaN so that an element the
kernel never writes fails the check.  Channel-slice kernels (pitch > C, the two halves of an IBN layer) must also leave
every channel outside their slice bit-identical.

Rounding budgets used below (u16 = 2^-11, the half-ulp of an fp16 result rounded to nearest):
  - a value the kernel rounds to fp16 once:            |got - ref| <= u16 * |ref|
  - fp32 tensor-core accumulation of exact fp16 products: 2^-19 * sum |terms|.  This is not a worst-case bound (that is
    K * 2^-24, about 2^-11.8 for the largest reduction here, K = 9 * 512, and the random-walk estimate sqrt(K) * 2^-24 is
    2^-17.9); it is ~10x the largest excess over the output rounding measured on an H100 (2^-22.4 of sum |terms|), so a
    kernel that rounded any partial sum to fp16 (2^-11 per rounding) fails it
  - statistics (mean, invstd): 1e-5 relative of float64, as test_train_gpu.py::test_bn_train_forward_backward."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U16 = 2.0 ** -11
ACC32 = 2.0 ** -19
PACK_CHUNK = 8192  # source elements per chunk of ctl_train_pack_weights / ctl_grad_check_multi
NAN16 = float("nan")


def _n():
    from ctl_b200 import _native as N

    return N, N.lib()


def _bits(t):
    """Bit pattern of a tensor (NaN == NaN), for 'unchanged' and 'exact' checks."""
    t = t.contiguous()
    return t.view({torch.float16: torch.int16, torch.float32: torch.int32}[t.dtype])


def _nan16(*shape):
    return torch.full(shape, NAN16, dtype=torch.float16, device="cuda")


def _nan32(*shape):
    return torch.full(shape, NAN16, dtype=torch.float32, device="cuda")


# ===================================================================================================================
# 1. ctl_train_pack_weights: fp16 forward operand [cout][k][k][cin] and flipped data-gradient operand [cin][k][k][cout]
# ===================================================================================================================
def _pack_table(entries):
    """The 48-byte entries of csrc/trunk_train.cu's pack table (ctl_trainer_bind): {src, fwd, dgrad, cout | cin << 32, k (pad 0),
    chunk_begin}; entries = [(src fp32 [cout][cin][k][k], fwd, dgrad or None)]."""
    rows, chunks = [], 0
    for src, fwd, dgr in entries:
        cout, cin, k, _ = src.shape
        rows.append([src.data_ptr(), fwd.data_ptr(), 0 if dgr is None else dgr.data_ptr(), cout | (cin << 32), k, chunks])
        chunks += (src.numel() + PACK_CHUNK - 1) // PACK_CHUNK
    return torch.tensor(rows, dtype=torch.int64).cuda(), len(rows), chunks


def _pack(srcs, with_dgrad=None):
    """Packs the device fp32 weights `srcs` in ONE launch into NaN-filled fp16 arenas with NaN guard gaps around every
    operand; returns [(fwd, dgrad or None)] views and the two arenas with the guard masks."""
    N, L = _n()
    guard = 24
    total = sum(s.numel() + guard for s in srcs) + guard
    arenas = (_nan16(total), _nan16(total))
    used = torch.zeros(total, dtype=torch.bool)
    views, entries, off = [], [], guard
    for i, s in enumerate(srcs):
        cout, cin, k, _ = s.shape
        fwd = arenas[0][off:off + s.numel()].view(cout, k, k, cin)
        dgr = arenas[1][off:off + s.numel()].view(cin, k, k, cout)
        if with_dgrad is not None and not with_dgrad[i]:
            dgr = None
        used[off:off + s.numel()] = True
        views.append((fwd, dgr))
        entries.append((s, fwd, dgr))
        off += s.numel() + guard
    table, n, chunks = _pack_table(entries)
    N.check(L.ctl_train_pack_weights(table.data_ptr(), n, chunks, N.stream_ptr()))
    torch.cuda.synchronize()
    return views, arenas, used


def test_train_pack_weights_exact():
    """Bit-exact against torch's own fp16 rounding and permutes, with 1x1 and 3x3 weights whose sizes are and are not
    multiples of the 8192-element chunk (so chunks straddle tensors), one entry without a data-gradient operand, and
    values that round to fp16 subnormals, to -0 and to +-inf.  Nothing outside the operands may be written."""
    g = torch.Generator().manual_seed(1)
    shapes = [(64, 64, 1, 1),      # 4096: less than one chunk
              (64, 64, 3, 3),      # 36864: 4.5 chunks
              (40, 24, 3, 3),      # 8640: just over one chunk, non-square
              (256, 64, 1, 1),     # 16384: exactly 2 chunks, packed without a data-gradient operand
              (72, 40, 3, 3),      # 25920
              (128, 256, 3, 3),    # 294912: 36 chunks
              (2048, 512, 1, 1),   # 1048576: layer4 conv3
              (8, 8, 3, 3)]        # 576: a tail entry smaller than a block's stride
    srcs = [torch.randn(*s, generator=g) * 0.05 for s in shapes]
    special = torch.tensor([1e-6, -3e-8, -1e-9, 65519.0, 65520.0, -7e4, 0.5 + 2.0 ** -12, 2.0 ** -24])
    srcs[0].view(-1)[:special.numel()] = special
    srcs[2].view(-1)[-special.numel():] = special
    dev = [s.cuda() for s in srcs]
    with_dgrad = [i != 3 for i in range(len(shapes))]
    views, arenas, used = _pack(dev, with_dgrad)
    for i, (s, (fwd, dgr)) in enumerate(zip(srcs, views)):
        want_f = s.half().permute(0, 2, 3, 1)
        assert torch.equal(_bits(fwd.cpu()), _bits(want_f)), f"forward operand of {tuple(s.shape)}"
        if dgr is not None:
            want_d = s.half().flip(2, 3).permute(1, 2, 3, 0)
            assert torch.equal(_bits(dgr.cpu()), _bits(want_d)), f"data-gradient operand of {tuple(s.shape)}"
    # guard gaps, and the data-gradient slot of the entry packed with dgrad = NULL, stay NaN
    nodg = torch.zeros_like(used)
    off = 24 + sum(s.numel() + 24 for s in srcs[:3])
    nodg[off:off + srcs[3].numel()] = True
    assert torch.isnan(arenas[0].cpu()[~used]).all()
    assert torch.isnan(arenas[1].cpu()[~used | nodg]).all()


# ===================================================================================================================
# 2. data-gradient convolution (the transposed convolution of every bottleneck conv), with and without the shortcut
#    gradient as `residual`
# ===================================================================================================================
# layer resolutions (layer1..layer3, layer4 with last_stride 1; last_stride 2 halves layer3's) of the training crops
MAPS = {"256x128": ((64, 32), (32, 16), (16, 8)), "320x320": ((80, 80), (40, 40), (20, 20)),
        "160x80": ((40, 20), (20, 10), (10, 5))}
# forward conv (cin, cout, k, stride) and the layer resolution index of its INPUT
GEOMS = {
    "s1_1x1_l1": (256, 64, 1, 1, 0),        # layer1.x conv1
    "s1_3x3_c64": (64, 64, 3, 1, 0),        # layer1 conv2: the dgrad is a 64 -> 64 3x3 (conv3x3_c64_kernel)
    "s1_1x1_expand": (64, 256, 1, 1, 0),    # layer1 conv3 / downsample: dgrad 256 -> 64
    "s2_3x3_l2": (128, 128, 3, 2, 0),       # layer2.0 conv2: zero-insertion upsample, then a stride-1 3x3
    "s2_1x1_l2": (256, 512, 1, 2, 0),       # layer2.0 downsample: 1x1 at low resolution, then upsample (+ residual)
    "s2_3x3_l3": (256, 256, 3, 2, 1),       # layer3.0 conv2
    "s2_1x1_l3": (512, 1024, 1, 2, 1),      # layer3.0 downsample
    "s1_3x3_l4": (512, 512, 3, 1, 2),       # layer4.0 conv2, last_stride 1
    "s1_1x1_l4": (1024, 2048, 1, 1, 2),     # layer4.0 downsample, last_stride 1
    "s2_3x3_l4": (512, 512, 3, 2, 2),       # layer4.0 conv2, last_stride 2
    "s2_1x1_l4": (1024, 2048, 1, 2, 2),     # layer4.0 downsample, last_stride 2
    "s1_1x1_l4_conv1": (2048, 512, 1, 1, 2),  # layer4.x conv1: dgrad 512 -> 2048
}
DGRAD_CASES = [(m, gname) for m in MAPS for gname in GEOMS
               # a stride-2 layer needs an even input map (the engine's zero-insertion doubles ho x wo)
               if not (GEOMS[gname][3] == 2 and any(v % 2 for v in MAPS[m][GEOMS[gname][4]]))]


def _dgrad_launches(N, L, dy, wd, n, h, w, cin, cout, k, stride, residual):
    """trunk_train.cu::conv_backward's data-gradient launches; dy [n][ho][wo][cout] -> dx [n][h][w][cin]."""
    ho, wo = dy.shape[1], dy.shape[2]
    zero_bias = torch.zeros(2048, device="cuda")
    dx = _nan16(n, h, w, cin)
    rp = N.ptr(residual)
    st = N.stream_ptr()
    if stride == 1:
        N.check(L.ctl_conv2d_nhwc_f16(dy.data_ptr(), n, ho, wo, cout, wd.data_ptr(), zero_bias.data_ptr(), rp, dx.data_ptr(),
                                      cin, k, 1, 0, 0, st))
    elif k == 1:
        low = _nan16(n, ho, wo, cin)
        N.check(L.ctl_conv2d_nhwc_f16(dy.data_ptr(), n, ho, wo, cout, wd.data_ptr(), zero_bias.data_ptr(), None,
                                      low.data_ptr(), cin, 1, 1, 0, 0, st))
        N.check(L.ctl_upsample2_zero_nhwc_f16(low.data_ptr(), n, ho, wo, cin, rp, dx.data_ptr(), st))
    else:
        up = _nan16(n, h, w, cout)
        N.check(L.ctl_upsample2_zero_nhwc_f16(dy.data_ptr(), n, ho, wo, cout, None, up.data_ptr(), st))
        N.check(L.ctl_conv2d_nhwc_f16(up.data_ptr(), n, h, w, cout, wd.data_ptr(), zero_bias.data_ptr(), rp, dx.data_ptr(),
                                      cin, 3, 1, 0, 0, st))
    torch.cuda.synchronize()
    return dx.cpu().double()


@pytest.mark.parametrize("map_name,geom", DGRAD_CASES)
def test_dgrad_conv_vs_conv2d_input(map_name, geom):
    """dx = torch.nn.grad.conv2d_input in float64 of the fp16 weight and fp16 dy (+ the fp16 shortcut gradient), with
    the weight operand packed by ctl_train_pack_weights as the engine does.
    Budget: one fp16 rounding of dx plus the fp32 accumulation allowance; the strided 1x1 path rounds twice (the
    low-resolution GEMM output, then low + residual), so it gets a second half-ulp of the un-residualed value."""
    N, L = _n()
    cin, cout, k, stride, li = GEOMS[geom]
    h, w = MAPS[map_name][li]
    n = 1 if map_name == "320x320" else 2
    pad = k // 2
    ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    g = torch.Generator().manual_seed(sum(map(ord, map_name + geom)))
    wt = torch.randn(cout, cin, k, k, generator=g) / (k * cout ** 0.5)   # fp32 parameter, packed to fp16 on the device
    dy = torch.randn(n, ho, wo, cout, generator=g).half()
    res = (torch.randn(n, h, w, cin, generator=g) * 0.5).half()
    [(_, wd)], _, _ = _pack([wt.cuda()])

    w16, dyn = wt.half().double(), dy.double().permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_input((n, cin, h, w), w16, dyn, stride=stride, padding=pad).permute(0, 2, 3, 1)
    mag = torch.nn.grad.conv2d_input((n, cin, h, w), w16.abs().float(), dyn.abs().float(), stride=stride,
                                     padding=pad).permute(0, 2, 3, 1).double()   # sum |terms| per output
    dyd, resd = dy.cuda(), res.cuda()
    for with_res in (False, True):
        got = _dgrad_launches(N, L, dyd, wd, n, h, w, cin, cout, k, stride, resd if with_res else None)
        want = ref + res.double() if with_res else ref
        tol = U16 * want.abs() + ACC32 * mag + 2.0 ** -25
        if stride == 2 and k == 1 and with_res:
            tol = tol + U16 * ref.abs()
        assert torch.isfinite(got).all(), "unwritten or non-finite outputs"
        err = (got - want).abs()
        bad = err > tol
        assert not bad.any(), (f"residual={with_res}: {int(bad.sum())} / {bad.numel()} off; max err/budget "
                               f"{float((err / tol).max()):.2f}; first bad [n, h, w, c] {bad.nonzero()[0].tolist()}")


# ===================================================================================================================
# 3. batch-statistics BatchNorm over a channel slice (pitch >= c), train forward + backward
# ===================================================================================================================
def _bn_slice_case(rows, c, pitch, relu, res, running, shift=0.0, seed=0):
    """BatchNorm2d (train) + [residual] + [ReLU] on channels [pitch - c, pitch) of an NHWC fp16 tensor of row pitch
    `pitch` -- the BatchNorm half of an IBN layer when pitch == 2c, the plain layer when pitch == c -- called with
    channel-offset base pointers and g_out aliasing dz, as the engines call it.  y = shift + N(0, 1) on the slice."""
    N, L = _n()
    off = pitch - c
    sl = slice(off, pitch)
    g = torch.Generator().manual_seed(seed + rows + 7 * c + pitch + int(shift))
    y = torch.randn(rows, pitch, generator=g) * 2
    y[:, sl] = torch.randn(rows, c, generator=g) + shift
    y = y.half()
    r = torch.randn(rows, pitch, generator=g).half()
    gamma, beta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.2
    rm, rv = torch.randn(c, generator=g) * 0.1, torch.rand(c, generator=g) + 0.5
    dz = (torch.randn(rows, pitch, generator=g) * 0.1).half()
    eps, mom, unscale = 1e-5, 0.1, 0.25

    yd = y[:, sl].double().requires_grad_(True)
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    mean, var = yd.mean(0), yd.var(0, unbiased=False)
    pre = (yd - mean) / torch.sqrt(var + eps) * gd + bd + (r[:, sl].double() if res else 0.0)
    zref = pre.clamp(min=0) if relu else pre
    zref16 = zref.detach().half()
    mask = (zref16 > 0).double() if relu else torch.ones_like(pre)
    (pre * (dz[:, sl].double() * mask)).sum().backward()

    b = 2 * off  # byte offset of the slice
    yc, rc_, dzc = y.cuda(), r.cuda(), dz.cuda()
    gam, bet = gamma.cuda(), beta.cuda()
    rmc, rvc = (rm.cuda(), rv.cuda()) if running else (None, None)
    nb = L.ctl_bn_workspace_bytes(rows, c)
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
    sm, si = _nan32(c), _nan32(c)
    out = _nan16(rows, pitch)
    N.check(L.ctl_bn_train_forward_nhwc_f16(yc.data_ptr() + b, rows, c, pitch, gam.data_ptr(), bet.data_ptr(), eps, mom,
                                            N.ptr(rmc), N.ptr(rvc), rc_.data_ptr() + b if res else None, int(relu),
                                            ws.data_ptr(), nb, sm.data_ptr(), si.data_ptr(), out.data_ptr() + b,
                                            N.stream_ptr()))
    torch.cuda.synchronize()
    istd = 1 / torch.sqrt(var + eps)
    np.testing.assert_allclose(sm.cpu().numpy(), mean.detach().numpy(), rtol=1e-5, atol=1e-6, err_msg="save_mean")
    np.testing.assert_allclose(si.cpu().numpy(), istd.detach().numpy(), rtol=1e-5, err_msg="save_invstd")
    if running:
        np.testing.assert_allclose(rmc.cpu().numpy(), (0.9 * rm.double() + 0.1 * mean.detach()).numpy(), rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(rvc.cpu().numpy(), (0.9 * rv.double() + 0.1 * yd.detach().var(0, unbiased=True)).numpy(),
                                   rtol=1e-5)
    o = out.cpu()
    assert torch.isfinite(o[:, sl]).all(), "unwritten forward outputs"
    err = (o[:, sl].double() - zref.detach()).abs().max()
    assert float(err) <= float(zref.abs().max()) * 2.0 ** -10 + 1e-6  # one fp16 rounding at the output's scale
    assert torch.isnan(o[:, :off]).all(), "forward wrote outside its channel slice"

    # backward: z is the reference's own fp16 output (same ReLU mask), g_out aliases dz (csrc/trunk_train.cu::bn_backward)
    zfull = torch.randn(rows, pitch, generator=g).half()
    zfull[:, sl] = zref16
    zc = zfull.cuda()
    dgam, dbet = _nan32(c), _nan32(c)
    dy = _nan16(rows, pitch)
    N.check(L.ctl_bn_train_backward_nhwc_f16(dzc.data_ptr() + b, zc.data_ptr() + b if relu else None, yc.data_ptr() + b,
                                             rows, c, pitch, gam.data_ptr(), sm.data_ptr(), si.data_ptr(), unscale,
                                             ws.data_ptr(), nb, dzc.data_ptr() + b if relu else None, dgam.data_ptr(),
                                             dbet.data_ptr(), dy.data_ptr() + b, N.stream_ptr()))
    torch.cuda.synchronize()
    np.testing.assert_allclose(dgam.cpu().numpy(), unscale * gd.grad.numpy(), rtol=2e-4,
                               atol=2e-4 * float(gd.grad.abs().max()), err_msg="dgamma")
    np.testing.assert_allclose(dbet.cpu().numpy(), unscale * bd.grad.numpy(), rtol=2e-4,
                               atol=2e-4 * float(bd.grad.abs().max()), err_msg="dbeta")
    dyo, dzo = dy.cpu(), dzc.cpu()
    dyr = yd.grad
    assert torch.isfinite(dyo[:, sl]).all(), "unwritten data gradients"
    assert float((dyo[:, sl].double() - dyr).abs().max()) <= float(dyr.abs().max()) * 2.0 ** -9 + 1e-7
    assert torch.isnan(dyo[:, :off]).all(), "backward wrote dy outside its channel slice"
    want_g = torch.where(mask > 0, dz[:, sl], 0.0) if relu else dz[:, sl]  # masked lanes are +0, as the kernel writes
    assert torch.equal(_bits(dzo[:, sl]), _bits(want_g)), "g = dz * mask (written over dz)"
    assert torch.equal(_bits(dzo[:, :off]), _bits(dz[:, :off])), "backward wrote g outside its channel slice"


BN_SLICE_CASES = [
    # rows, c, pitch, relu, residual, running statistics
    (2, 32, 32, 1, 0, 1), (333, 32, 32, 1, 1, 0), (800, 32, 32, 0, 0, 1),
    (2, 512, 512, 0, 0, 0), (333, 512, 512, 1, 1, 1), (800, 512, 512, 1, 0, 0),
    (2, 1024, 1024, 1, 1, 1), (333, 1024, 1024, 0, 0, 0), (800, 1024, 1024, 1, 1, 1),
    # IBN BatchNorm halves: channels [c, 2c) of a 2c-channel tensor, ReLU, no residual
    (2, 32, 64, 1, 0, 1), (333, 32, 64, 1, 0, 0), (800, 32, 64, 1, 0, 1),
    (2, 64, 128, 1, 0, 0), (333, 64, 128, 1, 0, 1), (800, 64, 128, 1, 0, 0),
    (2, 128, 256, 1, 0, 1), (333, 128, 256, 1, 0, 0), (800, 128, 256, 1, 0, 1),
]


@pytest.mark.parametrize("rows,c,pitch,relu,res,running", BN_SLICE_CASES)
def test_bn_train_channel_slice(rows, c, pitch, relu, res, running):
    """rows = 2 and 333 fill no block; 800 = a batch of 2 at the 320x320 crop's layer4 map (20 x 20)."""
    _bn_slice_case(rows, c, pitch, relu, res, running)


@pytest.mark.parametrize("shift", [0, 8, 64])
@pytest.mark.parametrize("rows,c,pitch", [(800, 64, 128), (333, 1024, 1024), (131072, 64, 64)])
def test_bn_train_shifted_mean(shift, rows, c, pitch):
    """Channels whose mean is `shift` standard deviations away from zero: statistics must stay within 1e-5 of float64
    (summing y and y^2 and subtracting mean^2 cancels catastrophically here).  131072 rows = a batch of 64 at the
    256x128 crop's layer1 map (64 x 32)."""
    _bn_slice_case(rows, c, pitch, 1, 0, 1, shift=float(shift))


# ===================================================================================================================
# 4. InstanceNorm + ReLU on the first `half` channels of an IBN layer (per-image statistics), train forward + backward
# ===================================================================================================================
def _instnorm_case(n, hw, half, shift=0.0, seed=0):
    N, L = _n()
    pitch = 2 * half
    sl = slice(0, half)
    g = torch.Generator().manual_seed(seed + 13 * hw + half + int(shift))
    y = torch.randn(n, hw, pitch, generator=g) * 2
    y[..., sl] = torch.randn(n, hw, half, generator=g) + shift
    y = y.half()
    gamma, beta = torch.rand(half, generator=g) + 0.5, torch.randn(half, generator=g) * 0.2
    dz = (torch.randn(n, hw, pitch, generator=g) * 0.1).half()
    eps, unscale = 1e-5, 0.125

    yd = y[..., sl].double().permute(0, 2, 1).requires_grad_(True)  # [n][half][hw]
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    pre = F.instance_norm(yd, weight=gd, bias=bd, eps=eps)
    zref = pre.clamp(min=0)
    zref16 = zref.detach().half()
    gref = torch.where(zref16 > 0, dz[..., sl].double().permute(0, 2, 1), 0.0)  # g = dz * mask; masked lanes are +0
    (pre * gref).sum().backward()
    mean = yd.detach().mean(2)
    istd = 1 / torch.sqrt(yd.detach().var(2, unbiased=False) + eps)

    yc, gam, bet = y.cuda(), gamma.cuda(), beta.cuda()
    sm, si = _nan32(n, half), _nan32(n, half)
    out = _nan16(n, hw, pitch)
    N.check(L.ctl_instnorm_train_forward_nhwc_f16(yc.data_ptr(), n, hw, pitch, half, gam.data_ptr(), bet.data_ptr(), eps,
                                                  sm.data_ptr(), si.data_ptr(), out.data_ptr(), N.stream_ptr()))
    torch.cuda.synchronize()
    np.testing.assert_allclose(sm.cpu().numpy(), mean.numpy(), rtol=1e-5, atol=1e-6, err_msg="save_mean")
    np.testing.assert_allclose(si.cpu().numpy(), istd.numpy(), rtol=1e-5, err_msg="save_invstd")
    o = out.cpu()
    zr = zref.detach().permute(0, 2, 1)
    assert torch.isfinite(o[..., sl]).all(), "unwritten forward outputs"
    assert float((o[..., sl].double() - zr).abs().max()) <= float(zr.abs().max()) * 2.0 ** -10 + 1e-6
    assert torch.isnan(o[..., half:]).all(), "InstanceNorm wrote into the BatchNorm half"

    zfull = torch.randn(n, hw, pitch, generator=g).half()
    zfull[..., sl] = zref16.permute(0, 2, 1)
    zc, dzc = zfull.cuda(), dz.cuda()
    dgp, dbp = _nan32(n, half), _nan32(n, half)
    dy = _nan16(n, hw, pitch)
    N.check(L.ctl_instnorm_train_backward_nhwc_f16(dzc.data_ptr(), zc.data_ptr(), yc.data_ptr(), n, hw, pitch, half,
                                                   gam.data_ptr(), sm.data_ptr(), si.data_ptr(), unscale, dgp.data_ptr(),
                                                   dbp.data_ptr(), dy.data_ptr(), N.stream_ptr()))
    torch.cuda.synchronize()
    # per-image partials: sum over the image's positions of g * xhat and of g
    xhat = (yd.detach() - mean[..., None]) * istd[..., None]
    dgp_ref, dbp_ref = (gref * xhat).sum(2), gref.sum(2)
    dgpc, dbpc = dgp.cpu().double(), dbp.cpu().double()
    np.testing.assert_allclose(dgpc.numpy(), unscale * dgp_ref.numpy(), rtol=2e-4, atol=2e-4 * float(dgp_ref.abs().max()))
    np.testing.assert_allclose(dbpc.numpy(), unscale * dbp_ref.numpy(), rtol=2e-4, atol=2e-4 * float(dbp_ref.abs().max()))
    # ... which sum over the images to the parameter gradients (x grad_unscale)
    np.testing.assert_allclose(dgpc.sum(0).numpy(), unscale * gd.grad.numpy(), rtol=2e-4,
                               atol=2e-4 * float(gd.grad.abs().max()), err_msg="dgamma")
    np.testing.assert_allclose(dbpc.sum(0).numpy(), unscale * bd.grad.numpy(), rtol=2e-4,
                               atol=2e-4 * float(bd.grad.abs().max()), err_msg="dbeta")
    dyo, dzo = dy.cpu(), dzc.cpu()
    dyr = yd.grad.permute(0, 2, 1)
    assert torch.isfinite(dyo[..., sl]).all(), "unwritten data gradients"
    assert float((dyo[..., sl].double() - dyr).abs().max()) <= float(dyr.abs().max()) * 2.0 ** -9 + 1e-7
    assert torch.isnan(dyo[..., half:]).all(), "InstanceNorm backward wrote dy into the BatchNorm half"
    assert torch.equal(_bits(dzo[..., sl]), _bits(gref.permute(0, 2, 1).half())), "g = dz * mask (written over dz)"
    assert torch.equal(_bits(dzo[..., half:]), _bits(dz[..., half:])), "InstanceNorm backward wrote into the BatchNorm half"


IN_HW = [8, 255, 256, 257, 800, 2048, 6400]  # both sides of the 256-thread row loop; 6400 = 320x320's 80 x 80


@pytest.mark.parametrize("half", [32, 64, 128])
@pytest.mark.parametrize("hw", IN_HW)
def test_instnorm_train_forward_backward(hw, half):
    _instnorm_case(2 if hw >= 2048 else 3, hw, half)


@pytest.mark.parametrize("shift", [8, 64])
@pytest.mark.parametrize("hw", IN_HW)
def test_instnorm_train_shifted_mean(hw, shift):
    """Instances whose mean is `shift` standard deviations away from zero: statistics within 1e-5 of float64."""
    _instnorm_case(2, hw, 64, shift=float(shift))


# ===================================================================================================================
# 5. dynamic loss scaling: overflow check (+ in-place rescale) and GradScaler.update()
# ===================================================================================================================
def _grad_table(grads):
    rows, chunks = [], 0
    for t in grads:
        rows.append([t.data_ptr(), t.numel(), chunks])
        chunks += (t.numel() + PACK_CHUNK - 1) // PACK_CHUNK
    return torch.tensor(rows, dtype=torch.int64).cuda(), len(rows), chunks


def _grad_check(grads, mul=1.0, mul_dev=None, flag=None):
    N, L = _n()
    flag = torch.zeros(1, dtype=torch.int32, device="cuda") if flag is None else flag
    table, n, chunks = _grad_table(grads)
    N.check(L.ctl_grad_check_multi(table.data_ptr(), n, chunks, float(mul), N.ptr(mul_dev), flag.data_ptr(), N.stream_ptr()))
    torch.cuda.synchronize()
    return flag


def _grad_set(seed):
    g = torch.Generator().manual_seed(seed)
    # 3 full chunks + a partial one, a tensor smaller than one block's stride, exactly one chunk
    return [torch.randn(3 * PACK_CHUNK + 77, generator=g), torch.randn(100, generator=g), torch.randn(PACK_CHUNK, generator=g)]


@pytest.mark.parametrize("bad", [float("inf"), float("-inf"), float("nan")])
@pytest.mark.parametrize("where", ["first_of_last_chunk", "last"])
def test_grad_check_flags_non_finite(bad, where):
    """inf / -inf / NaN in the first or the last element of a tensor's partial last chunk sets found_inf; with a factor
    of exactly 1 (mul = 1, *mul_device = 1) nothing is rewritten: every gradient keeps its bits."""
    host = _grad_set(3)
    idx = 3 * PACK_CHUNK if where == "first_of_last_chunk" else host[0].numel() - 1
    host[0][idx] = bad
    dev = [t.cuda() for t in host]
    assert int(_grad_check(dev)[0]) == 1
    one = torch.ones(1, device="cuda")
    assert int(_grad_check(dev, 1.0, one)[0]) == 1
    for t, d in zip(host, dev):
        assert torch.equal(_bits(d.cpu()), _bits(t))
    clean = [t.cuda() for t in _grad_set(3)]
    assert int(_grad_check(clean, 1.0, one)[0]) == 0


def test_grad_check_rescale_and_overflow_after_mul():
    """mul * (*mul_device) rescales in place as one fp32 product per element; finite values that overflow only after
    the rescale are flagged; found_inf OR-accumulates across calls (only the caller clears it)."""
    host = _grad_set(5)
    for mul, md in ((0.5, 0.25), (1.0, 2.0 ** -10), (3.0, None)):
        dev = [t.cuda() for t in host]
        mdd = None if md is None else torch.tensor([md], device="cuda")
        assert int(_grad_check(dev, mul, mdd)[0]) == 0
        f = torch.tensor(mul, dtype=torch.float32) * (1.0 if md is None else torch.tensor(md, dtype=torch.float32))
        for t, d in zip(host, dev):
            assert torch.equal(_bits(d.cpu()), _bits(t * f))
    big = _grad_set(5)
    big[0][3 * PACK_CHUNK + 76] = 3e38   # finite; x 2 overflows
    big[2][0] = -2e38                    # finite; x 2 overflows
    for mul, md in ((2.0, None), (0.5, 4.0)):
        dev = [t.cuda() for t in big]
        mdd = None if md is None else torch.tensor([md], device="cuda")
        assert int(_grad_check(dev, mul, mdd)[0]) == 1
        assert float(dev[0][3 * PACK_CHUNK + 76]) == float("inf") and float(dev[2][0]) == float("-inf")
    # OR-accumulation: clean after dirty keeps the flag; a clean call on a cleared flag leaves 0
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    clean = [t.cuda() for t in _grad_set(6)]
    assert int(_grad_check(clean, flag=flag)[0]) == 0
    dirty = [t.cuda() for t in big]
    assert int(_grad_check(dirty, 2.0, flag=flag)[0]) == 1
    assert int(_grad_check(clean, flag=flag)[0]) == 1
    assert int(_grad_check(clean, 1.0, torch.tensor([0.5], device="cuda"), flag=flag)[0]) == 1


def test_loss_scale_update_follows_grad_scaler():
    """ctl_loss_scale_update against GradScaler's update rule (torch._amp_update_scale_ on CPU tensors) over a scripted
    run of clean and overflowing steps across several growth intervals, including a growth that would overflow fp32
    (GradScaler keeps the old scale then).  After every step: state3 = {scale, scale / base, base / scale} as fp32,
    the growth tracker, last_found = this step's flag, and found_inf cleared."""
    N, L = _n()
    base, growth, backoff, interval = 1024.0, 2.0, 0.5, 3
    script = [0, 0, 0, 0, 0, 0, 1, 0, 0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0]
    for init in (65536.0, 2.0 ** 126):
        state = torch.tensor([init, init / base, base / init], dtype=torch.float32, device="cuda")
        ints = torch.zeros(3, dtype=torch.int32, device="cuda")  # tracker, found_inf, last_found
        ref_scale = torch.tensor([init], dtype=torch.float32)
        ref_tracker = torch.zeros(1, dtype=torch.int32)
        for step, found in enumerate(script):
            ints[1] = found
            N.check(L.ctl_loss_scale_update(state.data_ptr(), ints[0:1].data_ptr(), ints[1:2].data_ptr(), ints[2:3].data_ptr(),
                                            base, growth, backoff, interval, N.stream_ptr()))
            torch._amp_update_scale_(ref_scale, ref_tracker, torch.tensor([float(found)]), growth, backoff, interval)
            torch.cuda.synchronize()
            s = ref_scale.clone()
            want = torch.cat([s, s / base, base / s]).float()
            got = state.cpu()
            assert torch.equal(_bits(got), _bits(want)), (init, step, got.tolist(), want.tolist())
            assert ints.cpu().tolist() == [int(ref_tracker), 0, found], (init, step)
