"""GPU: the eval trunk's kernels other than the convolution GEMMs -- InstanceNorm + ReLU, max-pool, the tensor-core stem
and the pool + BatchNorm1d head -- one C entry point at a time, against float64 torch on the CPU computed on the same
fp16 or fp32 operands.

Shapes are the ones the eval trunk runs (ResNet50 and ResNet50-IBN-a at 256x128, 320x320 and 128x64 crops, and the
tensor-core stem's odd sides) plus the edges of each kernel's loops.  Every out-of-place output starts as NaN, so that
an element the kernel never writes fails.

Rounding budgets (u = 2^-24, half an fp32 ulp; an fp16 result rounded to nearest is within 2^-11 of its value, and
2^-10 leaves room for the fp32 arithmetic before that rounding):
  - InstanceNorm + ReLU, per element: 2^-10 |ref| + 1e-5 |gamma xhat| + 2^-22 (|x s| + |mu s| + |beta|) with
    s = gamma / sqrt(var + eps): the output rounding; statistics within 1e-5 of float64 (the standard of
    test_train_kernels_gpu.py); and the fp32 rounding of the kernel's fma(x, s, beta - mu s), whose two terms are far
    larger than the result when |mean| >> std.  Statistics formed as E[y^2] - mean^2 from fp32 sums fail it at
    mean/std 64 and in near-constant channels.
  - tensor-core stem: 2^-10 |ref| + 2^-20 sum |w| |x| over the 147 taps (fp32 accumulation of exact fp16 products)
  - max-pool: exact
  - global average pool: (HW + 1) u mean |x|, the worst case of a sequential fp32 sum scaled by fp32 1/HW; the
    BatchNorm1d head: one fp32 rounding of feat * scale + shift, evaluated from the device's own feat."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
EPS = 1e-5


def _n():
    from ctl_b200 import _native as N

    return N, N.lib()


def _bits(t):
    t = t.contiguous()
    return t.view({torch.float16: torch.int16, torch.float32: torch.int32}[t.dtype])


def _report(err, tol):
    bad = err > tol
    return (f"{int(bad.sum())} / {bad.numel()} off; max err/budget {float((err / tol).max()):.3f}; first bad index "
            f"{bad.nonzero()[0].tolist() if bad.any() else None}")


# ===================================================================================================================
# 1. ctl_instnorm_relu_nhwc_f16: InstanceNorm(affine) + ReLU in place on channels [0, half) of [n][hw][2 half]
# ===================================================================================================================
IN_SHAPES = [
    # n, hw, half: conv1 of every IBN-a block runs at the block's input map (layer2.0 / layer3.0: the previous layer's)
    (2, 2048, 32), (3, 2048, 64), (2, 512, 64), (3, 512, 128), (1, 128, 128),     # 256x128 crop
    (2, 6400, 32), (1, 6400, 64), (3, 1600, 64), (2, 1600, 128), (3, 400, 128),   # 320x320 crop
    (3, 32, 128),                                                                # 128x64 crop
    (2, 1, 64), (3, 255, 64), (1, 256, 64), (2, 257, 64),                        # both sides of the 256-thread row loop
    (128, 400, 128),                                                             # 320x320 eval batch: gridDim.y = 128
]
IN_CASES = [(n, hw, half, ratio, 1.0) for n, hw, half in IN_SHAPES for ratio in (0, 8, 64, 256)]
IN_CASES.append((2, 240, 64, 0.15, 2.0))  # 2 x 20 x 12 map of N(0.3, 2) values


@pytest.mark.parametrize("n,hw,half,ratio,scale", IN_CASES)
def test_instnorm_relu(n, hw, half, ratio, scale):
    """Channel j < half holds (N(0, 1) + ratio) * scale, i.e. mean/std = ratio, except channel 1, constant but for 1 %
    of its pixels (a near-uniform region), and channel 2, exactly constant (variance 0: the output is relu(beta));
    a third of the gammas are negative.  Channels [half, 2 half) must come back bit for bit."""
    N, L = _n()
    c = 2 * half
    g = torch.Generator().manual_seed(hw * 1009 + half * 17 + n + int(ratio))
    x = torch.randn(n, hw, c, generator=g) * 2
    x[..., :half] = (torch.randn(n, hw, half, generator=g) + ratio) * scale
    const = (ratio + 0.3) * scale
    x[..., 1] = const
    few = torch.randperm(hw, generator=g)[:max(1, hw // 100)]
    x[:, few, 1] = const + torch.randn(n, len(few), generator=g) * scale
    x[..., 2] = const
    x = x.half()
    sign = torch.where(torch.rand(half, generator=g) < 1 / 3, -1.0, 1.0)
    gamma, beta = (torch.rand(half, generator=g) + 0.5) * sign, torch.randn(half, generator=g) * 0.2

    xd = x[..., :half].double()
    gd, bd = gamma.double(), beta.double()
    mu, var = xd.mean(1, keepdim=True), xd.var(1, unbiased=False, keepdim=True)
    assert (var[:, 0, 2] == 0).all()
    rstd = 1 / torch.sqrt(var + EPS)
    xhat = (xd - mu) * rstd
    s = gd * rstd
    ref = (gd * xhat + bd).clamp(min=0)
    tol = 2.0 ** -10 * ref.abs() + 1e-5 * (gd * xhat).abs() + 2.0 ** -22 * ((xd * s).abs() + (mu * s).abs() + bd.abs())

    xc, gc, bc = x.cuda(), gamma.cuda(), beta.cuda()
    N.check(L.ctl_instnorm_relu_nhwc_f16(xc.data_ptr(), n, hw, c, half, gc.data_ptr(), bc.data_ptr(), EPS, N.stream_ptr()))
    torch.cuda.synchronize()
    got = xc.cpu()
    assert torch.equal(_bits(got[..., half:]), _bits(x[..., half:])), "InstanceNorm wrote into the BatchNorm half"
    o = got[..., :half].double()
    assert torch.isfinite(o).all(), "non-finite outputs"
    err = (o - ref).abs()
    assert not (err > tol).any(), _report(err, tol)


# ===================================================================================================================
# 2. ctl_maxpool3x3s2_nhwc_f16: 3x3 / 2, pad 1, on the tensor-core stem's output (64 channels)
# ===================================================================================================================
def _fill_window(x, oh, ow, chans, value):
    """Sets every in-bounds tap of output (oh, ow)'s window to `value` in channels `chans`."""
    h, w = x.shape[1:3]
    x[:, max(2 * oh - 1, 0):min(2 * oh + 2, h), max(2 * ow - 1, 0):min(2 * ow + 2, w), chans] = value


@pytest.mark.parametrize("n,h,w,relu", [
    (8, 160, 160, 0),  # 320x320 input
    (2, 55, 31, 0),    # 110x62 input: odd sides
    (3, 7, 5, 0), (2, 2, 3, 0), (2, 1, 1, 0),
    (3, 32, 24, 1),    # a 64x48 input's stem, after ReLU (IBN-a)
])
def test_maxpool3x3s2(n, h, w, relu):
    """== F.max_pool2d exactly.  Without ReLU (ResNet50's stem) the inputs are negative as often as not, and some
    windows (corners, centre) are all -65504 or all -inf (fp16 overflow) in some channels."""
    N, L = _n()
    g = torch.Generator().manual_seed(n * 1000 + h * 7 + w)
    x = torch.randn(n, h, w, 64, generator=g) * 4
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    if relu:
        x = x.clamp(min=0)
    else:
        for i, (oh, ow) in enumerate(dict.fromkeys([(0, 0), (ho - 1, wo - 1), (ho // 2, wo // 2)])):
            _fill_window(x, oh, ow, list(range(8)) + [20 + i], float("-inf"))
            _fill_window(x, oh, ow, list(range(8, 16)) + [40 + i], -65504.0)
    x = x.half()
    ref = F.max_pool2d(x.float().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    if not relu:
        assert (ref == float("-inf")).any() and (ref == -65504.0).any()
    xc = x.cuda()
    out = torch.full((n, ho, wo, 64), float("nan"), dtype=torch.float16, device="cuda")
    N.check(L.ctl_maxpool3x3s2_nhwc_f16(xc.data_ptr(), n, h, w, 64, out.data_ptr(), N.stream_ptr()))
    torch.cuda.synchronize()
    got = out.cpu().float()
    bad = got != ref
    assert not bad.any(), f"{int(bad.sum())} / {bad.numel()} off; first bad [n, h, w, c] {bad.nonzero()[0].tolist()}"


# ===================================================================================================================
# 3. ctl_stem_conv7x7_tc: conv 7x7 / 2, pad 3, 3 -> 64 (+bias, optional ReLU), fp32 NCHW in, fp16 NHWC out
# ===================================================================================================================
@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("n,h,w", [(4, 320, 320), (3, 110, 62), (2, 255, 127), (1, 7, 7), (3, 64, 48)])
def test_stem_conv7x7_tc(n, h, w, relu):
    """The stem of every input wider than the fused stem takes (e.g. 320x320), and odd sides whose output tiles
    (4 x 32 pixels) are partial; the kernel rounds the input and the weights to fp16, as the reference here does."""
    N, L = _n()
    g = torch.Generator().manual_seed(n * 1000 + h + w)
    x = torch.randn(n, 3, h, w, generator=g)
    wt = torch.randn(64, 3, 7, 7, generator=g) * 0.1
    b = torch.randn(64, generator=g) * 0.1
    x16, w16 = x.half().double(), wt.half().double()
    ref = F.conv2d(x16, w16, b.double(), 2, 3)
    if relu:
        ref = ref.clamp(min=0)
    mag = F.conv2d(x16.abs(), w16.abs(), None, 2, 3)
    ho, wo = ref.shape[2:]
    # operand [64][192]: k = (c * 7 + r) * 8 + s, s = 7 and k >= 168 zero
    wk192 = torch.zeros(64, 21, 8)
    wk192[:, :, :7] = wt.reshape(64, 21, 7)
    wk192 = torch.cat((wk192.reshape(64, 168), torch.zeros(64, 24)), 1).half().cuda()
    xc, bc = x.cuda(), b.cuda()
    out = torch.full((n, ho, wo, 64), float("nan"), dtype=torch.float16, device="cuda")
    N.check(L.ctl_stem_conv7x7_tc(xc.data_ptr(), n, h, w, wk192.data_ptr(), bc.data_ptr(), relu, out.data_ptr(),
                                  N.stream_ptr()))
    torch.cuda.synchronize()
    got = out.cpu().double().permute(0, 3, 1, 2)
    assert torch.isfinite(got).all(), "unwritten or non-finite outputs"
    err = (got - ref).abs()
    tol = 2.0 ** -10 * ref.abs() + 2.0 ** -20 * mag
    assert not (err > tol).any(), _report(err, tol)


# ===================================================================================================================
# 4. ctl_gap_bn_nhwc_f16: feat = mean over hw (fp32), emb = feat * scale + shift (folded eval BatchNorm1d)
# ===================================================================================================================
GAP_CASES = [(3, hw, c) for hw in (1, 32, 128, 400, 2048) for c in (512, 2048, 514)]  # 514: a partial last block
GAP_CASES += [(1, 2048, 2048), (1, 1, 514), (4, 128, 2048),
              (256, 128, 2048),  # the ResNet50 bench batch: 256 x layer4's 16 x 8 map
              (256, 32, 514)]


@pytest.mark.parametrize("data", ["zero_mean", "relu"])
@pytest.mark.parametrize("n,hw,c", GAP_CASES)
def test_gap_bn(n, hw, c, data):
    """feat only, emb only and both; zero-mean inputs and post-ReLU ones up to ~1e3 (where a sum that dropped or
    repeated a pixel, or accumulated in fp16, is far outside the fp32 bound)."""
    N, L = _n()
    g = torch.Generator().manual_seed(n * 100000 + hw * 10 + c)
    x = torch.randn(n, hw, c, generator=g)
    x = (x * 2 if data == "zero_mean" else x.clamp(min=0) * 300).half()
    scale, shift = torch.randn(c, generator=g), torch.randn(c, generator=g)
    xd = x.double()
    mu = xd.mean(1)
    feat_tol = (hw + 1) * U32 * xd.abs().mean(1)
    del xd

    xc, sc, shc = x.cuda(), scale.cuda(), shift.cuda()

    def run(want_feat, want_emb):
        feat = torch.full((n, c), float("nan"), device="cuda") if want_feat else None
        emb = torch.full((n, c), float("nan"), device="cuda") if want_emb else None
        N.check(L.ctl_gap_bn_nhwc_f16(xc.data_ptr(), n, hw, c, sc.data_ptr(), shc.data_ptr(), N.ptr(feat), N.ptr(emb),
                                      N.stream_ptr()))
        torch.cuda.synchronize()
        return (feat.cpu() if want_feat else None), (emb.cpu() if want_emb else None)

    feat_only, _ = run(True, False)
    _, emb_only = run(False, True)
    feat, emb = run(True, True)
    assert torch.isfinite(feat).all() and torch.isfinite(emb).all(), "unwritten or non-finite outputs"
    err = (feat.double() - mu).abs()
    assert not (err > feat_tol).any(), "feat: " + _report(err, feat_tol)
    ref = feat.double() * scale.double() + shift.double()
    err, tol = (emb.double() - ref).abs(), U32 * (1 + 2.0 ** -20) * ref.abs()
    assert not (err > tol).any(), "emb: " + _report(err, tol)
    assert torch.equal(_bits(feat_only), _bits(feat)), "feat differs with and without emb"
    assert torch.equal(_bits(emb_only), _bits(emb)), "emb differs with and without feat"
