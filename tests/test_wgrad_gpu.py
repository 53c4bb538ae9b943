"""GPU: the training step's weight-gradient GEMM (ctl_conv2d_wgrad_nhwc_f16[_ex]) and the stem's backward helpers
(im2col, the arg-max max-pool pair), one C entry point at a time, at the geometries and batch sizes of a training step,
against float64 references.

Every entry point is called with the arguments the training trunk passes (csrc/trunk_train.cu::conv_backward / the
stem), and every output buffer and workspace starts as NaN so that an element
the kernel never writes fails the check.

The weight gradient splits the pixel reduction K = n*Ho*Wo into S = `splits` ranges of 128-pixel tiles; each
(work item, range) unit accumulates its tiles with wgmma k16 steps, and the fp32 partial tiles are summed over the
splits in a fixed order.  S comes from ctl_conv2d_wgrad_workspace_bytes (the workspace holds S partial tiles), m_tiles from a
Python copy of pick_tile, and L = 8 * ceil(m_tiles / S) is the number of k16 steps in the longest unit.

Reference: dw[co][r][s][ci] = sum_{n,ho,wo} dy[n,ho,wo,co] * x[n, ho*st + r - pad, wo*st + s - pad, ci], k*k float64
GEMMs on the GPU of the flattened dy against the shifted, strided, zero-padded x, chunked over images; sum |terms| is
the same computation on |dy| and |x|.

Rounding budgets used below (u16 = 2^-11, the half-ulp of an fp16 result rounded to nearest):
  - operands in {-1, 0, +1}: every product and partial sum is an integer below 2^24 (K <= 3.3 M), so any correct
    kernel returns the exact sum whatever its order or rounding; outputs are compared exactly
  - training-like operands: |got - ref| <= 8 * 2^-24 * (sqrt(L) + sqrt(S)) * sum |terms|.  An fp32 chain of L
    additions rounded to nearest errs by about 2^-24 * sqrt(L) * sum |terms| (the S partials add a sqrt(S) term);
    8 is about 5x the 5-sigma error of such a chain.  On same-sign terms a chain that truncates errs by about
    2^-24 * L / 2 * sum |terms| or more.  Measured on an H100 with one wgmma chain per unit, the error was up to
    0.99 * L * 2^-24 * sum |terms| (44x the sqrt(L) unit at L = 2328); the kernel therefore restarts its chain every
    8 pixel tiles (64 k16 steps) and adds the chains with FADD
  - max-pool gradient (at most 4 fp16 terms summed in fp32, rounded once): u16 * |ref| + 2^-22 * sum |terms|."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U16 = 2.0 ** -11
U32 = 2.0 ** -24
SCALE = 2.0 ** -10   # out_scale of the scaled forms: a power of two, so scaling is exact
NAN = float("nan")


def _n():
    from ctl_b200 import _native as N

    return N, N.lib()


def _bits(t):
    t = t.contiguous()
    return t.view({torch.float16: torch.int16, torch.float32: torch.int32}[t.dtype])


def _nan32(*shape):
    return torch.full(shape, NAN, dtype=torch.float32, device="cuda")


def _nan_ws(nbytes):
    """A workspace whose every fp32 word is NaN (0xFFFFFFFF)."""
    return torch.full((nbytes,), 255, dtype=torch.uint8, device="cuda")


def _gen(key):
    return torch.Generator(device="cuda").manual_seed(sum(map(ord, key)) * 7919 + len(key))


# ===================================================================================================================
# 0. float64 reference and the kernel's plan
# ===================================================================================================================
def _ref_wgrad(x, dy, k, stride, absolute=False, chunk_elems=1 << 27):
    """float64 dw [cout][k][k][cin] of NHWC x [n][h][w][cin] and dy [n][ho][wo][cout] (any device): per chunk of
    images, one GEMM per tap of dy^T against the tap's shifted, strided, zero-padded view of x.  absolute=True gives
    sum |terms| instead."""
    n, h, w, cin = x.shape
    _, ho, wo, cout = dy.shape
    pad = k // 2
    out = torch.zeros(cout, k, k, cin, dtype=torch.float64, device=x.device)
    per_img = (h + 2 * pad) * (w + 2 * pad) * cin + ho * wo * (cin + cout)
    step = max(1, chunk_elems // per_img)
    for i in range(0, n, step):
        xc, dc = x[i:i + step].double(), dy[i:i + step].double()
        if absolute:
            xc, dc = xc.abs(), dc.abs()
        xp = F.pad(xc, (0, 0, pad, pad, pad, pad))
        dt = dc.reshape(-1, cout).t()
        for r in range(k):
            for s in range(k):
                xs = xp[:, r:r + stride * (ho - 1) + 1:stride, s:s + stride * (wo - 1) + 1:stride, :]
                out[:, r, s, :] += dt @ xs.reshape(-1, cin)
    return out


def _pick_tile(ho, wo):
    """common.h::pick_tile: the TH x TW = 128 pixel tile of an Ho x Wo map with the least over-covered area."""
    best, bth, btw = -1, 1, 128
    tw = 128
    while tw >= 1:
        th = 128 // tw
        cover = -(-ho // th) * th * -(-wo // tw) * tw
        if best < 0 or cover < best:
            best, bth, btw = cover, th, tw
        tw >>= 1
    return bth, btw


def _plan(L, n, h, w, cin, cout, k, stride, label=""):
    """splits from the workspace size the ABI asks for, m_tiles from pick_tile; printed so that a failure names the
    regime it ran in."""
    pad = k // 2
    ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    th, tw = _pick_tile(ho, wo)
    m_tiles = n * -(-ho // th) * -(-wo // tw)
    cout_pad = -(-cout // 128) * 128
    nbytes = L.ctl_conv2d_wgrad_workspace_bytes(n, h, w, cin, cout, k, stride)
    per_split = cout_pad * k * k * cin * 4
    assert nbytes > 256 and (nbytes - 256) % per_split == 0, (nbytes, per_split)
    splits = (nbytes - 256) // per_split
    n_items = cout_pad // 128 * k * k * (cin // (128 if cin % 128 == 0 else 64))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert 1 <= splits <= m_tiles
    assert splits == max(1, min(-(-2 * sms // n_items), m_tiles)), (splits, n_items, sms, m_tiles)
    per_unit = -(-m_tiles // splits)
    print(f"[wgrad plan] {label} n={n} {h}x{w} {cin}->{cout} k{k} s{stride}: tile {th}x{tw}, m_tiles={m_tiles}, "
          f"splits={splits}, tiles/unit={per_unit}")
    return dict(ho=ho, wo=wo, m_tiles=m_tiles, splits=splits, per_unit=per_unit, L=8 * per_unit, nbytes=nbytes)


@pytest.mark.parametrize("k,stride", [(1, 1), (3, 1), (1, 2), (3, 2)])
def test_reference_matches_conv2d_weight(k, stride):
    """The GPU reference (chunked over images) equals torch.nn.grad.conv2d_weight in CPU float64, bit for bit, on
    integer operands, at small odd and even maps."""
    g = _gen(f"ref{k}{stride}")
    for n, h, w, cin, cout in ((3, 8, 6, 8, 16), (2, 7, 5, 16, 8), (4, 10, 4, 24, 40)):
        if stride == 2 and (h % 2 or w % 2):
            continue
        pad = k // 2
        ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
        x = torch.randint(-3, 4, (n, h, w, cin), generator=g, device="cuda").half()
        dy = torch.randint(-3, 4, (n, ho, wo, cout), generator=g, device="cuda").half()
        want = torch.nn.grad.conv2d_weight(x.cpu().double().permute(0, 3, 1, 2), (cout, cin, k, k),
                                           dy.cpu().double().permute(0, 3, 1, 2), stride=stride,
                                           padding=pad).permute(0, 2, 3, 1)
        got = _ref_wgrad(x, dy, k, stride, chunk_elems=2 * h * w * cin)  # several chunks
        assert torch.equal(got.cpu(), want), (n, h, w, cin, cout)
        mag = _ref_wgrad(x, dy, k, stride, absolute=True)
        want_mag = torch.nn.grad.conv2d_weight(x.cpu().double().abs().permute(0, 3, 1, 2), (cout, cin, k, k),
                                               dy.cpu().double().abs().permute(0, 3, 1, 2), stride=stride,
                                               padding=pad).permute(0, 2, 3, 1)
        assert torch.equal(mag.cpu(), want_mag)


# input maps of the training crops: the stem's output (H/2, W/2) and the inputs of layer1, layer2, layer3 (= layer4's
# with last_stride 1)
MAPS = {"256x128": ((128, 64), (64, 32), (32, 16), (16, 8)),
        "320x320": ((160, 160), (80, 80), (40, 40), (20, 20)),
        "160x80": ((80, 40), (40, 20), (20, 10), (10, 5))}
TRAIN_N = {"256x128": 256, "320x320": 128, "160x80": 64}   # bench default 16x16, config 4 32x4, and a 64-image batch
# weight-gradient GEMM (cin, cout, k, stride) and the MAPS index of its input
GEOMS = {
    "stem_192_64": (192, 64, 1, 1, 0),      # the stem's 7x7 through the im2col GEMM: 3 channel chunks, half a cout tile
    "l1_0_conv1": (64, 64, 1, 1, 1),
    "l1_conv1": (256, 64, 1, 1, 1),
    "l1_conv2": (64, 64, 3, 1, 1),
    "l1_conv3": (64, 256, 1, 1, 1),         # also layer1.0.downsample
    "l2_0_conv2_s2": (128, 128, 3, 2, 1),
    "l2_0_down_s2": (256, 512, 1, 2, 1),
    "l3_0_conv2_s2": (256, 256, 3, 2, 2),
    "l3_conv2": (256, 256, 3, 1, 3),
    "l4_conv2": (512, 512, 3, 1, 3),        # last_stride 1
    "l4_0_conv2_s2": (512, 512, 3, 2, 3),   # last_stride 2
    "l4_conv1": (2048, 512, 1, 1, 3),
    "l4_conv3": (512, 2048, 1, 1, 3),
    "l4_0_down": (1024, 2048, 1, 1, 3),
}
CASES = [(m, gname, n) for m in MAPS for gname in GEOMS for n in (2, TRAIN_N[m])
         # stride 2 needs an even input map (the layer4 10x5 map of 160x80 crops with last_stride 2 is rejected)
         if not (GEOMS[gname][3] == 2 and any(v % 2 for v in MAPS[m][GEOMS[gname][4]]))]
CASES.append(("160x80", "l4_conv2", 1))   # 10x5 map, one image: m_tiles = 1, splits = 1
CASE_IDS = [f"{m}-{gname}-n{n}" for m, gname, n in CASES]


def _case(m, gname, n):
    cin, cout, k, stride, li = GEOMS[gname]
    h, w = MAPS[m][li]
    return n, h, w, cin, cout, k, stride


def _wgrad(N, L, x, dy, n, h, w, cin, cout, k, stride, ws, form):
    """One call in one of the engines' output forms, into a NaN-filled dw.
    raw:   ctl_conv2d_wgrad_nhwc_f16, [cout][k][k][cin] (the stem's call);
    op:    _ex with out_scale = SCALE in the operand layout (the 3x3 form goes through the 1x1 reduction with 9 cin);
    param: _ex with out_scale = SCALE in torch.nn.Conv2d.weight's layout [cout][cin][k][k] (every bottleneck conv)."""
    st = N.stream_ptr()
    if form == "param":
        dw = _nan32(cout, cin, k, k)
    else:
        dw = _nan32(cout, k, k, cin)
    if form == "raw":
        N.check(L.ctl_conv2d_wgrad_nhwc_f16(x.data_ptr(), n, h, w, cin, dy.data_ptr(), cout, k, stride, ws.data_ptr(),
                                            ws.numel(), dw.data_ptr(), st))
    else:
        N.check(L.ctl_conv2d_wgrad_nhwc_f16_ex(x.data_ptr(), n, h, w, cin, dy.data_ptr(), cout, k, stride, ws.data_ptr(),
                                               ws.numel(), dw.data_ptr(), SCALE, int(form == "param"), st))
    torch.cuda.synchronize()
    return dw


# ===================================================================================================================
# 1. coverage: operands in {-1, 0, +1}, exact at every geometry and batch size, in all three output forms
# ===================================================================================================================
@pytest.mark.parametrize("m,gname,n", CASES, ids=CASE_IDS)
def test_wgrad_exact_ternary(m, gname, n):
    """Every pixel tile, tap, parity view, channel chunk, cout tile and split boundary counted exactly once.  A second
    call reproduces the bits after a call of another shape refilled the workspace."""
    N, L = _n()
    n, h, w, cin, cout, k, stride = _case(m, gname, n)
    p = _plan(L, n, h, w, cin, cout, k, stride, f"{m} {gname}")
    if (m, gname, n) == ("160x80", "l4_conv2", 1):
        assert p["m_tiles"] == 1 and p["splits"] == 1
    g = _gen(f"ternary {m} {gname} {n}")
    x = torch.randint(-1, 2, (n, h, w, cin), generator=g, device="cuda", dtype=torch.float16)
    dy = torch.randint(-1, 2, (n, p["ho"], p["wo"], cout), generator=g, device="cuda", dtype=torch.float16)
    ref = _ref_wgrad(x, dy, k, stride).float()   # integers below 2^24: exact in fp32
    # another shape (different splits, m_tiles and tile) that shares the workspace
    other = (3, 12, 10, 128, 128, 3, 1) if (cin, k) != (128, 3) else (3, 12, 10, 64, 192, 1, 1)
    on, oh, ow, oci, oco, ok, ost = other
    xo = torch.randint(-1, 2, (on, oh, ow, oci), generator=g, device="cuda", dtype=torch.float16)
    dyo = torch.randint(-1, 2, (on, oh, ow, oco), generator=g, device="cuda", dtype=torch.float16)
    ws = _nan_ws(max(p["nbytes"], L.ctl_conv2d_wgrad_workspace_bytes(*other)))

    raw = _wgrad(N, L, x, dy, n, h, w, cin, cout, k, stride, ws, "raw")
    bad = raw != ref
    assert not bad.any(), (f"raw: {int(bad.sum())} / {bad.numel()} wrong; first [co, r, s, ci] "
                           f"{bad.nonzero()[0].tolist()}: got {float(raw[bad][0])}, want {float(ref[bad][0])}")
    op = _wgrad(N, L, x, dy, n, h, w, cin, cout, k, stride, ws, "op")
    assert torch.equal(op, ref * SCALE), "operand layout, out_scale 2^-10"
    par = _wgrad(N, L, x, dy, n, h, w, cin, cout, k, stride, ws, "param")
    assert torch.equal(par, (ref * SCALE).permute(0, 3, 1, 2)), "parameter layout, out_scale 2^-10"

    oref = _ref_wgrad(xo, dyo, ok, ost).float()
    assert torch.equal(_wgrad(N, L, xo, dyo, on, oh, ow, oci, oco, ok, ost, ws, "raw"), oref)
    again = _wgrad(N, L, x, dy, n, h, w, cin, cout, k, stride, ws, "raw")
    assert torch.equal(_bits(again), _bits(raw)), "second call after another shape"
    again = _wgrad(N, L, x, dy, n, h, w, cin, cout, k, stride, ws, "param")
    assert torch.equal(_bits(again), _bits(par)), "second parameter-layout call"


# ===================================================================================================================
# 2. rounding budget on training-like operands
# ===================================================================================================================
def _operands(regime, g, xshape, dyshape):
    if regime == "zero_mean":
        x = torch.randn(xshape, generator=g, device="cuda", dtype=torch.float16)
        dy = (torch.randn(dyshape, generator=g, device="cuda") * 2.0 ** -6).half()
    else:   # a saved post-ReLU activation and a gradient with a per-element positive offset
        x = torch.randn(xshape, generator=g, device="cuda", dtype=torch.float16).clamp_(min=0)
        dy = ((0.5 + 0.25 * torch.randn(dyshape, generator=g, device="cuda")) * 2.0 ** -6).half()
    return x, dy


def _check_budget(got, ref, mag, p, label):
    """|got - ref| <= 8 * 2^-24 * (sqrt(L) + sqrt(S)) * sum |terms|; prints the largest err / (2^-24 sqrt(L) sum|t|)."""
    err = (got.double() - ref).abs()
    assert torch.isfinite(got).all(), f"{label}: unwritten or non-finite outputs"
    unit = U32 * math.sqrt(p["L"]) * mag
    ratio = float(torch.where(mag > 0, err / unit.clamp(min=1e-300), torch.zeros_like(err)).max())
    print(f"[wgrad rounding] {label}: L={p['L']} S={p['splits']} max err/(2^-24 sqrt(L) sum|t|) = {ratio:.3f}")
    tol = 8 * U32 * (math.sqrt(p["L"]) + math.sqrt(p["splits"])) * mag
    bad = err > tol
    assert not bad.any(), (f"{label}: {int(bad.sum())} / {bad.numel()} over budget; max err/budget "
                           f"{float((err / tol.clamp(min=1e-300)).max()):.2f}; ratio {ratio:.2f}")
    return ratio


@pytest.mark.parametrize("regime", ["zero_mean", "same_sign"])
@pytest.mark.parametrize("m,gname,n", CASES, ids=CASE_IDS)
def test_wgrad_rounding_budget(m, gname, n, regime):
    """(a) x ~ N(0,1), dy ~ 2^-6 N(0,1); (b) x = relu(N(0,1)), dy = 2^-6 (0.5 + 0.25 N(0,1)): the partial sums grow
    linearly along the chain, so the accumulator's rounding mode shows."""
    N, L = _n()
    n, h, w, cin, cout, k, stride = _case(m, gname, n)
    p = _plan(L, n, h, w, cin, cout, k, stride, f"{m} {gname}")
    x, dy = _operands(regime, _gen(f"{regime} {m} {gname} {n}"), (n, h, w, cin), (n, p["ho"], p["wo"], cout))
    ref = _ref_wgrad(x, dy, k, stride)
    mag = _ref_wgrad(x, dy, k, stride, absolute=True)
    ws = _nan_ws(p["nbytes"])
    got = _wgrad(N, L, x, dy, n, h, w, cin, cout, k, stride, ws, "raw")
    _check_budget(got, ref, mag, p, f"{m} {gname} n={n} {regime}")


# ===================================================================================================================
# 3. the stem's backward at the real shapes: im2col, the im2col weight gradient, the arg-max max-pool pair
# ===================================================================================================================
def _im2col_ref(x):
    """[n*ho*wo][192] fp16 with k = (c*7 + r)*8 + s, s = 7 and k >= 168 zero (the F.unfold construction of
    test_train_gpu.py::test_pool_gap_upsample_im2col_backward_helpers)."""
    n, _, h, w = x.shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    unf = F.unfold(x, 7, padding=3, stride=2).reshape(n, 3, 7, 7, ho * wo).permute(0, 4, 1, 2, 3)
    ref = torch.zeros(n, ho * wo, 3, 7, 8, device=x.device)
    ref[..., :7] = unf
    return torch.cat((ref.reshape(n * ho * wo, 168), torch.zeros(n * ho * wo, 24, device=x.device)), 1).half()


@pytest.mark.parametrize("h,w", [(256, 128), (320, 320), (160, 80), (16, 512), (15, 511)])
def test_stem_im2col_exact(h, w):
    """Bit-exact at the training crops and at the widest row the kernel stages (W = 512) and an odd neighbour."""
    N, L = _n()
    n = 2
    x = torch.randn(n, 3, h, w, generator=_gen(f"im2col {h} {w}"), device="cuda")
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    col = torch.full((n * ho * wo, 192), NAN, dtype=torch.float16, device="cuda")
    N.check(L.ctl_stem_im2col_f16(x.data_ptr(), n, h, w, col.data_ptr(), N.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(_bits(col), _bits(_im2col_ref(x)))


def test_stem_im2col_rejects_unsupported_shapes():
    N, L = _n()
    x = torch.zeros(2, 3, 16, 513, device="cuda")
    col = torch.full((2 * 8 * 257, 192), NAN, dtype=torch.float16, device="cuda")
    for h, w in ((16, 513), (6, 16)):
        with pytest.raises(ValueError):
            N.check(L.ctl_stem_im2col_f16(x.data_ptr(), 2, h, w, col.data_ptr(), N.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.isnan(col.float()).all(), "a rejected call wrote its output"


def test_stem_weight_gradient_as_the_trainer_chains_it():
    """im2col -> wgrad (cin 192, cout 64, 1x1) -> the [64][192] -> [64][3][7][7] unpack, against float64
    conv2d_weight of the fp16-rounded image at 256x128 with n = 256, within the section-2 budget; the padding columns
    (s = 7, k >= 168) come out exactly zero."""
    N, L = _n()
    n, H, W = 256, 256, 128
    h, w = H // 2, W // 2
    g = _gen("stem chain")
    x = torch.rand(n, 3, H, W, generator=g, device="cuda") * 4 - 1   # positive-leaning normalised image
    dy = ((0.5 + 0.25 * torch.randn(n, h, w, 64, generator=g, device="cuda")) * 2.0 ** -6).half()
    col = torch.full((n * h * w, 192), NAN, dtype=torch.float16, device="cuda")
    N.check(L.ctl_stem_im2col_f16(x.data_ptr(), n, H, W, col.data_ptr(), N.stream_ptr()))
    p = _plan(L, n, h, w, 192, 64, 1, 1, "stem chain")
    ws = _nan_ws(p["nbytes"])
    dw = _wgrad(N, L, col, dy, n, h, w, 192, 64, 1, 1, ws, "raw").reshape(64, 192)
    assert torch.equal(_bits(dw[:, 168:]), _bits(torch.zeros(64, 24, device="cuda"))), "k >= 168 not +0"
    pad_s = dw[:, :168].reshape(64, 3, 7, 8)[..., 7]
    assert torch.equal(_bits(pad_s.contiguous()), _bits(torch.zeros_like(pad_s))), "s = 7 not +0"
    got = dw[:, :168].reshape(64, 3, 7, 8)[..., :7]   # stem_train_unpack_kernel's order (before the 1 / loss-scale)
    xd, dyd = x.half().double(), dy.double().permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_weight(xd, (64, 3, 7, 7), dyd, stride=2, padding=3)
    mag = torch.nn.grad.conv2d_weight(xd.abs(), (64, 3, 7, 7), dyd.abs(), stride=2, padding=3)
    _check_budget(got, ref, mag, p, "stem chain 256x128 n=256")


def _pool_ref(x, dy):
    """float64 max-pool 3x3 / 2 / pad 1 backward of NHWC x, dy: each window's gradient to its FIRST maximum in
    window order (r, then s), as torch's max_pool2d; also sum |terms| (the same scatter of |dy|)."""
    n, h, w, c = x.shape
    ho, wo = dy.shape[1], dy.shape[2]
    xn = F.pad(x.double().permute(0, 3, 1, 2), (1, 1, 1, 1), value=float("-inf"))
    win = F.unfold(xn.reshape(n * c, 1, h + 2, w + 2), 3, stride=2).reshape(n, c, 9, ho * wo)
    top = win.max(2, keepdim=True).values
    order = torch.arange(9, device=x.device).view(1, 1, 9, 1)
    first = torch.where(win == top, order, 9).min(2, keepdim=True).values
    onehot = (order == first).double()

    def scatter(d):
        cols = onehot * d.double().permute(0, 3, 1, 2).reshape(n, c, 1, ho * wo)
        out = F.fold(cols.reshape(n * c, 9, ho * wo), (h + 2, w + 2), 3, stride=2)
        return out.reshape(n, c, h + 2, w + 2)[:, :, 1:-1, 1:-1].permute(0, 2, 3, 1)

    return scatter(dy), scatter(dy.abs())


@pytest.mark.parametrize("h,w", [(128, 64), (160, 160), (80, 40), (7, 5)])
def test_maxpool_argmax_pair_with_ties(h, w):
    """Stem-output maps of the three crops and an odd map.  Inputs are full of exact ties (post-ReLU zeros and values
    from {0.5, 1, 1.5}): the pooled output equals F.max_pool2d exactly, and both backward kernels route each window's
    gradient to its first maximum."""
    N, L = _n()
    n, c = 2, 64
    g = _gen(f"pool {h} {w}")
    x = (torch.randint(-2, 4, (n, h, w, c), generator=g, device="cuda") * 0.5).clamp_(min=0).half()
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    dy = torch.randn(n, ho, wo, c, generator=g, device="cuda").half()
    pooled = torch.full((n, ho, wo, c), NAN, dtype=torch.float16, device="cuda")
    arg = torch.full((n, ho, wo, c), 255, dtype=torch.uint8, device="cuda")
    st = N.stream_ptr()
    N.check(L.ctl_maxpool3x3s2_argmax_nhwc_f16(x.data_ptr(), n, h, w, c, pooled.data_ptr(), arg.data_ptr(), st))
    dx = torch.full((n, h, w, c), NAN, dtype=torch.float16, device="cuda")
    N.check(L.ctl_maxpool3x3s2_backward_argmax_nhwc_f16(arg.data_ptr(), dy.data_ptr(), n, h, w, c, dx.data_ptr(), st))
    dx2 = torch.full((n, h, w, c), NAN, dtype=torch.float16, device="cuda")
    N.check(L.ctl_maxpool3x3s2_backward_nhwc_f16(x.data_ptr(), dy.data_ptr(), n, h, w, c, dx2.data_ptr(), st))
    torch.cuda.synchronize()
    want = F.max_pool2d(x.float().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).half()
    assert torch.equal(_bits(pooled), _bits(want)), "pooled output"
    ref, mag = _pool_ref(x, dy)
    tol = U16 * ref.abs() + 2.0 ** -22 * mag
    for name, got in (("argmax pair", dx), ("recomputing backward", dx2)):
        err = (got.double() - ref).abs()
        bad = err > tol
        assert not bad.any(), (f"{name}: {int(bad.sum())} / {bad.numel()} off; first [n, h, w, c] "
                               f"{bad.nonzero()[0].tolist()}")


# ===================================================================================================================
# 4. argument contract
# ===================================================================================================================
def test_wgrad_argument_contract():
    """ValueError, nothing written: a workspace one byte short of what ctl_conv2d_wgrad_workspace_bytes asks for
    (the message names both sizes), dw misaligned by 4 bytes, stride 2 with an odd H or W, cin or cout not a multiple
    of 64.  The workspace query returns 0 for the unsupported shapes."""
    N, L = _n()
    st = N.stream_ptr()
    n, h, w, cin, cout, k, stride = 2, 16, 8, 128, 128, 3, 2
    x = torch.zeros(n, h + 1, w + 1, 2048, dtype=torch.float16, device="cuda")
    dy = torch.zeros(n, h, w, 2048, dtype=torch.float16, device="cuda")
    need = L.ctl_conv2d_wgrad_workspace_bytes(n, h, w, cin, cout, k, stride)
    ws = _nan_ws(need + 64)
    dw = _nan32(cout * k * k * cin + 4)

    def call(n_, h_, w_, ci, co, k_, s_, nbytes=None, dw_ptr=None):
        N.check(L.ctl_conv2d_wgrad_nhwc_f16(x.data_ptr(), n_, h_, w_, ci, dy.data_ptr(), co, k_, s_, ws.data_ptr(),
                                            need if nbytes is None else nbytes, dw.data_ptr() if dw_ptr is None else dw_ptr,
                                            st))

    with pytest.raises(ValueError) as e:
        call(n, h, w, cin, cout, k, stride, nbytes=need - 1)
    assert str(need - 1) in str(e.value) and str(need) in str(e.value), str(e.value)
    with pytest.raises(ValueError):
        call(n, h, w, cin, cout, k, stride, dw_ptr=dw.data_ptr() + 4)
    for bad in ((n, 9, 8, cin, cout, 3, 2), (n, 8, 9, cin, cout, 1, 2), (n, 10, 5, 512, 512, 3, 2),
                (n, h, w, 96, cout, 3, 1), (n, h, w, cin, 96, 1, 1), (n, h, w, 32, 64, 1, 1)):
        assert L.ctl_conv2d_wgrad_workspace_bytes(*bad) == 0, bad
        with pytest.raises(ValueError):
            call(*bad)
    torch.cuda.synchronize()
    assert torch.isnan(dw).all(), "a rejected call wrote dw"
    call(n, h, w, cin, cout, k, stride)   # the exact size is accepted
    torch.cuda.synchronize()
    assert torch.equal(dw[:cout * k * k * cin], torch.zeros_like(dw[:cout * k * k * cin]))
