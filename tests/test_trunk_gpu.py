"""GPU parity tests of the trunk inference forward (csrc/conv.cu) through the C ABI.

Checker for single ops: float64 torch-CPU convolution of the SAME fp16-rounded operands (so
only the fp32 accumulation order and the final fp16 rounding differ): tolerance 1 fp16 ulp of
the output magnitude (2^-10 relative) + 1e-3 absolute.
Checker for the whole trunk: oracle.trunk_forward_fp16sim (same rounding points), tolerance
3e-3 of the feature scale; and the fp32 reference's golden features within 1e-2 (an fp16
trunk cannot meet 1e-4 against fp32 -- SURVEY section 7; DESIGN.md 'Parity')."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden
from oracle import ctl_oracle as O

pytestmark = pytest.mark.gpu


def _conv_case(n, h, w, cin, cout, k, stride, relu, residual, relu_from=0, seed=0):
    from ctl_b200 import _native as N

    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, h, w, cin, generator=g) * 0.5).half()
    wt = (torch.randn(cout, k, k, cin, generator=g) / (k * (cin ** 0.5))).half()
    bias = torch.randn(cout, generator=g) * 0.1
    pad = 1 if k == 3 else 0
    ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    res = (torch.randn(n, ho, wo, cout, generator=g) * 0.5).half() if residual else None
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), wt.double().permute(0, 3, 1, 2), bias.double(), stride, pad)
    ref = ref.permute(0, 2, 3, 1)
    if res is not None:
        ref = ref + res.double()
    if relu:
        ref[..., relu_from:] = ref[..., relu_from:].clamp(min=0)
    xd, wd, bd = x.cuda(), wt.cuda(), bias.cuda()
    rd = res.cuda() if res is not None else None
    out = torch.full((n, ho, wo, cout), float("nan"), dtype=torch.float16, device="cuda")
    N.check(N.lib().ctl_conv2d_nhwc_f16(xd.data_ptr(), n, h, w, cin, wd.data_ptr(), bd.data_ptr(), N.ptr(rd),
                                        out.data_ptr(), cout, k, stride, int(relu), relu_from, N.stream_ptr()))
    torch.cuda.synchronize()
    got = out.cpu().double()
    assert torch.isfinite(got).all(), "unwritten or non-finite outputs"
    err = (got - ref).abs()
    tol = ref.abs() * 2.0 ** -10 + 1e-3
    bad = err > tol
    assert not bad.any(), (f"{int(bad.sum())} / {bad.numel()} outputs off; max err {float(err.max()):.4e}; first bad "
                           f"index {bad.nonzero()[0].tolist()}")


@pytest.mark.parametrize("case", [
    # n, h, w, cin, cout, k, stride, relu, residual
    (2, 64, 32, 64, 64, 1, 1, True, False),
    (2, 64, 32, 64, 256, 1, 1, True, True),
    (2, 64, 32, 256, 64, 1, 1, True, False),
    (2, 64, 32, 64, 64, 3, 1, True, False),
    (3, 32, 16, 128, 128, 3, 1, True, False),
    (3, 16, 8, 512, 512, 3, 1, True, False),
    (2, 64, 32, 128, 128, 3, 2, True, False),
    (3, 32, 16, 256, 256, 3, 2, True, False),
    (2, 64, 32, 256, 512, 1, 2, False, False),
    (3, 16, 8, 1024, 2048, 1, 1, False, False),
    (3, 16, 8, 2048, 512, 1, 1, True, False),
    (5, 16, 8, 512, 2048, 1, 1, True, True),
    (2, 20, 20, 256, 256, 3, 1, True, False),     # 320x320 geometry: partial tiles
    (1, 80, 80, 64, 64, 3, 1, True, False),
    (2, 40, 40, 128, 128, 3, 2, True, False),
    (1, 7, 5, 64, 128, 3, 1, False, True),        # tiny, heavily over-covered tile
])
def test_conv_shapes(case):
    _conv_case(*case)


@pytest.mark.parametrize("case", [
    # n, ho, wo, cin1, cin2, cout, stride2
    (2, 64, 32, 64, 64, 256, 1),      # layer1.0: conv3 + stride-1 shortcut
    (2, 32, 16, 128, 256, 512, 2),    # layer2.0: shortcut sampled at stride 2
    (4, 16, 8, 256, 512, 1024, 2),
    (2, 16, 8, 512, 1024, 2048, 1),   # layer4.0 with last_stride 1
    (3, 20, 20, 128, 256, 512, 2),    # odd tile count -> single-CTA kernel, partial tiles
    (1, 6, 5, 64, 64, 128, 1),
])
def test_conv_dual_shortcut(case):
    """ctl_conv1x1_dual_nhwc_f16 == relu(W3 x1 + Wd x2[::s, ::s] + b) in float64 on the same fp16 operands."""
    from ctl_b200 import _native as N

    n, ho, wo, c1, c2, cout, s2 = case
    g = torch.Generator().manual_seed(n * 1000 + cout)
    x1 = (torch.randn(n, ho, wo, c1, generator=g) * 0.5).half()
    x2 = (torch.randn(n, ho * s2, wo * s2, c2, generator=g) * 0.5).half()
    w = (torch.randn(cout, c1 + c2, generator=g) / ((c1 + c2) ** 0.5)).half()
    bias = torch.randn(cout, generator=g) * 0.1
    ref = torch.einsum("nhwc,oc->nhwo", x1.double(), w[:, :c1].double()) + \
        torch.einsum("nhwc,oc->nhwo", x2[:, ::s2, ::s2].double(), w[:, c1:].double()) + bias.double()
    ref = ref.clamp(min=0)
    x1d, x2d, wd, bd = x1.cuda(), x2.cuda(), w.cuda(), bias.cuda()
    out = torch.full((n, ho, wo, cout), float("nan"), dtype=torch.float16, device="cuda")
    N.check(N.lib().ctl_conv1x1_dual_nhwc_f16(x1d.data_ptr(), c1, x2d.data_ptr(), ho * s2, wo * s2, c2, s2, n,
                                              wd.data_ptr(), bd.data_ptr(), out.data_ptr(), cout, 1, N.stream_ptr()))
    torch.cuda.synchronize()
    got = out.cpu().double()
    assert torch.isfinite(got).all(), "unwritten or non-finite outputs"
    err = (got - ref).abs()
    bad = err > ref.abs() * 2.0 ** -10 + 1e-3
    assert not bad.any(), f"{int(bad.sum())} / {bad.numel()} outputs off; max err {float(err.max()):.4e}"


def test_conv_residual_many_tiles():
    """Residual layers at a size where every CTA pair walks several tiles and n-tiles: the staging-slab ring (5 slabs,
    residual prefetched 3 sub-tiles ahead) wraps many times and crosses tile boundaries."""
    _conv_case(64, 16, 8, 512, 2048, 1, 1, True, True, seed=9)
    _conv_case(48, 32, 16, 128, 512, 1, 1, True, True, seed=10)
    _conv_case(16, 32, 16, 128, 128, 3, 1, False, True, seed=11)   # 128-wide pair tile with a residual (training dgrad)


def test_conv_relu_from_channel():
    _conv_case(2, 32, 16, 256, 128, 1, 1, True, False, relu_from=64, seed=3)


@pytest.mark.parametrize("tag,ibn,hw", [("r50", False, (256, 128)), ("ibn", True, (128, 64))])
def test_full_trunk_matches_checker_and_reference_golden(tag, ibn, hw):
    from ctl_b200.modelling.backbones.engine import TrunkEngine

    g = load_golden("trunk.npz")
    sd = O.make_trunk_state(seed=7, ibn=ibn)
    x = torch.randn(2, 3, *hw, generator=torch.Generator().manual_seed(21))
    head = dict(weight=torch.rand(2048) + 0.5, bias=torch.randn(2048) * 0.1, running_mean=torch.randn(2048) * 0.1,
                running_var=torch.rand(2048) + 0.5)
    eng = TrunkEngine(sd, "cuda", ibn=ibn, bn_head=head)
    out = eng.forward(x.cuda(), want_emb=True)
    feat = out["global_feat"].cpu()
    with torch.no_grad():
        _, sim = O.trunk_forward_fp16sim(x, sd, ibn=ibn)
    scale = float(sim.abs().max())
    err_sim = float((feat - sim).abs().max())
    err_ref = float((feat - torch.from_numpy(g[f"{tag}_eval_feat"])).abs().max())
    print(f"{tag}: |feat|max {scale:.4f}  err vs fp16-sim {err_sim:.3e}  err vs fp32 reference {err_ref:.3e}")
    assert err_sim <= 3e-3 * scale
    assert err_ref <= 1e-2 * scale
    emb_ref = F.batch_norm(feat, head["running_mean"], head["running_var"], head["weight"], head["bias"], False, 0.1, 1e-5)
    np.testing.assert_allclose(out["emb"].cpu().numpy(), emb_ref.numpy(), rtol=1e-5, atol=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 64, 48), (2, 256, 128), (40, 64, 32), (5, 128, 64), (1, 8, 8)])
def test_stem_pool_fused(shape):
    """conv1 + folded bn1 (+ReLU) + maxpool in one kernel (wgmma windows over raw input rows) against the fp16-operand
    convolution followed by max_pool2d; ranges that start inside an image and cross images are both exercised."""
    from ctl_b200 import _native as N
    from ctl_b200.modelling.backbones.engine import pack_stem_fused

    L = N.lib()
    n, H, W = shape
    g = torch.Generator().manual_seed(11)
    x = torch.randn(n, 3, H, W, generator=g)
    w = torch.randn(64, 3, 7, 7, generator=g) * 0.1
    b = torch.randn(64, generator=g) * 0.1
    xd, bd, wd = x.cuda(), b.cuda(), pack_stem_fused(w.cuda())
    pad = torch.zeros(L.ctl_stem_pad_bytes(n, H, W), dtype=torch.uint8, device="cuda")
    for relu in (0, 1):
        ref = F.conv2d(x.half().double(), w.half().double(), b.double(), 2, 3)
        if relu:
            ref = ref.clamp(min=0)
        refp = F.max_pool2d(ref, 3, 2, 1)
        hp, wp = refp.shape[2:]
        out = torch.full((n, hp, wp, 64), float("nan"), dtype=torch.float16, device="cuda")
        for _ in range(2):  # the second call reuses the staging buffer (borders must still be zero)
            N.check(L.ctl_stem_pool_fused(xd.data_ptr(), n, H, W, pad.data_ptr(), wd.data_ptr(), bd.data_ptr(), relu,
                                          out.data_ptr(), N.stream_ptr()))
        torch.cuda.synchronize()
        got = out.cpu().double().permute(0, 3, 1, 2)
        assert torch.isfinite(got).all()
        assert float((got - refp).abs().max()) <= float(refp.abs().max()) * 2.0 ** -10 + 1e-4


@pytest.mark.parametrize("tag,ibn,hw,big", [("r50", False, (256, 128), 256), ("ibn", True, (320, 320), 128)])
def test_batch_invariance_at_bench_shapes(tag, ibn, hw, big):
    """The bench configurations themselves (256 x 256x128 ResNet50 = metric M1; 128 x 320x320 IBN-a = config 4's per-GPU
    eval shape): image i of the big batch must be BIT-IDENTICAL to the same image run in a batch of 2 -- the kernels
    are deterministic and no reduction crosses images, so different persistent tile ranges / CTA-pair waves must not
    change a single bit.  The small batch is the one the reference goldens pin (test_full_trunk_...)."""
    from ctl_b200.modelling.backbones.engine import GraphedForward, TrunkEngine

    sd = O.make_trunk_state(seed=7, ibn=ibn)
    head = dict(weight=torch.rand(2048) + 0.5, bias=torch.randn(2048) * 0.1, running_mean=torch.randn(2048) * 0.1,
                running_var=torch.rand(2048) + 0.5)
    eng = TrunkEngine(sd, "cuda", ibn=ibn, bn_head=head)
    x = torch.randn(big, 3, *hw, generator=torch.Generator().manual_seed(33)).cuda()
    full = eng.forward(x, want_emb=True)
    feat, emb = full["global_feat"].clone(), full["emb"].clone()
    assert torch.isfinite(feat).all()
    for lo in (0, big // 2 - 1, big - 2):
        small = eng.forward(x[lo:lo + 2].contiguous(), want_emb=True)
        assert torch.equal(small["global_feat"], feat[lo:lo + 2]), f"{tag}: images {lo},{lo + 1} differ between batch {big} and 2"
        assert torch.equal(small["emb"], emb[lo:lo + 2])
    # the CUDA-graph replay the bench times is the same computation
    graphed = GraphedForward(eng, x, want_emb=True)()
    assert torch.equal(graphed["emb"], emb)


# north_star asks for 1e-4 relative on fp32 embeddings.  The reference's own configs run the trunk under fp16 autocast
# (USE_MIXED_PRECISION, utils/misc.py:111), and the REFERENCE ITSELF then sits 3.9e-4 (R50 256x128) / 4.9e-4 (IBN-a
# 320x320) / 6.7e-4 (IBN-a 128x64) of the feature scale away from its fp32 run (tests/golden/trunk_autocast.npz,
# `*_amp_vs_fp32`, produced by oracle/make_golden.py from the unmodified reference).  An fp16 trunk is therefore pinned
# against the reference AT ITS OWN PRECISION: the engine must be as close to the reference-under-autocast as two correct
# fp16 evaluations of the same network are to each other, and not further from fp32 than 3x the reference's own distance.
AMP_TOL = 2e-3


@pytest.mark.parametrize("tag,ibn,hw", [("r50", False, (256, 128)), ("ibn320", True, (320, 320)), ("ibn", True, (128, 64))])
def test_trunk_matches_reference_under_autocast(tag, ibn, hw):
    from ctl_b200.modelling.backbones.engine import TrunkEngine

    g = load_golden("trunk_autocast.npz")
    sd = O.make_trunk_state(seed=7, ibn=ibn)
    x = torch.randn(2, 3, *hw, generator=torch.Generator().manual_seed(21))
    t = x.double()
    np.testing.assert_allclose(np.array([float(t.sum()), float((t * t).sum())]), g[f"{tag}_in_checksum"], rtol=1e-9)
    feat = TrunkEngine(sd, "cuda", ibn=ibn).forward(x.cuda())["global_feat"].cpu()
    amp, f32 = torch.from_numpy(g[f"{tag}_eval_feat_amp"]), torch.from_numpy(g[f"{tag}_eval_feat_fp32"])
    scale = float(f32.abs().max())
    e_amp = float((feat - amp).abs().max()) / scale
    e_f32 = float((feat - f32).abs().max()) / scale
    ref_own = float(g[f"{tag}_amp_vs_fp32"])
    print(f"{tag}: engine vs reference-under-autocast {e_amp:.3e}; engine vs reference fp32 {e_f32:.3e}; "
          f"reference autocast vs its own fp32 {ref_own:.3e}  (north_star 1e-4 is an fp32-vs-fp32 bound)")
    assert e_amp <= AMP_TOL
    assert e_f32 <= 3.0 * ref_own


@pytest.mark.parametrize("ibn,hw,n", [(False, (256, 128), 6), (True, (320, 320), 3), (True, (128, 64), 5), (False, (96, 48), 2)])
def test_trunk_stage_calls_match_embed_forward(ibn, hw, n):
    """SURVEY 8b: TrunkEngine's three stage calls (ctl_embed_stem -> ctl_embed_blocks -> ctl_embed_head) must reproduce
    ctl_embed_forward, the one-call entry point for C hosts, on the same handle BIT FOR BIT and with the same launch
    count, with and without the BatchNorm1d head, across re-packs."""
    from ctl_b200 import _native as N
    from ctl_b200.modelling.backbones.engine import TrunkEngine

    L = N.lib()
    sd = O.make_trunk_state(seed=5, ibn=ibn)
    head = dict(weight=torch.rand(2048) + 0.5, bias=torch.randn(2048) * 0.1, running_mean=torch.randn(2048) * 0.1,
                running_var=torch.rand(2048) + 0.5)
    x = torch.randn(n, 3, *hw, generator=torch.Generator().manual_seed(8)).cuda()
    eng = TrunkEngine(sd, "cuda", ibn=ibn, bn_head=head)
    ws = torch.empty(L.ctl_embed_workspace_bytes(eng._h, n, *hw), dtype=torch.uint8, device="cuda")

    def embed_forward(want_emb):
        feat = torch.empty(n, 2048, device="cuda")
        emb = torch.empty(n, 2048, device="cuda") if want_emb else None
        N.check(L.ctl_embed_forward(eng._h, x.data_ptr(), n, hw[0], hw[1], feat.data_ptr(), N.ptr(emb), ws.data_ptr(),
                                    ws.numel(), N.stream_ptr()))
        return feat, emb

    out = eng.forward(x, want_emb=True)
    feat, emb = embed_forward(True)
    assert torch.equal(out["global_feat"], feat) and torch.equal(out["emb"], emb)
    assert L.ctl_embed_launches(eng._h) == eng.launches_per_forward
    eng.pack(O.make_trunk_state(seed=6, ibn=ibn))  # re-pack (parameters changed), this time without a head
    out2 = eng.forward(x, want_emb=True)
    assert "emb" not in out2
    feat2, _ = embed_forward(False)
    assert torch.equal(out2["global_feat"], feat2) and not torch.equal(feat2, feat)
    with pytest.raises(ValueError, match="bn_head"):
        N.check(L.ctl_embed_forward(eng._h, x.data_ptr(), n, hw[0], hw[1], feat.data_ptr(), emb.data_ptr(), ws.data_ptr(),
                                    ws.numel(), N.stream_ptr()))
    bad = {k: v for k, v in sd.items() if k != "layer2.1.bn2.running_var"}
    with pytest.raises(ValueError, match="layer2.1.bn2.running_var"):
        eng.pack(bad)


@pytest.mark.parametrize("tag,layers,ibn,hw", [
    ("r101", (3, 4, 23, 3), False, (128, 64)),
    ("r101_ibn", (3, 4, 23, 3), True, (128, 64)),
    # 110 x 62 takes the tensor-core stem, whose conv output (55 x 31) has odd sides: layer1's output is then larger
    # than the stem's, and the workspace must be sized for it
    ("r50_odd_stem", (3, 4, 6, 3), False, (110, 62)),
])
def test_trunk_variants_match_checker(tag, layers, ibn, hw):
    """The deeper trunks Baseline evaluates (MODEL.NAME resnet101 / resnet101_ibn_a) through the same handle, against
    the fp16-rounding checker at the tolerance of test_full_trunk_matches_checker_and_reference_golden."""
    from ctl_b200.modelling.backbones.engine import TrunkEngine

    sd = O.make_trunk_state(seed=7, ibn=ibn, layers=layers)
    x = torch.randn(2, 3, *hw, generator=torch.Generator().manual_seed(21))
    feat = TrunkEngine(sd, "cuda", ibn=ibn, layers=layers).forward(x.cuda())["global_feat"].cpu()
    with torch.no_grad():
        _, sim = O.trunk_forward_fp16sim(x, sd, ibn=ibn, layers=layers)
    scale = float(sim.abs().max())
    err = float((feat - sim).abs().max())
    print(f"{tag}: |feat|max {scale:.4f}  err vs fp16-sim {err:.3e}")
    assert err <= 3e-3 * scale


def test_bottlenecks_never_write_their_input():
    """bench.py replays the bottleneck segment many times on one stem output: the segment must leave it untouched and
    compute the same bits every time."""
    from ctl_b200.modelling.backbones.engine import TrunkEngine

    eng = TrunkEngine(O.make_trunk_state(seed=3), "cuda")
    x = torch.randn(4, 3, 256, 128, generator=torch.Generator().manual_seed(2)).cuda()
    a, n, h, w = eng.stem(x)
    before = a.clone()
    y1, h1, w1 = eng.bottlenecks(a, n, h, w)
    y1 = y1.clone()
    y2, h2, w2 = eng.bottlenecks(a, n, h, w)
    assert torch.equal(a, before)
    assert (h1, w1) == (h2, w2) and torch.equal(y1, y2)


def test_graph_outlives_calls_at_other_shapes():
    """A CUDA graph captured at one input shape reads the handle's stem staging buffer and its own workspace: both must
    stay valid after eager forwards and captures at other shapes (fused and tensor-core stems)."""
    from ctl_b200.modelling.backbones.engine import GraphedForward, TrunkEngine

    head = dict(weight=torch.rand(2048) + 0.5, bias=torch.randn(2048) * 0.1, running_mean=torch.randn(2048) * 0.1,
                running_var=torch.rand(2048) + 0.5)
    eng = TrunkEngine(O.make_trunk_state(seed=4), "cuda", bn_head=head)
    gen = torch.Generator().manual_seed(6)
    xa = torch.randn(4, 3, 128, 64, generator=gen).cuda()
    ga = GraphedForward(eng, xa, want_emb=True)
    for shape in ((2, 3, 96, 48), (3, 3, 64, 160)):
        xb = torch.randn(*shape, generator=gen).cuda()
        eng.forward(xb, want_emb=True)
        gb = GraphedForward(eng, xb, want_emb=True)
        assert torch.equal(gb()["emb"], eng.forward(xb, want_emb=True)["emb"])
    torch.cuda.synchronize()
    out = ga()
    ref = eng.forward(xa, want_emb=True)
    assert torch.equal(out["emb"], ref["emb"]) and torch.equal(out["global_feat"], ref["global_feat"])


@pytest.mark.parametrize("ibn,shape", [(False, (6, 256, 128)), (True, (3, 64, 32)), (False, (2, 96, 160))])
def test_forward_u8_matches_normalize_then_forward(ibn, shape):
    """TrunkEngine.forward_u8 (ToTensor + Normalize folded into the fused stem's input packing, ctl_stem_pool_fused_u8)
    == forward(normalize_batch(images)) bit for bit: the same IEEE (u / 255 - mean) / std, rounded to fp16 once.
    (96 x 160: wider than the fused stem takes -> the normalize_batch route.)"""
    from ctl_b200.datasets.transforms import normalize_batch
    from ctl_b200.modelling.backbones.engine import TrunkEngine

    n, H, W = shape
    sd = O.make_trunk_state(seed=9, ibn=ibn)
    head = dict(weight=torch.rand(2048) + 0.5, bias=torch.randn(2048) * 0.1, running_mean=torch.randn(2048) * 0.1,
                running_var=torch.rand(2048) + 0.5)
    eng = TrunkEngine(sd, "cuda", ibn=ibn, bn_head=head)
    img = torch.randint(0, 256, (n, H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(4)).cuda()
    a = eng.forward_u8(img, want_emb=True)
    b = eng.forward(normalize_batch(img), want_emb=True)
    assert torch.equal(a["global_feat"], b["global_feat"]) and torch.equal(a["emb"], b["emb"])
    with pytest.raises(ValueError, match="uint8"):
        eng.forward_u8(img.float())
