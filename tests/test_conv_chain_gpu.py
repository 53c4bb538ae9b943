"""GPU: ctl_conv1x1_chain_nhwc_f16 (a bottleneck's last 1x1 and the next block's conv1 in one launch) against the two
stand-alone launches it replaces, on the same fp16 operands.  The chained launch adds no rounding point and keeps the
k order and wgmma shape of the stand-alone conv1, so both outputs must be bit-identical (torch.equal)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _chain_case(n, ho, wo, cin1, cout, cout2, form, stride2=1, relu_from2=0, seed=0):
    """form: "dual" (K-concatenated shortcut x2 read at stride2), "res" (residual) or "plain" (neither)."""
    from ctl_b200 import _native as N

    L = N.lib()
    assert L.ctl_conv1x1_chain_supported(cout, cout2) == 1
    g = torch.Generator().manual_seed(seed)
    cin2 = cin1 * 2 if stride2 == 2 else cin1
    h2, w2 = ho * stride2, wo * stride2
    x1 = (torch.randn(n, ho, wo, cin1, generator=g) * 0.5).half().cuda()
    x2 = (torch.randn(n, h2, w2, cin2, generator=g) * 0.5).half().cuda() if form == "dual" else None
    k1 = cin1 + (cin2 if form == "dual" else 0)
    w = (torch.randn(cout, k1, generator=g) / k1 ** 0.5).half().cuda()
    b = (torch.randn(cout, generator=g) * 0.1).cuda()
    res = (torch.randn(n, ho, wo, cout, generator=g) * 0.5).half().cuda() if form == "res" else None
    w2_ = (torch.randn(cout2, cout, generator=g) / cout ** 0.5).half().cuda()
    b2 = (torch.randn(cout2, generator=g) * 0.1).cuda()
    st = N.stream_ptr()

    ref = torch.full((n, ho, wo, cout), float("nan"), dtype=torch.float16, device="cuda")
    ref2 = torch.full((n, ho, wo, cout2), float("nan"), dtype=torch.float16, device="cuda")
    if form == "dual":
        N.check(L.ctl_conv1x1_dual_nhwc_f16(x1.data_ptr(), cin1, x2.data_ptr(), h2, w2, cin2, stride2, n, w.data_ptr(),
                                            b.data_ptr(), ref.data_ptr(), cout, 1, st))
    else:
        N.check(L.ctl_conv2d_nhwc_f16(x1.data_ptr(), n, ho, wo, cin1, w.data_ptr(), b.data_ptr(), N.ptr(res), ref.data_ptr(),
                                      cout, 1, 1, 1, 0, st))
    N.check(L.ctl_conv2d_nhwc_f16(ref.data_ptr(), n, ho, wo, cout, w2_.data_ptr(), b2.data_ptr(), None, ref2.data_ptr(),
                                  cout2, 1, 1, 1, relu_from2, st))

    out = torch.full_like(ref, float("nan"))
    out2 = torch.full_like(ref2, float("nan"))
    N.check(L.ctl_conv1x1_chain_nhwc_f16(x1.data_ptr(), cin1, N.ptr(x2), h2, w2, cin2 if x2 is not None else 0,
                                         stride2, n, w.data_ptr(), b.data_ptr(), N.ptr(res), out.data_ptr(), cout,
                                         w2_.data_ptr(), b2.data_ptr(), cout2, relu_from2, out2.data_ptr(), st))
    torch.cuda.synchronize()
    assert torch.isfinite(ref2).all() and torch.isfinite(out2).all(), "unwritten outputs"
    assert torch.equal(out, ref), f"block output differs at {int((out != ref).sum())} elements"
    assert torch.equal(out2, ref2), f"chained conv1 output differs at {int((out2 != ref2).sum())} elements"


@pytest.mark.parametrize("case", [
    # n, ho, wo, cin1, cout, cout2, form, stride2 -- the six chained boundaries of ResNet50 at 256x128
    (2, 64, 32, 64, 256, 64, "dual", 1),     # layer1.0 -> layer1.1.conv1
    (2, 64, 32, 64, 256, 64, "res", 1),      # layer1.1 -> layer1.2.conv1
    (2, 64, 32, 64, 256, 128, "res", 1),     # layer1.2 -> layer2.0.conv1
    (3, 32, 16, 128, 512, 128, "dual", 2),   # layer2.0 -> layer2.1.conv1 (shortcut sampled at stride 2)
    (3, 32, 16, 128, 512, 128, "res", 1),    # layer2.1 / layer2.2 -> next conv1
    (2, 32, 16, 128, 512, 128, "plain", 1),  # no residual, no second source
])
def test_chain_boundaries(case):
    _chain_case(*case)


@pytest.mark.parametrize("case", [
    # IBN-a: the InstanceNorm half of the next conv1 stays raw (ReLU from channel cout2 / 2 on)
    (2, 64, 32, 64, 256, 64, "res", 1, 32),
    (2, 32, 16, 128, 512, 128, "res", 1, 64),
    (2, 32, 16, 128, 512, 128, "dual", 2, 64),
])
def test_chain_ibn_relu_from(case):
    _chain_case(*case)


@pytest.mark.parametrize("case", [
    # 320x320 crops: layer1 at 80x80, layer2 at 40x40 -- partial tiles at the image borders
    (2, 80, 80, 64, 256, 64, "dual", 1),
    (2, 80, 80, 64, 256, 128, "res", 1),
    (2, 40, 40, 128, 512, 128, "dual", 2),
    (2, 40, 40, 128, 512, 128, "res", 1),
])
def test_chain_partial_tiles(case):
    _chain_case(*case)


def test_chain_many_tiles():
    """Every CTA walks several m-tiles, each of four n-tiles: the operand ring, the staging slabs and the second
    accumulator cross tile boundaries many times; 144 and 256 m-tiles are not multiples of the 132 SMs."""
    _chain_case(64, 32, 16, 128, 512, 128, "res", seed=5)
    _chain_case(9, 64, 32, 64, 256, 64, "dual", seed=6)
    _chain_case(9, 64, 32, 64, 256, 128, "res", seed=7)
