"""The tile schedule of the unchained convolution GEMM (conv_gemm_kernel<BN, 0>, csrc/conv.cu "Tile order").

With more than one n-tile, CTA c of the grid takes tiles c, c + grid, c + 2 grid, ... of the n-fastest tile order; with
one n-tile, each CTA takes a contiguous range.  Every unchained convolution shape of the ResNet50 256x128 (bench) and
ResNet50-IBN-a 320x320 eval trunks runs here at a batch that keeps the grid below the SM count, next to a single tile and
launches of both kinds whose tile count is not a multiple of the 132-CTA grid.  Each result must
- cover every output element (the output is prefilled with NaN),
- match a float64 convolution of the same fp16 operands within 1 fp16 ulp of the output magnitude + 1e-3, and
- be bit-identical to what contiguous per-CTA tile ranges for every launch computed (the per-tile arithmetic is the same).
The last check compares the SHA-256 of the output bytes with tests/golden/conv_schedule.npz, captured from the
contiguous-range build on the same seeded inputs (`python tests/test_conv_schedule_gpu.py OUT.npz`): the outputs
themselves would be tens of MB.
"""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

# conv2d: (n, h, w, cin, cout, k, stride, residual, relu_from); every case applies ReLU from channel relu_from on
CONV = {
    # ResNet50, 256x128, last_stride 1 (layer1 64x32, layer2 32x16, layers 3-4 16x8: one 16x8 tile per image)
    "r50.l1.0.conv1": (2, 64, 32, 64, 64, 1, 1, False, 0),
    "r50.l2.0.conv2": (2, 64, 32, 128, 128, 3, 2, False, 0),
    "r50.l2.conv2": (2, 32, 16, 128, 128, 3, 1, False, 0),
    "r50.l2.3.conv3": (2, 32, 16, 128, 512, 1, 1, True, 0),
    "r50.l3.0.conv1": (2, 32, 16, 512, 256, 1, 1, False, 0),
    "r50.l3.0.conv2": (2, 32, 16, 256, 256, 3, 2, False, 0),
    "r50.l3.conv1": (2, 16, 8, 1024, 256, 1, 1, False, 0),
    "r50.l3.conv2": (2, 16, 8, 256, 256, 3, 1, False, 0),
    "r50.l3.conv3": (2, 16, 8, 256, 1024, 1, 1, True, 0),
    "r50.l4.0.conv1": (2, 16, 8, 1024, 512, 1, 1, False, 0),
    "r50.l4.conv2": (2, 16, 8, 512, 512, 3, 1, False, 0),
    "r50.l4.conv1": (2, 16, 8, 2048, 512, 1, 1, False, 0),
    "r50.l4.conv3": (2, 16, 8, 512, 2048, 1, 1, True, 0),
    # ResNet50-IBN-a, 320x320, last_stride 1 (80x80, 40x40, 20x20: partial tiles); conv1 of layers 1-3 leaves its
    # instance-normalised half without ReLU
    "ibn.l1.0.conv1": (1, 80, 80, 64, 64, 1, 1, False, 32),
    "ibn.l2.0.conv2": (1, 80, 80, 128, 128, 3, 2, False, 0),
    "ibn.l2.conv2": (1, 40, 40, 128, 128, 3, 1, False, 0),
    "ibn.l2.3.conv3": (1, 40, 40, 128, 512, 1, 1, True, 0),
    "ibn.l3.0.conv1": (1, 40, 40, 512, 256, 1, 1, False, 128),
    "ibn.l3.0.conv2": (1, 40, 40, 256, 256, 3, 2, False, 0),
    "ibn.l3.conv1": (1, 20, 20, 1024, 256, 1, 1, False, 128),
    "ibn.l3.conv2": (1, 20, 20, 256, 256, 3, 1, False, 0),
    "ibn.l3.conv3": (1, 20, 20, 256, 1024, 1, 1, True, 0),
    "ibn.l4.0.conv1": (1, 20, 20, 1024, 512, 1, 1, False, 0),
    "ibn.l4.conv2": (1, 20, 20, 512, 512, 3, 1, False, 0),
    "ibn.l4.conv1": (1, 20, 20, 2048, 512, 1, 1, False, 0),
    "ibn.l4.conv3": (1, 20, 20, 512, 2048, 1, 1, True, 0),
    # schedule edges: one tile; more tiles than the 132-CTA grid, not a multiple of it
    "one_tile": (1, 16, 8, 1024, 256, 1, 1, False, 0),
    "tiles133_bn256": (133, 16, 8, 1024, 256, 1, 1, False, 0),
    "tiles134_nt2": (67, 16, 8, 2048, 512, 1, 1, False, 0),
    "tiles280_nt8_res": (35, 16, 8, 512, 2048, 1, 1, True, 0),
    "tiles160_bn128_3x3": (40, 32, 16, 128, 128, 3, 1, False, 0),
    "tiles144_bn64": (9, 64, 32, 64, 64, 1, 1, False, 0),
}
# K-concatenated conv3 + downsample (ctl_conv1x1_dual_nhwc_f16): (n, ho, wo, cin1, cin2, cout, stride2)
DUAL = {
    "r50.l3.0.dual": (2, 16, 8, 256, 512, 1024, 2),
    "r50.l4.0.dual": (2, 16, 8, 512, 1024, 2048, 1),
    "ibn.l3.0.dual": (1, 20, 20, 256, 512, 1024, 2),
    "ibn.l4.0.dual": (1, 20, 20, 512, 1024, 2048, 1),
    "tiles136_dual_nt8": (17, 16, 8, 512, 1024, 2048, 1),
}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv_schedule.npz")


def _seed(name):
    return int.from_bytes(hashlib.sha256(name.encode()).digest()[:4], "little")


def run_conv(name):
    """-> (device output as fp16 on the host, float64 reference) of CONV[name]."""
    from ctl_b200 import _native as N

    n, h, w, cin, cout, k, stride, residual, relu_from = CONV[name]
    g = torch.Generator().manual_seed(_seed(name))
    x = (torch.randn(n, h, w, cin, generator=g) * 0.5).half()
    wt = (torch.randn(cout, k, k, cin, generator=g) / (k * cin ** 0.5)).half()
    bias = torch.randn(cout, generator=g) * 0.1
    pad = k // 2
    ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    res = (torch.randn(n, ho, wo, cout, generator=g) * 0.5).half() if residual else None
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), wt.double().permute(0, 3, 1, 2), bias.double(), stride, pad)
    ref = ref.permute(0, 2, 3, 1).contiguous()
    if res is not None:
        ref += res.double()
    ref[..., relu_from:] = ref[..., relu_from:].clamp(min=0)
    xd, wd, bd = x.cuda(), wt.cuda(), bias.cuda()
    rd = res.cuda() if res is not None else None
    out = torch.full((n, ho, wo, cout), float("nan"), dtype=torch.float16, device="cuda")
    N.check(N.lib().ctl_conv2d_nhwc_f16(xd.data_ptr(), n, h, w, cin, wd.data_ptr(), bd.data_ptr(), N.ptr(rd),
                                        out.data_ptr(), cout, k, stride, 1, relu_from, N.stream_ptr()))
    torch.cuda.synchronize()
    return out.cpu(), ref


def run_dual(name):
    """-> (device output as fp16 on the host, float64 reference) of DUAL[name]: relu(W3 x1 + Wd x2[::s, ::s] + b)."""
    from ctl_b200 import _native as N

    n, ho, wo, c1, c2, cout, s2 = DUAL[name]
    g = torch.Generator().manual_seed(_seed(name))
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
    return out.cpu(), ref


def digest(t):
    return np.frombuffer(hashlib.sha256(t.contiguous().view(torch.int16).numpy().tobytes()).digest(), np.uint8)


def _check(name, got, ref):
    assert not torch.isnan(got).any(), f"{name}: {int(torch.isnan(got).sum())} outputs never written"
    got = got.double()
    err = (got - ref).abs()
    bad = err > ref.abs() * 2.0 ** -10 + 1e-3
    assert not bad.any(), (f"{name}: {int(bad.sum())} / {bad.numel()} outputs off; max err {float(err.max()):.4e}; "
                           f"first bad index {bad.nonzero()[0].tolist()}")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN, allow_pickle=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CONV) + list(DUAL))
def test_conv_schedule(name, golden):
    got, ref = (run_conv if name in CONV else run_dual)(name)
    _check(name, got, ref)
    assert np.array_equal(digest(got), golden[name]), f"{name}: output bits differ from the contiguous-range build"


def test_golden_covers_every_case():
    assert sorted(np.load(GOLDEN, allow_pickle=False).files) == sorted(list(CONV) + list(DUAL))


if __name__ == "__main__":  # capture: python tests/test_conv_schedule_gpu.py OUT.npz
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import ctl_b200  # noqa: F401

    caps = {}
    for name in list(CONV) + list(DUAL):
        got, ref = (run_conv if name in CONV else run_dual)(name)
        _check(name, got, ref)
        caps[name] = digest(got)
    np.savez(sys.argv[1], **caps)
    print(f"captured {len(caps)} digests to {sys.argv[1]}")
