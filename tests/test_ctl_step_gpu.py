"""GPU: ctl_loss_step called directly through the C ABI against the float64 reference with the explicit tie rule
(oracle/ctl_step_oracle.py), at the batch shapes, mock-row patterns, feature columns and loss weights the goldens of
tests/test_losses_gpu.py do not reach.

Every call gets a workspace of 0xFF bytes and outputs prefilled with NaN, so an element no kernel writes fails.  Each
output isolates a group of kernels: parts[2] the image-level mining and reduction, parts[4..7] the rounds, d_centers
center_grad_kernel, d_bn_weight bn_backward_kernel, d_fc_weight the dZ^T y GEMM, the running statistics
bn_forward_kernel and d_feats combine_grad_kernel (every term).

Tolerances, from an fp32 error model.  The batches (oracle.ctl_step_oracle.step_batch) are integer lattices at a
power-of-two scale, so every Gram entry, squared norm and squared distance the step computes is exact and its
distances are correctly rounded: mining is exact, and what remains are the fp32 sums over slots, rows and columns
(relative error ~ u sqrt(n), u = 2^-24, a few 1e-6 at n <= 2048) and the softmax / log-sum-exp.  RTOL_EXACT = 2e-5
covers those with room.  With the offset column (|x|^2 ~ 2e6) a squared distance carries up to ~2 of rounding, 1e-6
relative at the d^2 ~ 1e6 of those batches, and a hinge of ~10 sums two distances of ~1e3, so those batches get the
goldens' 1e-4 as the ceiling.  The same rtol holds for every output.  A gradient element is a signed sum of terms
(rowsum E - Cm E and the head's terms in d_feats, the GEMMs over C and B in d_fc_weight, the sums over rows in
d_bn_weight and d_centers) each at most about the tensor's largest entry, so its rounding is bounded relative to that
entry, not to its own size: gradients and running statistics also get an absolute floor of rtol times the tensor's
largest |entry|.  (Measured on one H100 80GB HBM3 at a 700 W power limit: at most 3e-6 of that largest entry, and
7e-7 relative on the eight outputs.)
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import ctl_oracle as O
from oracle import ctl_step_oracle as S

pytestmark = pytest.mark.gpu

RTOL_EXACT = 2e-5
RTOL_INEXACT = 1e-4
# Precondition: the chosen distance beats every candidate that is not bit-identical to it by this relative gap, and
# |hinge| / d_ap is at least this (unless the chosen positive and negative rows are identical).  Exact lattices:
# 8 roundings of a correctly rounded square root.  Offset column: 10x the 1e-6 distance error above.
GAP_EXACT = 2.0**-20
GAP_INEXACT = 1e-5

DEFAULT = dict(margin=0.5, center_weight=5e-4, xent_weight=1.0, triplet_weight=1.0, ctl_weight=1.0, label_smooth=0.1,
               bn_momentum=0.1)
DISTINCT = dict(margin=0.3, center_weight=5e-3, xent_weight=0.7, triplet_weight=1.3, ctl_weight=0.9, label_smooth=0.2,
                bn_momentum=0.3)

# name: (P, K, D, C, real counts, ties, columns, weights, seed)
CASES = {
    # the reference default (IMS_PER_BATCH 64, NUM_INSTANCE 4)
    "p16k4_d2048": (16, 4, 2048, 751, None, False, False, DEFAULT, 1),
    "p16k4_d2048_ties": (16, 4, 2048, 751, None, True, False, DISTINCT, 2),
    # NT = 144: partial Gram tiles in M and N; B = 72: a k-remainder in dZ^T y; C = 1041: a C remainder
    "p18k4_d512": (18, 4, 512, 1041, None, False, False, DISTINCT, 3),
    "p18k4_d512_ties_columns": (18, 4, 512, 1041, None, True, True, DEFAULT, 4),
    # one partial tile; D % 16 = 8: k-remainders in the Gram and -Cm E GEMMs
    "p5k3_d520": (5, 3, 520, 23, None, False, False, DISTINCT, 5),
    "p5k3_d520_ties_columns": (5, 3, 520, 23, None, True, True, DEFAULT, 6),
    # 2P = 192 > 128 candidates per round slot (a second pass of the mining stride loop); T = 1152 slots
    "p96k4_d512": (96, 4, 512, 751, None, False, False, DEFAULT, 7),
    "p96k4_d512_ties": (96, 4, 512, 751, None, True, False, DISTINCT, 8),
    # K at its bound
    "p2k64_d256": (2, 64, 256, 7, None, False, False, DISTINCT, 9),
    "p2k64_d256_ties_columns": (2, 64, 256, 7, None, True, True, DEFAULT, 10),
    # real counts (2, 2, 6): rounds 2..5 skipped, n_valid_rounds = 2
    "p3k6_d72_skipped_rounds": (3, 6, 72, 5, (2, 2, 6), False, False, DEFAULT, 11),
    "p3k6_d72_skipped_rounds_ties_columns": (3, 6, 72, 5, (2, 2, 6), True, True, DISTINCT, 12),
}


def _batch(name):
    P, K, D, Cn, counts, ties, columns, w, seed = CASES[name]
    return S.step_batch(P, K, D, Cn, seed, counts=counts, ties=ties, columns=columns), K, w, columns


def _cfg(b, K, w):
    from ctl_b200 import _native as N

    B, D = b["feats"].shape
    return N.LossConfig(B, D, B // K, K, b["centers"].shape[0], w["margin"], w["center_weight"], w["xent_weight"],
                        w["triplet_weight"], w["ctl_weight"], 1e-5, w["bn_momentum"], w["label_smooth"])


def _buffers(b, cfg):
    """Device inputs, NaN-prefilled outputs and a workspace of 0xFF bytes."""
    from ctl_b200 import _native as N

    nan = float("nan")
    d = dict(f=b["feats"].cuda(), lab=b["labels"].int().cuda(), real=b["is_real"].to(torch.uint8).cuda(),
             c=b["centers"].cuda(), bw=b["bn_weight"].cuda(), bb=b["bn_bias"].cuda(), rm=b["running_mean"].cuda(),
             rv=b["running_var"].cuda(), fw=b["fc_weight"].cuda(), out=torch.full((8,), nan, device="cuda"))
    d.update(df=torch.full_like(d["f"], nan), dc=torch.full_like(d["c"], nan), dbw=torch.full_like(d["bw"], nan),
             dfw=torch.full_like(d["fw"], nan))
    need = N.lib().ctl_loss_workspace_bytes(C.byref(cfg))
    assert need > 0
    d["ws"] = torch.full((need,), 0xFF, dtype=torch.uint8, device="cuda")
    return d


ORDER = ("f", "lab", "real", "c", "bw", "bb", "rm", "rv", "fw", "out", "df", "dc", "dbw", "dfw", "ws")
OUT_KEYS = ("out", "df", "dc", "dbw", "dfw", "rm", "rv")


def _step(cfg, d, ws_bytes=None):
    from ctl_b200 import _native as N

    ws_bytes = d["ws"].numel() if ws_bytes is None else ws_bytes
    return N.lib().ctl_loss_step(C.byref(cfg), *(d[k].data_ptr() for k in ORDER), ws_bytes, N.stream_ptr())


def _reference(b, K, w):
    return S.ctl_step_reference(b["feats"], b["labels"], b["is_real"], K, b["centers"], b["bn_weight"], b["bn_bias"],
                                b["fc_weight"], running_mean=b["running_mean"], running_var=b["running_var"],
                                bn_momentum=w["bn_momentum"], margin=w["margin"], center_weight=w["center_weight"],
                                xent_weight=w["xent_weight"], triplet_weight=w["triplet_weight"],
                                ctl_weight=w["ctl_weight"], label_smooth=w["label_smooth"])


def _assert_unambiguous(ref, columns):
    """The precondition: a failure below is a kernel fault, not an fp32 near-tie of the inputs.  On the exact lattices
    an exact tie of distinct rows is a tie in fp32 too, broken by the same lowest-index rule."""
    gap = GAP_INEXACT if columns else GAP_EXACT
    for name, info, margin in ref["problems"]:
        gp, gn, gh = S.ambiguity(info, margin, exact=not columns)
        assert min(gp, gn, gh) >= gap, (name, gp, gn, gh)


def _close(got, want, rtol, floor, what):
    want = np.asarray(want, dtype=np.float64)
    got = np.asarray(got, dtype=np.float64)
    atol = floor * float(np.abs(want).max()) if want.size else 0.0
    np.testing.assert_allclose(got, want, rtol=rtol, atol=atol, err_msg=what)


def _check(name, d, ref, b, rtol):
    out = d["out"].cpu().numpy()
    for i, k in enumerate(S.NAMES):
        _close(out[i], ref["out"][k], rtol, 0.0, f"{name}: parts[{i}] {k}")
    d_f, d_c, d_bw, d_fw = ref["grads"]
    _close(d["df"].cpu(), d_f, rtol, rtol, f"{name}: d_feats")
    dc = d["dc"].cpu()
    present = torch.zeros(dc.shape[0], dtype=torch.bool)
    present[b["labels"]] = True
    assert (dc[~present] == 0).all(), f"{name}: d_centers rows of absent labels"
    _close(dc[present], d_c[present], rtol, rtol, f"{name}: d_centers")
    _close(d["dbw"].cpu(), d_bw, rtol, rtol, f"{name}: d_bn_weight")
    _close(d["dfw"].cpu(), d_fw, rtol, rtol, f"{name}: d_fc_weight")
    rm, rv = ref["running"]
    _close(d["rm"].cpu(), rm, rtol, rtol, f"{name}: running_mean")
    _close(d["rv"].cpu(), rv, rtol, rtol, f"{name}: running_var")


@pytest.mark.parametrize("name", list(CASES))
def test_ctl_step_matches_float64_reference(name):
    """Every output of one ctl_loss_step call against the float64 reference.  With ties, each row's d_feats is the
    lowest-index reference's (the kernel's documented tie rule), and the sums over identical rows equal the
    torch-mined restatement's (oracle.ctl_oracle.ctl_step_losses)."""
    b, K, w, columns = _batch(name)
    ref = _reference(b, K, w)
    _assert_unambiguous(ref, columns)
    cfg = _cfg(b, K, w)
    d = _buffers(b, cfg)
    assert _step(cfg, d) == 0
    torch.cuda.synchronize()
    _check(name, d, ref, b, RTOL_INEXACT if columns else RTOL_EXACT)
    if "mock_rows" in b["meta"]:
        info = ref["problems"][0][1]
        a = b["meta"]["tie_anchor"]
        assert info["groups"][info["p"][a]] == info["groups"][info["n"][a]]
        leaves = [b[k].double().requires_grad_(True) for k in ("feats", "centers", "bn_weight", "fc_weight")]
        alt = O.ctl_step_losses(leaves[0], b["labels"], b["is_real"], K, leaves[1], leaves[2], b["bn_bias"].double(),
                                leaves[3], margin=w["margin"], center_loss_weight=w["center_weight"],
                                query_xent_weight=w["xent_weight"], query_contrastive_weight=w["triplet_weight"],
                                centroid_contrastive_weight=w["ctl_weight"], epsilon=w["label_smooth"])
        (g_alt,) = torch.autograd.grad(alt["total"], leaves[:1])
        groups = torch.from_numpy(info["groups"])

        def sums(g):
            return torch.zeros(int(groups.max()) + 1, g.shape[1], dtype=torch.float64).index_add_(0, groups, g.double())

        rtol = RTOL_INEXACT if columns else RTOL_EXACT
        _close(sums(d["df"].cpu()), sums(g_alt), rtol, rtol, f"{name}: d_feats sums over identical rows")


def test_ctl_step_margin_zero_tie_passes_the_gradient():
    """margin = 0 on a bitwise tie (one mock vector is both the farthest positive and the nearest negative of a real
    anchor): the hinge is exactly 0 and, as in torch's MarginRankingLoss, its gradient passes; every row's d_feats is
    the lowest-index reference's, whose tied rows carry a non-zero share of it."""
    b = S.step_batch(18, 4, 512, 1041, 13, ties=True)
    w = {**DISTINCT, "margin": 0.0}
    ref = _reference(b, 4, w)
    _assert_unambiguous(ref, False)
    info = ref["problems"][0][1]
    a = b["meta"]["tie_anchor"]
    assert info["dm"][a, info["p"][a]] == info["dm"][a, info["n"][a]]
    off = S.ctl_step_reference(b["feats"], b["labels"], b["is_real"], 4, b["centers"], b["bn_weight"], b["bn_bias"],
                               b["fc_weight"], **{k: v for k, v in w.items() if k != "margin"}, margin=-1e-9)
    share = (ref["grads"][0] - off["grads"][0])[info["p"][a]]
    cfg = _cfg(b, 4, w)
    d = _buffers(b, cfg)
    assert _step(cfg, d) == 0
    torch.cuda.synchronize()
    _check("margin0", d, ref, b, RTOL_EXACT)
    got = d["df"].cpu().double()[info["p"][a]]
    want = ref["grads"][0][info["p"][a]]
    assert float(share.abs().max()) > 100 * float((got - want).abs().max())


def test_ctl_step_graph_replay_and_repeat_are_bit_identical():
    """96 x 4 with identical mock rows and the special columns: two eager calls and the replay of a captured CUDA graph
    give identical bits in every output (fixed-order reductions, no atomics on floats, no host synchronisation)."""
    b = S.step_batch(96, 4, 512, 751, 14, ties=True, columns=True)
    cfg = _cfg(b, 4, DISTINCT)
    d = _buffers(b, cfg)
    rm0, rv0 = d["rm"].clone(), d["rv"].clone()
    runs = []
    for _ in range(2):
        d["rm"].copy_(rm0)
        d["rv"].copy_(rv0)
        assert _step(cfg, d) == 0
        torch.cuda.synchronize()
        runs.append({k: d[k].clone() for k in OUT_KEYS})
    for k in ("out", "df", "dc", "dbw", "dfw"):
        d[k].fill_(float("nan"))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        assert _step(cfg, d) == 0
    d["rm"].copy_(rm0)
    d["rv"].copy_(rv0)
    graph.replay()
    torch.cuda.synchronize()
    runs.append({k: d[k].clone() for k in OUT_KEYS})
    assert all(bool(torch.isfinite(runs[0][k]).all()) for k in OUT_KEYS)
    for other in runs[1:]:
        for k in OUT_KEYS:
            assert torch.equal(runs[0][k].view(torch.int32), other[k].view(torch.int32)), k


def test_ctl_step_short_workspace_writes_nothing():
    """A workspace one byte short is CTL_ERR_WORKSPACE before any device work: every output keeps its NaN sentinel and
    the running statistics are untouched."""
    from ctl_b200 import _native as N

    b, K, w, _ = _batch("p5k3_d520")
    cfg = _cfg(b, K, w)
    d = _buffers(b, cfg)
    rm0, rv0 = d["rm"].clone(), d["rv"].clone()
    assert _step(cfg, d, d["ws"].numel() - 1) == -2
    assert b"workspace too small" in N.lib().ctl_last_error()
    torch.cuda.synchronize()
    for k in ("out", "df", "dc", "dbw", "dfw"):
        assert torch.isnan(d[k]).all(), k
    assert torch.equal(d["rm"], rm0) and torch.equal(d["rv"], rv0)
