"""CPU: the float64 CTL-step reference with an explicit tie rule (oracle/ctl_step_oracle.py) against the restatement
pinned to the reference's goldens (oracle/ctl_oracle.ctl_step_losses), the seeded batches the GPU tests run on, and
the host-side argument contract of ctl_loss_step."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import ctl_oracle as O
from oracle import ctl_step_oracle as S

WEIGHTS = dict(margin=0.3, center_weight=5e-3, xent_weight=0.7, triplet_weight=1.3, ctl_weight=0.9,
               label_smooth=0.2)


def _losses_kw(margin, dist, w):
    return dict(margin=margin, center_loss_weight=w["center_weight"], query_xent_weight=w["xent_weight"],
                query_contrastive_weight=w["triplet_weight"], centroid_contrastive_weight=w["ctl_weight"],
                epsilon=w["label_smooth"], dist_func=dist)


def _both(b, K, margin, dist, w=WEIGHTS):
    """(ctl_step_reference, (outputs, grads) of ctl_step_losses) on one batch, float64."""
    ref = S.ctl_step_reference(b["feats"], b["labels"], b["is_real"], K, b["centers"], b["bn_weight"], b["bn_bias"],
                               b["fc_weight"], dist_func=dist, **{**w, "margin": margin})
    leaves = [b[k].double().requires_grad_(True) for k in ("feats", "centers", "bn_weight", "fc_weight")]
    out = O.ctl_step_losses(leaves[0], b["labels"], b["is_real"], K, leaves[1], leaves[2], b["bn_bias"].double(),
                            leaves[3], **_losses_kw(margin, dist, w))
    grads = torch.autograd.grad(out["total"], leaves)
    return ref, ({k: float(v.detach()) for k, v in out.items()}, grads)


@pytest.mark.parametrize("margin", [0.3, None])
@pytest.mark.parametrize("dist", ["euclidean", "cosine"])
@pytest.mark.parametrize("shape", [(18, 4, 64, 41, None), (3, 6, 72, 5, (2, 2, 6)), (2, 64, 32, 7, (2, 64))])
def test_reference_matches_ctl_step_losses_without_ties(shape, dist, margin):
    """On batches without exact ties the two restatements are the same function: the eight outputs and the gradients
    w.r.t. feats, centers, bn.weight and fc.weight agree to float64 rounding.  (3, 6) has real counts (2, 2, 6), so
    rounds 2..5 are skipped; (2, 64) keeps two real rows in its first class, so 62 of its 64 rounds are."""
    P, K, D, Cn, counts = shape
    b = S.step_batch(P, K, D, Cn, seed=7, counts=counts)
    ref, (out, grads) = _both(b, K, margin, dist)
    n_rounds = sum(1 for k, _, _ in ref["problems"] if k.startswith("round"))
    assert n_rounds == {18: 4, 3: 2, 2: 2}[P]
    for k in S.NAMES:
        np.testing.assert_allclose(ref["out"][k], out[k], rtol=1e-12, atol=1e-15)
    for got, want in zip(ref["grads"], grads):
        np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-10, atol=1e-12 * float(want.abs().max()))


def _group_sums(grad, groups):
    out = torch.zeros(groups.max() + 1, grad.shape[1], dtype=grad.dtype)
    return out.index_add_(0, torch.from_numpy(groups), grad)


@pytest.mark.parametrize("margin", [0.5, 0.0])
def test_reference_matches_ctl_step_losses_on_tie_groups(margin):
    """With identical mock rows the two restatements may hand a tied gradient to different rows, but every value, and
    the gradient summed over each group of identical rows (what reaches the trunk's weights: the rows are one image),
    agree.  The batch has the tie the fused step must get right: one vector is both the farthest positive and the
    nearest negative of a real anchor, and a class of identical rows sits at the distance clamp."""
    P, K = 6, 4
    b = S.step_batch(P, K, 64, 41, seed=3, ties=True)
    ref, (out, grads) = _both(b, K, margin, "euclidean")
    info = ref["problems"][0][1]
    a = b["meta"]["tie_anchor"]
    assert info["groups"][info["p"][a]] == info["groups"][info["n"][a]]  # the tie is there
    assert info["p"][a] == b["meta"]["mock_rows"][0] and info["n"][a] == K + 2  # lowest index on both sides
    for k in S.NAMES:
        np.testing.assert_allclose(ref["out"][k], out[k], rtol=1e-12, atol=1e-15)
    groups = info["groups"]
    np.testing.assert_allclose(_group_sums(ref["grads"][0], groups).numpy(), _group_sums(grads[0], groups).numpy(),
                               rtol=1e-10, atol=1e-12 * float(grads[0].abs().max()))
    for got, want in zip(ref["grads"][1:], grads[1:]):
        np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-10, atol=1e-12 * float(want.abs().max()))


def test_hinge_at_exactly_zero_passes_the_gradient():
    """torch's MarginRankingLoss (what TripletLoss uses) passes the gradient at a hinge of exactly 0, and so does the
    reference's clamp: on a margin-0 tie, switching that one hinge off (margin -1e-9) removes exactly the anchor's
    pair of opposite gradients on its two tied rows and nothing else."""
    x1, x2 = torch.ones(1, requires_grad=True), torch.ones(1, requires_grad=True)
    torch.nn.MarginRankingLoss(margin=0.0)(x2, x1, torch.ones(1)).backward()
    assert float(x1.grad) == 1.0 and float(x2.grad) == -1.0
    b = S.step_batch(6, 4, 64, 41, seed=3, ties=True)
    run = [S.ctl_step_reference(b["feats"], b["labels"], b["is_real"], 4, b["centers"], b["bn_weight"], b["bn_bias"],
                                b["fc_weight"], margin=m) for m in (0.0, -1e-9)]
    info = run[0]["problems"][0][1]
    a = b["meta"]["tie_anchor"]
    p, n = info["p"][a], info["n"][a]
    diff = run[0]["grads"][0] - run[1]["grads"][0]
    assert float(diff[p].abs().max()) > 1e-3
    torch.testing.assert_close(diff[p], -diff[n], rtol=1e-9, atol=1e-15)
    rest = np.setdiff1d(np.arange(len(diff)), [p, n])
    assert float(diff[rest].abs().max()) < 1e-12


def test_step_batch_is_exact_and_has_its_ties():
    """The seeded batches' promises: integer lattice rows (every fp32 sum of products exact), the mock rows one vector,
    the duplicated class one vector equal to its center, and the offset column summing to exactly 1000 per real row."""
    b = S.step_batch(5, 3, 520, 23, seed=1, ties=True, columns=True)
    f, real = b["feats"].double(), b["is_real"]
    mock = b["meta"]["mock_rows"]
    assert len(mock) == 2 and (f[mock] == f[mock[0]]).all()
    dup = b["meta"]["dup_rows"]
    assert (f[dup] == f[dup[0]]).all() and (b["centers"][b["labels"][dup[0]]] == b["feats"][dup[0]]).all()
    sp = b["meta"]["special"]
    assert (f[:, sp[:2]] == 0).all() and (f[:, sp[2]] == f[0, sp[2]]).all()
    assert float(f[real, sp[3]].sum()) == 1000.0 * int(real.sum())
    assert float(f[real, sp[3]].std()) > 5e-3
    b = S.step_batch(96, 4, 512, 751, seed=1)
    x = b["feats"].double() / b["meta"]["scale"]
    assert (x == x.round()).all() and float((x * x).sum(1).max()) < 2**23


def _cfg(B, D, P, K, Cn):
    from ctl_b200 import _native as N

    return N.LossConfig(B, D, P, K, Cn, 0.5, 5e-4, 1.0, 1.0, 1.0, 1e-5, 0.1, 0.1)


def test_loss_step_argument_contract():
    """Rejected before any device work: K above the 64 rounds StepMeta holds, B != P K; the workspace size of a bad
    configuration is 0.  K = 64 passes the configuration check (ctl_loss_step then stops at the null pointers)."""
    from ctl_b200 import _native as N

    L = N.lib()
    assert L.ctl_loss_workspace_bytes(C.byref(_cfg(128, 256, 2, 64, 7))) > 0
    nulls = [None] * 15
    assert L.ctl_loss_step(C.byref(_cfg(128, 256, 2, 64, 7)), *nulls, 0, None) == -1
    assert b"null pointer" in L.ctl_last_error()
    for bad in (_cfg(130, 256, 2, 65, 7), _cfg(63, 256, 16, 4, 751), _cfg(64, 0, 16, 4, 751), _cfg(0, 256, 0, 4, 7)):
        assert L.ctl_loss_workspace_bytes(C.byref(bad)) == 0
        assert L.ctl_loss_step(C.byref(bad), *nulls, 0, None) == -1
        assert b"batch contract" in L.ctl_last_error() or b"bad dims" in L.ctl_last_error()
    assert L.ctl_loss_step(C.byref(_cfg(130, 256, 2, 65, 7)), *nulls, 0, None) == -1
    assert b"K <= 64" in L.ctl_last_error()
