"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the fused CTL loss step (`ctl_loss_step`) with an explicit tie
rule, and the seeded batches its tests run on.

`oracle.ctl_oracle.ctl_step_losses` mines with torch's max / min, and which of several exactly equal distances those
pick is not part of any contract.  `ctl_loss_step` takes the LOWEST row index on an exact tie (its tree reductions
order equal values by index).  Exact ties are normal in training: every mock row is the trunk's output on the same
all-zero image (datasets/bases.py pads a short identity with `torch.zeros_like(img)`), so all mock rows of a batch
carry the same feature vector, and mock rows are candidates of the image-level mining.  `ctl_step_reference` therefore
picks every mined positive and negative itself (first occurrence of the max / min, ties between bit-identical rows made
exact) and evaluates the eight outputs by autograd through gathers at those fixed indices.

Only tests/ may import this module; the product never does.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import ctl_oracle as O

NAMES = ("total", "xent", "triplet", "center", "ctl", "dist_ap", "dist_an", "l2_centroid")


def _row_groups(X: torch.Tensor) -> np.ndarray:
    """Group id of every row: rows with bit-identical values share one."""
    _, inv = torch.unique(X.detach(), dim=0, return_inverse=True)
    return inv.numpy()


def pair_dist(X: torch.Tensor, groups: np.ndarray, dist_func: str = "euclidean") -> torch.Tensor:
    """[n, n] distances of the rows of X as losses/triplet_loss.py:27-65 defines them, differentiable.  A pair of
    bit-identical rows gets exactly the clamp value (1e-12 under the square root for euclidean) and a zero gradient,
    which the Gram formula reaches only up to rounding."""
    ident = torch.from_numpy(groups[:, None] == groups[None, :])
    if dist_func == "euclidean":
        sq = (X * X).sum(1)
        s = sq[:, None] + sq[None, :] - 2.0 * (X @ X.t())
        return torch.where(ident, torch.zeros_like(s), s).clamp(min=1e-12).sqrt()
    xn = X / X.norm(dim=1, keepdim=True).clamp(min=1e-12)
    s = 1.0 - xn @ xn.t()
    return torch.where(ident, torch.zeros_like(s), s).abs().clamp(min=1e-12)


def mine(d: torch.Tensor, groups: np.ndarray, labels: np.ndarray, cand: np.ndarray):
    """Batch-hard mining of every row: the farthest same-label candidate and the nearest other-label candidate, the
    LOWEST index on an exact tie.  The distance to a row is read from the column of the first row of its identity
    group, so the distances to bit-identical rows are equal bit for bit.  Returns (p, n, dm, pos, neg); -1 where a
    row has no candidate."""
    first = np.zeros(groups.max() + 1, dtype=np.int64)
    for i in range(len(groups) - 1, -1, -1):
        first[groups[i]] = i
    dm = d.detach().numpy()[:, first[groups]]
    same = labels[:, None] == labels[None, :]
    pos = same & cand[None, :]
    neg = ~same & cand[None, :]
    p = np.where(pos.any(1), np.argmax(np.where(pos, dm, -np.inf), axis=1), -1)
    n = np.where(neg.any(1), np.argmin(np.where(neg, dm, np.inf), axis=1), -1)
    return p, n, dm, pos, neg


def batch_hard(X, labels, anchors, cand, margin, dist_func):
    """TripletLoss (losses/triplet_loss.py:139-173) over the rows of X with the given anchor and candidate masks:
    MarginRankingLoss(margin) or, for margin None, SoftMarginLoss.  Returns (loss, dist_ap, dist_an, info); the
    hinge is torch's clamp_min, whose gradient passes at exactly 0."""
    groups = _row_groups(X)
    labels = np.asarray(labels)
    d = pair_dist(X, groups, dist_func)
    p, n, dm, pos, neg = mine(d, groups, labels, np.asarray(cand, dtype=bool))
    a = np.flatnonzero(np.asarray(anchors, dtype=bool))
    assert (p[a] >= 0).all() and (n[a] >= 0).all(), "an anchor without a positive or a negative candidate"
    ap, an = d[a, p[a]], d[a, n[a]]
    h = (ap - an + margin).clamp(min=0) if margin is not None else F.softplus(ap - an)
    info = dict(dm=dm, groups=groups, pos=pos, neg=neg, p=p, n=n, a=a)
    return h.mean(), ap, an, info


def ctl_step_reference(feats, labels, is_real, K, centers, bn_weight, bn_bias, fc_weight, *, running_mean=None,
                       running_var=None, margin=0.5, center_weight=5e-4, xent_weight=1.0, triplet_weight=1.0,
                       ctl_weight=1.0, bn_eps=1e-5, bn_momentum=0.1, label_smooth=0.1, dist_func="euclidean"):
    """train_ctl_model.py:54-152 in float64 on a pid-major batch of P blocks of K rows, in closed form (SURVEY A.1):
    round r's queries are the real rows cK + r, its centroids the means of the other real rows of each such class, and
    the round is skipped unless more than one class has a centroid.  Every class must keep at least two real rows.

    Returns dict(out={name: float} in NAMES order, grads=(d_feats, d_centers, d_bn_weight, d_fc_weight) of `total`,
    running=(mean, var) after nn.BatchNorm1d's update with `bn_momentum` (None without running statistics),
    problems=[(name, info, margin)] for `ambiguity`)."""
    f = feats.detach().double().requires_grad_(True)
    c = centers.detach().double().requires_grad_(True)
    bw = bn_weight.detach().double().requires_grad_(True)
    fw = fc_weight.detach().double().requires_grad_(True)
    real = torch.as_tensor(is_real).bool()
    labels = torch.as_tensor(labels).long()
    B, D = f.shape
    P = B // K
    assert P * K == B
    lab_np, real_np = labels.numpy(), real.numpy()
    R = real.view(P, K)
    assert (R.sum(1) >= 2).all(), "batch contract: every class keeps at least two real rows"
    problems = []
    # :62-67 image level: anchors are the real rows, every row (mock rows too) is a candidate
    l_q, _, _, info = batch_hard(f, lab_np, real_np, np.ones(B, dtype=bool), margin, dist_func)
    problems.append(("image", info))
    l_q = l_q * triplet_weight
    # :69-77 center loss, BatchNorm1d (batch statistics) -> bias-free fc -> label-smoothed CE, real rows only
    fr, yr = f[real], labels[real]
    l_cen = center_weight * O.center_loss(fr, yr, c)
    rm = None if running_mean is None else running_mean.detach().double().clone()
    rv = None if running_var is None else running_var.detach().double().clone()
    y = F.batch_norm(fr, rm, rv, bw, bn_bias.detach().double(), True, bn_momentum, bn_eps)
    l_x = O.cross_entropy_label_smooth(y @ fw.t(), yr, fw.shape[0], label_smooth) * xent_weight
    # :79-145 the K centroid rounds
    F3 = f.view(P, K, D)
    lab_c = labels.view(P, K)[:, 0]
    others = ~torch.eye(K, dtype=torch.bool)
    losses, aps, ans, l2s = [], [], [], []
    for r in range(K):
        M = R[:, r][:, None] & R & others[r][None, :]  # [class, slot]: the members averaged into round r's centroids
        n_c = M.sum(1)
        if int((n_c > 0).sum()) <= 1:  # train_ctl_model.py:113
            continue
        cls = R[:, r]
        cent = (M[cls].double()[:, :, None] * F3[cls]).sum(1) / n_c[cls].double()[:, None]
        emb = torch.cat((F3[cls, r], cent))
        lab = torch.cat((lab_c[cls], lab_c[cls])).numpy()
        ones = np.ones(len(lab), dtype=bool)
        l_r, ap, an, info = batch_hard(emb, lab, ones, ones, margin, dist_func)
        problems.append((f"round{r}", info))
        losses.append(l_r)
        aps.append(ap.detach().mean())
        ans.append(an.detach().mean())
        l2s.append(cent.detach().norm(dim=1).mean())
    l_ctl = torch.stack(losses).mean() * ctl_weight
    total = l_ctl + l_cen + l_x + l_q  # :150-152
    grads = torch.autograd.grad(total, (f, c, bw, fw))
    vals = (total, l_x, l_q, l_cen, l_ctl, torch.stack(aps).mean(), torch.stack(ans).mean(), torch.stack(l2s).mean())
    return dict(out={k: float(v.detach()) for k, v in zip(NAMES, vals)}, grads=tuple(g.detach() for g in grads),
                running=None if rm is None else (rm, rv), problems=[(k, i, margin) for k, i in problems])


def ambiguity(info, margin, exact=False):
    """How far a mining problem is from an fp32 near-tie, over its anchors: the smallest relative gap between the
    chosen positive (negative) distance and the best candidate that is NOT bit-identical to the chosen row, and the
    smallest |hinge| relative to d_ap (hinge only; skipped where the chosen positive and negative rows are
    bit-identical, which makes the hinge exactly the margin).  `exact`: the inputs are such that the fp32 arithmetic
    under test reproduces every float64 distance tie, so candidates at exactly the chosen distance are ties, not
    near-ties.  Returns (gap_p, gap_n, gap_h); inf where nothing competes."""
    dm, g, pos, neg, p, n, a = (info[k] for k in ("dm", "groups", "pos", "neg", "p", "n", "a"))
    gp = gn = gh = math.inf
    for i in a:
        dp, dn = dm[i, p[i]], dm[i, n[i]]
        rp = pos[i] & (g != g[p[i]])
        rn = neg[i] & (g != g[n[i]])
        if exact:
            rp &= dm[i] != dp
            rn &= dm[i] != dn
        if rp.any():
            gp = min(gp, (dp - dm[i, rp].max()) / dp)
        if rn.any():
            gn = min(gn, (dm[i, rn].min() - dn) / dn)
        if margin is not None and g[p[i]] != g[n[i]]:
            gh = min(gh, abs(dp - dn + margin) / dp)
    return gp, gn, gh


# --------------------------------------------------------------------------------------
# seeded batches
# --------------------------------------------------------------------------------------


def _pow2(x):
    return 2.0 ** round(math.log2(x))


def step_batch(P, K, D, C, seed, *, counts=None, ties=False, columns=False):
    """Inputs of one CTL step on a pid-major batch of P labels x K rows (labels distinct, drawn from [0, C)).
    `counts[c]` real rows per class, mock rows trailing them; by default every row is real.

    Rows are `scale` times integer vectors rho_c + n_c z, with rho_c ~ round(omega tau N(0, I)) per class,
    z ~ round(tau / n_c N(0, I)) and n_c = counts[c] - 1, the number of rows averaged into the class's centroids.  So
    every centroid is an integer vector too, and with |row|^2 < 2^23 integer units (asserted) every Gram entry, squared
    norm and squared distance ctl_loss_step computes is EXACT in fp32: its distances are the correctly rounded square
    roots of the float64 ones, and only a tie or a relative gap below the last rounding can mine differently.
    `scale` is a power of two putting pairwise distances near 1, next to the margins.

    `ties`: classes 0 and 1 keep exactly two real rows; all their mock rows hold ONE vector m, placed between the
    farthest positive and the nearest negative of a real row `a` of class 0, so that m is both for `a` (d_ap == d_an
    bit for bit); the mock rows of a class also tie among themselves as positives.  With P >= 3 the last class holds K
    copies of one vector v next to a real row of class 1: every positive pair of that class (image level, and rounds,
    whose centroids are v exactly) and its center (set to v) sit at distance 0 exactly, at the 1e-12 clamps.

    `columns`: unit scale, pairwise distances near 1e3 (margins are then negligible); two all-zero columns, one
    constant column and, last, one column 1000 + k / 128 with integer k (spread about 1e-2) summing to 0 over the
    real rows.  Every partial sum of that column is exact in fp32, so the batch mean is exactly 1000 and the column
    tests the two-pass variance, not the rounding of the mean.  It also makes the distances inexact: ctl_loss_step's
    squared distances are then within about 2 of the float64 ones (roundings at |x|^2 ~ 2e6).

    Returns dict(feats, labels, is_real, centers, bn_weight, bn_bias, fc_weight, running_mean, running_var, meta)."""
    g = torch.Generator().manual_seed(seed)
    B = P * K

    def randn(*shape):
        return torch.randn(*shape, generator=g, dtype=torch.float64)

    labels = torch.randperm(C, generator=g)[:P].repeat_interleave(K)
    if counts is None:
        counts = [2 if (ties and c < 2) else K for c in range(P)]
    is_real = torch.zeros(P, K, dtype=torch.bool)
    for c, m in enumerate(counts):
        is_real[c, :m] = True
    is_real = is_real.view(-1)
    tau, omega = (_pow2(math.sqrt(1e6 / (2 * D))), 0.45) if columns else (16.0, 0.9)
    scale = 1.0 if columns else _pow2(1.0 / (tau * math.sqrt(2 * D)))
    x = torch.empty(B, D, dtype=torch.float64)
    for c in range(P):
        n_c = max(counts[c] - 1, 1)
        x[c * K:(c + 1) * K] = torch.round(omega * tau * randn(D)) + n_c * torch.round(tau / n_c * randn(K, D))
    special = [0, D // 3, D // 2, D - 1] if columns else []
    if columns:
        x[:, special[:2]] = 0.0
        x[:, special[2]] = 3.0
    meta = dict(scale=scale, special=special)
    centers = torch.round(tau * randn(C, D))
    real_np, lab_np = is_real.numpy(), labels.numpy()
    if ties and P >= 3:
        dup = P - 1
        noise = torch.round(0.1 * tau * randn(D))
        noise[special] = 0.0
        v = x[K] + noise  # next to the first row of class 1
        x[dup * K:(dup + 1) * K] = v
        meta["dup_rows"] = list(range(dup * K, (dup + 1) * K))
    if ties:
        # m: at a distance from `a` half-way between a's farthest real positive and its nearest real negative
        d = torch.cdist(x, x).numpy()
        best = None
        for a in np.flatnonzero(real_np & (np.arange(B) // K == 0)):
            same = (lab_np == lab_np[a]) & real_np
            far, near = d[a, same].max(), d[a, ~same & real_np].min()
            if best is None or near - far > best[1] - best[0]:
                best = (far, near, a)
        far, near, a = best
        assert near > far, "no real row of class 0 has its positives closer than its negatives"
        direction = randn(D)
        direction[special] = 0.0
        x[~is_real] = torch.round(x[a] + direction / direction.norm() * (0.5 * (far + near)))
        meta.update(tie_anchor=int(a), mock_rows=np.flatnonzero(~real_np).tolist())
    if columns:
        k = torch.randint(-2, 3, (B,), generator=g, dtype=torch.float64)
        k[~is_real] = 0  # the mock rows stay identical
        k[meta.get("dup_rows", [])] = 0  # so do the duplicated rows
        j = next(i for i in range(B) if real_np[i] and i not in meta.get("dup_rows", []))
        k[j] -= k.sum()  # the column sums to exactly 1000 B' over the real rows
        x[:, special[3]] = 1000.0 + k / 128.0
    if "dup_rows" in meta:
        centers[labels[meta["dup_rows"][0]]] = x[meta["dup_rows"][0]]
    assert columns or float((x * x).sum(1).max()) < 2**23  # so |x|^2 + |y|^2 is exact too
    return dict(
        feats=(x * scale).float(), labels=labels, is_real=is_real, centers=(centers * scale).float(),
        bn_weight=(0.5 + torch.rand(D, generator=g)), bn_bias=0.1 * torch.randn(D, generator=g),
        fc_weight=torch.randn(C, D, generator=g) / math.sqrt(D),
        running_mean=0.1 * tau * scale * torch.randn(D, generator=g), running_var=0.5 + torch.rand(D, generator=g),
        meta=meta)
