"""GPU parity tests of the loss path (through the C ABI) against the golden vectors produced
by the UNMODIFIED reference's CTLModel.training_step, and against the oracle restatement.
Tolerance: north_star's 1e-4 relative on fp32 losses / gradients (written per assertion)."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import ctl_oracle as O
from oracle.make_golden import DIM, LOSS_CASES, NUM_CLASSES, checksum, head_state

pytestmark = pytest.mark.gpu
RTOL = 1e-4


def _close(a, b, rtol=RTOL, atol=0.0):
    np.testing.assert_allclose(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64), rtol=rtol, atol=atol)


@pytest.mark.parametrize("name", list(LOSS_CASES))
def test_ctl_step_matches_reference_training_step(name):
    from ctl_b200 import _native as N
    from ctl_b200.losses._fn import CTLStepFn

    g = load_golden(f"loss_{name}.npz")
    P, K, pad, seed, scale = LOSS_CASES[name]
    feats, labels, is_real = O.synth_batch(P, K, DIM, NUM_CLASSES, seed, pad, scale)
    _close(checksum(feats), g["in_checksum"], 1e-12)
    hs = head_state(seed)
    f = feats.cuda().requires_grad_(True)
    centers = hs["centers"].cuda().requires_grad_(True)
    bn_w = hs["bn_weight"].cuda().requires_grad_(True)
    fc_w = hs["fc_weight"].cuda().requires_grad_(True)
    run_mean, run_var = torch.zeros(DIM).cuda(), torch.ones(DIM).cuda()
    cfg = N.LossConfig(P * K, DIM, P, K, NUM_CLASSES, 0.5, 5e-4, 1.0, 1.0, 1.0, 1e-5, 0.1, 0.1)
    total, parts = CTLStepFn.apply(f, centers, bn_w, fc_w, hs["bn_bias"].cuda(), run_mean, run_var, labels.cuda(),
                                   is_real.cuda(), cfg)
    total.backward()
    parts = parts.cpu().numpy()
    for i, key in enumerate(("total", "xent", "triplet", "center", "ctl", "dist_ap", "dist_an", "l2_centroid")):
        _close(parts[i], float(g[key]), RTOL)
    gscale = np.abs(g["grad_feats"]).max()
    _close(f.grad.cpu().numpy(), g["grad_feats"], RTOL, 1e-4 * gscale)
    rows = torch.from_numpy(g["grad_centers_rows_idx"])
    gc = centers.grad.cpu()
    # the reference multiplies centers.grad by 1/CENTER_LOSS_WEIGHT afterwards (train_ctl_model.py:157-158)
    _close(gc[rows].numpy() / 5e-4, g["grad_centers_rows"], RTOL, 1e-5 * np.abs(g["grad_centers_rows"]).max())
    _close(float(gc.abs().sum()) / 5e-4, float(g["grad_centers_abs_sum"]), RTOL)
    _close(bn_w.grad.cpu().numpy(), g["grad_bn_weight"], 1e-3, 1e-4 * np.abs(g["grad_bn_weight"]).max())
    _close(fc_w.grad.cpu()[rows].numpy(), g["grad_fc_rows"], 1e-3, 1e-4 * np.abs(g["grad_fc_rows"]).max())
    cs = checksum(fc_w.grad.cpu())
    assert abs(cs[0] - g["grad_fc_checksum"][0]) < 1e-3  # a sum of ~1.5M signed terms: absolute tolerance
    _close(cs[1], g["grad_fc_checksum"][1], 1e-3)
    _close(run_mean.cpu().numpy(), g["bn_running_mean"], RTOL, 1e-6)
    _close(run_var.cpu().numpy(), g["bn_running_var"], RTOL, 1e-6)


def test_standalone_losses_match_oracle():
    from ctl_b200.losses.center_loss import CenterLoss
    from ctl_b200.losses.triplet_loss import (CrossEntropyLabelSmooth, TripletLoss, cosine_dist, euclidean_dist,
                                              hard_example_mining)

    feats, labels, is_real = O.synth_batch(12, 4, 512, 100, seed=9, pad_fraction=0.3)
    # The checker runs the oracle restatement in float64: small fp32 matmuls on the GPU machine's
    # host CPU were observed to be ~2e-4 off (reduced-precision oneDNN path), which would mask
    # real 1e-4 errors.  TripletLoss with an anchor mask, vs autograd through the oracle.
    fo = feats.double().requires_grad_(True)
    lo, apo, ano = O.triplet_loss(fo, labels, 0.5, mask=is_real)
    lo.backward()
    fg = feats.cuda().requires_grad_(True)
    lg, apg, ang = TripletLoss(0.5)(fg, labels.cuda(), mask=is_real.cuda())
    lg.backward()
    _close(lg.item(), lo.item())
    _close(apg.cpu().numpy(), apo.detach().numpy())
    _close(ang.cpu().numpy(), ano.detach().numpy())
    _close(fg.grad.cpu().numpy(), fo.grad.numpy(), RTOL, 1e-4 * float(fo.grad.abs().max()))
    # ragged label multiset (the reference's view() cannot do this; the masked form can)
    lab2 = torch.tensor([0, 0, 0, 1, 1, 2, 2, 2, 2, 3, 3, 4, 4, 4, 5, 5])
    f2 = torch.randn(16, 256, generator=torch.Generator().manual_seed(1))
    l2o, _, _ = O.triplet_loss(f2.double(), lab2, 0.3)
    l2g, _, _ = TripletLoss(0.3)(f2.cuda(), lab2.cuda())
    _close(l2g.item(), l2o.item())
    # distances
    d = euclidean_dist(feats.cuda(), feats[:7].cuda()).cpu()
    d_or = O.euclidean_dist(feats.double(), feats[:7].double())
    # self pairs: sqrt of the fp32 cancellation noise of |x|^2+|x|^2-2x.x (~1e-3 at |x|^2~520), the same
    # quirk as the reference's own d(a,a) (SURVEY A.1); everything else to 1e-5 below
    assert float((d - d_or).abs().max()) < 0.1
    off = ~torch.eye(48, 7, dtype=torch.bool)
    _close(d[off].numpy(), d_or[off].numpy(), 1e-5)
    _close(cosine_dist(feats.cuda(), feats[:7].cuda()).cpu().numpy(),
           O.cosine_dist(feats.double(), feats[:7].double()).numpy(), 0, 2e-6)
    dm = O.euclidean_dist(feats, feats)
    ap, an, pi, ni = hard_example_mining(dm.cuda(), labels.cuda(), return_inds=True)
    apo2, ano2 = O.hard_example_mining(dm, labels)
    assert torch.equal(ap.cpu(), apo2) and torch.equal(an.cpu(), ano2)
    # CenterLoss
    cl = CenterLoss(100, 512).cuda()
    xo = feats.double().requires_grad_(True)
    co = cl.centers.detach().cpu().double().requires_grad_(True)
    O.center_loss(xo, labels, co).backward()
    xg = feats.cuda().requires_grad_(True)
    loss_g = cl(xg, labels.cuda())
    loss_g.backward()
    _close(loss_g.item(), O.center_loss(feats.double(), labels, co.detach()).item())
    _close(xg.grad.cpu().numpy(), xo.grad.numpy(), RTOL, 1e-6)
    _close(cl.centers.grad.cpu().numpy(), co.grad.numpy(), RTOL, 1e-6)
    # CrossEntropyLabelSmooth
    z = torch.randn(48, 100, generator=torch.Generator().manual_seed(2)) * 3
    zo = z.double().requires_grad_(True)
    O.cross_entropy_label_smooth(zo, labels, 100).backward()
    zg = z.cuda().requires_grad_(True)
    lx = CrossEntropyLabelSmooth(100)(zg, labels.cuda())
    lx.backward()
    _close(lx.item(), O.cross_entropy_label_smooth(z.double(), labels, 100).item())
    _close(zg.grad.cpu().numpy(), zo.grad.numpy(), RTOL, 1e-7)


def test_centroids_match_reference_golden():
    from ctl_b200 import reduce as RD
    from ctl_b200 import retrieval as R

    g = load_golden("centroids.npz")
    nq, ng = int(g["num_q"]), int(g["num_g"])
    feats, pids, cams = O.synth_retrieval(nq, ng, int(g["num_ids"]), DIM, 3.0, 11, num_cams=4)
    for respect, tag in ((False, "nocam"), (True, "cam")):
        emb, lab, cam = RD.validation_create_centroids(feats.cuda(), pids, cams, nq, respect)
        _close(emb.cpu().numpy(), g[f"{tag}_emb"], 1e-5, 1e-7)
        assert np.array_equal(lab, g[f"{tag}_lab"])
        if respect:
            assert [len(c) for c in cam] == g[f"{tag}_cam_len"].tolist()
        else:
            assert np.array_equal(cam, g[f"{tag}_cam"])
        qp = R.build_planes(emb[:nq], normalize=True)
        gp = R.build_planes(emb[nq:], normalize=True)
        res = R.evaluate_streamed(qp, gp, lab[:nq], lab[nq:], cam[:nq], cam[nq:], 50, respect)
        assert np.array_equal(res.cmc, g[f"{tag}_cmc"])
        _close(res.mAP, float(g[f"{tag}_mAP"]), 1e-9)
        _close(res.single_performance[:, 2].astype(np.float64), g[f"{tag}_ap"], 1e-9)
    pid_index = {}
    for i, p in enumerate(pids[nq:].tolist()):
        pid_index.setdefault(p, []).append(i)
    cents, cp = RD.calculate_centroids(feats[nq:].numpy(), pid_index)
    _close(cents, g["inf_centroids"], 1e-5, 1e-7)
    assert np.array_equal(cp, g["inf_pids"])
    v = torch.randn(6, 5, 64).cuda()
    _close(RD._calculate_centroids(v, 1).cpu().numpy(), (v.sum(1) / 5).cpu().numpy(), 1e-6, 1e-7)


@pytest.mark.parametrize("margin,dist", [(None, "euclidean"), (0.3, "cosine"), (None, "cosine")])
def test_triplet_loss_soft_margin_and_cosine_variants(margin, dist):
    """TripletLoss(margin=None) (nn.SoftMarginLoss on dist_an - dist_ap) and dist_func='cosine'
    (losses/triplet_loss.py:44-65,127-137,157-158): value, mined distances and the gradient (through the row normalisation
    for cosine) against autograd through the float64 oracle restatement, and against the reference's own class (its loss
    and gradient on this batch: tests/golden/triplet_variants.npz, oracle/make_golden.py:gen_triplet_variants)."""
    from ctl_b200.losses.triplet_loss import TripletLoss

    feats, labels, is_real = O.synth_batch(10, 4, 384, 100, seed=4, pad_fraction=0.2)
    feats = feats * 0.3 + 0.05
    for mask in (None, is_real):
        fo = feats.double().requires_grad_(True)
        lo, apo, ano = O.triplet_loss(fo, labels, margin, mask=mask, dist_func=dist)
        lo.backward()
        fg = feats.cuda().requires_grad_(True)
        lg, apg, ang = TripletLoss(margin, dist)(fg, labels.cuda(), mask=None if mask is None else mask.cuda())
        lg.backward()
        _close(lg.item(), lo.item())
        _close(apg.cpu().numpy(), apo.detach().numpy(), RTOL, 1e-6)
        _close(ang.cpu().numpy(), ano.detach().numpy(), RTOL, 1e-6)
        _close(fg.grad.cpu().numpy(), fo.grad.numpy(), RTOL, 1e-4 * float(fo.grad.abs().max()))
    g = load_golden("triplet_variants.npz")
    _close(checksum(feats), g["in_checksum"], 1e-12)
    lr, gr = float(g[f"{margin}_{dist}_loss"]), g[f"{margin}_{dist}_grad"]
    fg = feats.cuda().requires_grad_(True)
    lg, apg, ang = TripletLoss(margin, dist)(fg, labels.cuda())
    lg.backward()
    _close(lg.item(), lr, 2e-4)
    _close(fg.grad.cpu().numpy(), gr, 2e-4, 2e-4 * float(np.abs(gr).max()))


# ---- the stand-alone drop-ins and the composed path, against float64 at the shapes of tests/test_ctl_step_gpu.py ----


def _lattice(n, d, n_cls, seed):
    """n rows in classes of n / n_cls consecutive rows: integer class centres plus integer noise, times the power of two
    that puts distances near 1 (every Gram entry exact in fp32)."""
    g = torch.Generator().manual_seed(seed)
    labels = torch.arange(n_cls).repeat_interleave(n // n_cls)
    x = torch.round(3 * torch.randn(n_cls, d, generator=g)).repeat_interleave(n // n_cls, 0)
    x = x + torch.round(8 * torch.randn(n, d, generator=g))
    return (x * 2.0 ** round(np.log2(1 / (8 * np.sqrt(2 * d))))).float(), labels


@pytest.mark.parametrize("soft", [False, True])
@pytest.mark.parametrize("cosine", [False, True])
@pytest.mark.parametrize("n,d", [(200, 72), (300, 520)])
def test_triplet_fn_multi_tile(n, d, cosine, soft):
    """TripletFn at n = 200 and 300 (a multi-tile Gram with a partial tile; more than 128 candidates per anchor, so the
    mining stride loop runs twice) and d = 72, 520 (k-remainders of 8): loss, mined distances and gradient against the
    float64 batch-hard reference, with half the anchors masked off; every anchor masked off gives 0 and a zero
    gradient, without NaN."""
    from ctl_b200.losses._fn import TripletFn
    from oracle import ctl_step_oracle as S

    x, labels = _lattice(n, d, n // 5, seed=n + d)
    margin = None if soft else 0.3
    mask = torch.arange(n) % 2 == 0
    xo = x.double().requires_grad_(True)
    lo, apo, ano, info = S.batch_hard(xo, labels.numpy(), mask.numpy(), np.ones(n, dtype=bool), margin,
                                      "cosine" if cosine else "euclidean")
    gp, gn, gh = S.ambiguity(info, margin, exact=not cosine)
    assert min(gp, gn, gh) >= (1e-5 if cosine else 2.0**-20), (gp, gn, gh)  # no fp32 near-tie in the inputs
    lo.backward()
    xg = x.cuda().requires_grad_(True)
    lg, apg, ang = TripletFn.apply(xg, labels.cuda(), mask.cuda(), margin, soft, cosine)
    lg.backward()
    _close(lg.item(), lo.item(), 2e-5)
    _close(apg.cpu().numpy()[mask.numpy()], apo.detach().numpy(), 1e-5)
    _close(ang.cpu().numpy()[mask.numpy()], ano.detach().numpy(), 1e-5)
    _close(xg.grad.cpu().numpy(), xo.grad.numpy(), RTOL, 2e-5 * float(xo.grad.abs().max()))
    xg.grad = None
    lz, _, _ = TripletFn.apply(xg, labels.cuda(), torch.zeros(n, dtype=torch.bool, device="cuda"), margin, soft, cosine)
    lz.backward()
    assert float(lz.detach()) == 0.0 and bool((xg.grad == 0).all())


@pytest.mark.parametrize("P,K,D,Cn,seed", [(18, 4, 512, 1041, 13), (5, 3, 520, 23, 6)])
def test_triplet_fn_margin_zero_tie_passes_the_gradient(P, K, D, Cn, seed):
    """TripletFn (mine_single_kernel, shared with ctl_losses_composed and the base-model step) with margin 0 and the
    anchors masked to the real rows, on a batch whose identical mock rows hold one vector that is both the farthest
    positive and the nearest negative of a real anchor: the hinge is exactly 0 and its gradient passes, as in torch's
    MarginRankingLoss.  Every row's gradient equals the float64 reference's with the lowest-index tie rule, and the
    tied rows' share of it is far above the comparison's tolerance."""
    from ctl_b200.losses._fn import TripletFn
    from oracle import ctl_step_oracle as S

    b = S.step_batch(P, K, D, Cn, seed, ties=True)
    x, labels, real = b["feats"], b["labels"], b["is_real"]
    cand = np.ones(len(labels), dtype=bool)
    xo = x.double().requires_grad_(True)
    lo, apo, ano, info = S.batch_hard(xo, labels.numpy(), real.numpy(), cand, 0.0, "euclidean")
    gp, gn, gh = S.ambiguity(info, 0.0, exact=True)
    assert min(gp, gn, gh) >= 2.0**-20, (gp, gn, gh)  # no fp32 near-tie in the inputs
    a = b["meta"]["tie_anchor"]
    p, n = info["p"][a], info["n"][a]
    assert info["groups"][p] == info["groups"][n] and info["dm"][a, p] == info["dm"][a, n]  # the bitwise tie
    lo.backward()
    xoff = x.double().requires_grad_(True)
    S.batch_hard(xoff, labels.numpy(), real.numpy(), cand, -1e-9, "euclidean")[0].backward()  # that hinge switched off
    share = float((xo.grad - xoff.grad)[p].abs().max())
    xg = x.cuda().requires_grad_(True)
    lg, apg, ang = TripletFn.apply(xg, labels.cuda(), real.cuda(), 0.0, False, False)
    lg.backward()
    m = real.numpy()
    _close(lg.item(), lo.item(), 2e-5)
    _close(apg.cpu().numpy()[m], apo.detach().numpy(), 1e-5)
    _close(ang.cpu().numpy()[m], ano.detach().numpy(), 1e-5)
    atol = 2e-5 * float(xo.grad.abs().max())
    assert share > 100 * atol
    _close(xg.grad.cpu().numpy(), xo.grad.numpy(), RTOL, atol)


@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_xent_smooth_fn_large_logits(eps):
    """XentSmoothFn at C = 1041 with logits of +-300 (exp overflows fp32 without the max subtraction) and with
    epsilon = 0 (plain cross-entropy): value and gradient against float64."""
    from ctl_b200.losses._fn import XentSmoothFn

    g = torch.Generator().manual_seed(5)
    b, c = 72, 1041
    z = 300.0 * (2 * torch.rand(b, c, generator=g) - 1)
    t = torch.randint(0, c, (b,), generator=g)
    z[torch.arange(0, b, 3), t[::3]] = 300.0  # some rows' target at the top logit
    zo = z.double().requires_grad_(True)
    lo = O.cross_entropy_label_smooth(zo, t, c, eps)
    lo.backward()
    zg = z.cuda().requires_grad_(True)
    lg = XentSmoothFn.apply(zg, t.cuda(), eps)
    lg.backward()
    _close(lg.item(), lo.item(), 1e-5)
    # the kernel rounds the log-sum-exp to fp32 near |lse| = 300, i.e. to ulp(300) / 2 = 2^-16 absolute, so log p = z -
    # lse carries that error, and p with it (relative); where p nearly cancels the target, dz = (p - t) / b keeps it
    # as an absolute error: within 2 of those per row
    _close(zg.grad.cpu().numpy(), zo.grad.numpy(), RTOL, 2 * 2.0**-16 / b)


def test_center_loss_fn_row_at_its_center():
    """CenterLossFn with one row exactly at its center (distance 0 in fp32 as well, below the 1e-12 clamp): that row's
    gradient is exactly 0 and it adds nothing to its center's gradient; the rest against float64."""
    from ctl_b200.losses._fn import CenterLossFn

    x, labels = _lattice(72, 520, 18, seed=3)
    centers = (torch.round(8 * torch.randn(40, 520, generator=torch.Generator().manual_seed(4))) * 2.0**-8).float()
    labels = labels + 20
    labels[5] = 3  # a label of its own
    centers[3] = x[5]
    xo, co = x.double().requires_grad_(True), centers.double().requires_grad_(True)
    lo = O.center_loss(xo, labels, co)
    lo.backward()
    xg, cg = x.cuda().requires_grad_(True), centers.cuda().requires_grad_(True)
    lg = CenterLossFn.apply(xg, cg, labels.cuda())
    lg.backward()
    assert bool((xg.grad[5] == 0).all()) and bool((cg.grad[3] == 0).all())
    _close(lg.item(), lo.item(), 1e-5)
    _close(xg.grad.cpu().numpy(), xo.grad.numpy(), 1e-5, 1e-6 * float(xo.grad.abs().max()))
    _close(cg.grad.cpu().numpy(), co.grad.numpy(), 1e-5, 1e-6 * float(co.grad.abs().max()))


class _Cfg(dict):
    __getattr__ = dict.__getitem__


@pytest.mark.parametrize("margin,dist", [(0.6, "cosine"), (None, "euclidean")])
def test_ctl_losses_composed_matches_float64_reference(margin, dist):
    """ctl_losses_composed (the cosine and SoftMargin CTL configurations) at 18 x 4 with D = 512, C = 1041 and
    non-unit weights: the eight outputs and the gradients w.r.t. features, centers, bn.weight and fc.weight against
    the float64 reference."""
    from ctl_b200.modelling import ctl_model as M
    from oracle import ctl_step_oracle as S

    P, K, D, Cn = 18, 4, 512, 1041
    b = S.step_batch(P, K, D, Cn, seed=21)
    w = dict(center_weight=5e-3, xent_weight=0.7, triplet_weight=1.3, ctl_weight=0.9)
    ref = S.ctl_step_reference(b["feats"], b["labels"], b["is_real"], K, b["centers"], b["bn_weight"], b["bn_bias"],
                               b["fc_weight"], margin=margin, dist_func=dist, **w)
    for name, info, m in ref["problems"]:
        gp, gn, gh = S.ambiguity(info, m, exact=dist == "euclidean")
        assert min(gp, gn, gh) >= 1e-5, (name, gp, gn, gh)
    cfg = _Cfg(
        MODEL=_Cfg(NAME="resnet18", LAST_STRIDE=1, PRETRAINED=False, PRETRAIN_PATH="", BACKBONE_EMB_SIZE=D,
                   USE_CENTROIDS=False, KEEP_CAMID_CENTROIDS=True, RESUME_TRAINING=False),
        SOLVER=_Cfg(MARGIN=margin, DISTANCE_FUNC=dist, CENTER_LOSS_WEIGHT=w["center_weight"],
                    QUERY_XENT_WEIGHT=w["xent_weight"], QUERY_CONTRASTIVE_WEIGHT=w["triplet_weight"],
                    CENTROID_CONTRASTIVE_WEIGHT=w["ctl_weight"]),
        DATALOADER=_Cfg(NUM_INSTANCE=K), TEST=_Cfg(FEAT_NORM=True, ONLY_TEST=False, VISUALIZE="no"),
        USE_MIXED_PRECISION=True)
    model = M.CTLModel(cfg, num_classes=Cn, num_query=4).cuda().train()
    with torch.no_grad():
        model.center_loss.centers.copy_(b["centers"])
        model.bn.weight.copy_(b["bn_weight"])
        model.bn.bias.copy_(b["bn_bias"])
        model.fc_query.weight.copy_(b["fc_weight"])
    f = b["feats"].cuda().requires_grad_(True)
    total, parts = M.ctl_losses_composed(model, f, b["labels"].cuda(), b["is_real"].cuda())
    total.backward()
    _close(parts.cpu().numpy(), [ref["out"][k] for k in S.NAMES], 2e-5, 1e-7)
    got = (f.grad, model.center_loss.centers.grad, model.bn.weight.grad, model.fc_query.weight.grad)
    for gg, want in zip(got, ref["grads"]):
        _close(gg.cpu().numpy(), want.numpy(), RTOL, 2e-5 * float(want.abs().max()))
