"""GPU: the reference-named module surface (Baseline, CTLModel hooks) on the H100 engine."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import ctl_oracle as O
from oracle.make_golden import DIM, LOSS_CASES, NUM_CLASSES, head_state

pytestmark = pytest.mark.gpu


class _Cfg(dict):
    __getattr__ = dict.__getitem__


def _cfg(**over):
    c = _Cfg(
        MODEL=_Cfg(NAME="resnet50", LAST_STRIDE=1, PRETRAINED=False, PRETRAIN_PATH="", BACKBONE_EMB_SIZE=2048,
                   USE_CENTROIDS=False, KEEP_CAMID_CENTROIDS=True, RESUME_TRAINING=False),
        SOLVER=_Cfg(MARGIN=0.5, DISTANCE_FUNC="euclidean", CENTER_LOSS_WEIGHT=5e-4, QUERY_XENT_WEIGHT=1.0,
                    QUERY_CONTRASTIVE_WEIGHT=1.0, CENTROID_CONTRASTIVE_WEIGHT=1.0),
        DATALOADER=_Cfg(NUM_INSTANCE=4), TEST=_Cfg(FEAT_NORM=True, ONLY_TEST=False, VISUALIZE="no"),
        USE_MIXED_PRECISION=True)
    for k, v in over.items():
        a, b = k.split("__")
        c[a][b] = v
    return c


def test_ctl_model_hooks():
    from ctl_b200.modelling.ctl_model import CTLModel

    torch.manual_seed(0)
    model = CTLModel(_cfg(), num_classes=NUM_CLASSES, num_query=24).cuda()
    # state_dict layout of the reference checkpoint (SURVEY section 5)
    keys = list(model.state_dict().keys())
    assert "backbone.base.conv1.weight" in keys and "center_loss.centers" in keys and "fc_query.weight" in keys
    assert "bn.running_var" in keys and len([k for k in keys if k.startswith("backbone.base.")]) == 318
    # validation_step == oracle embed_forward on the same weights
    sd = O.make_trunk_state(seed=3)
    model.backbone.base.load_state_dict(sd)
    model.backbone.invalidate()
    with torch.no_grad():
        model.bn.running_mean.normal_(0, 0.1)
        model.bn.running_var.uniform_(0.5, 1.5)
        model.bn.weight.uniform_(0.5, 1.5)
    x = torch.randn(4, 3, 256, 128, generator=torch.Generator().manual_seed(2))
    out = model.validation_step((x.cuda(), torch.arange(4), torch.zeros(4, dtype=torch.long), torch.arange(4)), 0)
    bn_sd = {k: v.detach().cpu() for k, v in model.bn.state_dict().items()}
    with torch.no_grad():
        ref = O.embed_forward(x, sd, bn_sd)
    scale = float(ref.abs().max())
    assert float((out["emb"].cpu() - ref).abs().max()) <= 1e-2 * scale  # fp16 trunk vs fp32 oracle
    model.train()
    assert model.backbone(x.cuda())[1].requires_grad  # train mode: differentiable H100 training engine
    # training_step tail from prescribed features == the reference's training_step golden (train mode, like the reference)
    name = "p8k4_pad"
    g = load_golden(f"loss_{name}.npz")
    P, K, pad, seed, scale_f = LOSS_CASES[name]
    feats, labels, is_real = O.synth_batch(P, K, DIM, NUM_CLASSES, seed, pad, scale_f)
    hs = head_state(seed)
    with torch.no_grad():
        model.center_loss.centers.copy_(hs["centers"])
        model.bn.weight.copy_(hs["bn_weight"])
        model.bn.bias.copy_(hs["bn_bias"])
        model.fc_query.weight.copy_(hs["fc_weight"])
    f = feats.cuda().requires_grad_(True)
    res = model.training_step_from_features(f, labels.cuda(), is_real.cuda())
    res["loss"].backward()
    np.testing.assert_allclose(float(res["loss"]), float(g["total"]), rtol=1e-4)
    np.testing.assert_allclose(f.grad.cpu().numpy(), g["grad_feats"], rtol=1e-4, atol=1e-4 * np.abs(g["grad_feats"]).max())
    assert model.center_loss.centers.grad is not None and model.fc_query.weight.grad is not None


def test_validation_epoch_end_centroid_metric():
    """validation_epoch_end with MODEL.USE_CENTROIDS (both camid modes) vs the reference goldens."""
    from ctl_b200.modelling.ctl_model import CTLModel

    g = load_golden("centroids.npz")
    nq, ng = int(g["num_q"]), int(g["num_g"])
    feats, pids, cams = O.synth_retrieval(nq, ng, int(g["num_ids"]), DIM, 3.0, 11, num_cams=4)
    for keep, tag in ((False, "nocam"), (True, "cam")):
        model = CTLModel(_cfg(MODEL__USE_CENTROIDS=True, MODEL__KEEP_CAMID_CENTROIDS=keep), num_classes=10, num_query=nq)
        outs = [{"emb": feats[i:i + 200].cuda(), "labels": torch.from_numpy(pids[i:i + 200]),
                 "camid": torch.from_numpy(cams[i:i + 200])} for i in range(0, nq + ng, 200)]
        cmc, mAP, topk = model.validation_epoch_end(outs)
        assert np.array_equal(cmc, g[f"{tag}_cmc"])
        np.testing.assert_allclose(mAP, float(g[f"{tag}_mAP"]), rtol=1e-9)
        np.testing.assert_allclose(topk, g[f"{tag}_topk"], rtol=1e-9)


def _tiny_model(seed=0):
    from ctl_b200.modelling.ctl_model import CTLModel

    torch.manual_seed(seed)
    cfg = _cfg()
    cfg["SOLVER"].update(dict(OPTIMIZER_NAME="Adam", BASE_LR=3.5e-4, WEIGHT_DECAY=5e-4, CENTER_LR=0.5,
                              LR_SCHEDULER_NAME="multistep_lr", LR_STEPS=(40, 70), GAMMA=0.1, USE_WARMUP_LR=True,
                              WARMUP_EPOCHS=10))
    model = CTLModel(cfg, num_classes=16, num_query=4).cuda().train()
    model.backbone.base.load_state_dict(O.make_trunk_state(seed=11))
    g = torch.Generator().manual_seed(2)
    x = torch.randn(16, 3, 64, 32, generator=g).cuda()
    labels = (torch.arange(4).repeat_interleave(4) + 1).cuda()
    batch = (x, labels, torch.zeros(16, dtype=torch.long).cuda(), torch.ones(16, dtype=torch.bool).cuda())
    return model, batch


def test_batch_contract_violations_raise():
    """ADVICE r1: the mining kernels take a row's class from its position; a batch that is not pid-major, repeats a pid in
    two blocks, or carries a label outside [0, C) must be an error, not a silently different loss or an out-of-bounds
    access of the centers."""
    from ctl_b200.losses.center_loss import CenterLoss

    model, (x, labels, cam, real) = _tiny_model()
    feats = torch.randn(16, 2048, device="cuda")
    for bad, what in ((labels.roll(1), "not constant"), (torch.tensor([1] * 8 + [2] * 4 + [1] * 4).cuda(), "two blocks"),
                      (labels + 100, "outside")):
        model.__dict__.pop("_ctl_batch_checked", None)
        with pytest.raises(ValueError, match=what):
            model.training_step_from_features(feats, bad, real)
    model.__dict__.pop("_ctl_batch_checked", None)
    out = model.training_step_from_features(feats, labels, real)
    assert torch.isfinite(out["loss"])
    cl = CenterLoss(num_classes=16, feat_dim=2048)
    assert torch.isfinite(cl(feats, labels))
    with pytest.raises(ValueError, match="outside"):
        cl(feats, labels + 16)


def test_training_step_with_attached_optimizers_is_the_reference_iteration():
    """training_step with optimizers attached == zero_grad, forward, losses, backward, warm-up LR, Adam step, center
    rescale + SGD step (train_ctl_model.py:38-179), bit-identical to driving the same sequence by hand."""
    a, batch = _tiny_model(seed=5)
    b, _ = _tiny_model(seed=5)
    (oa, oca), _ = a.configure_optimizers()
    (ob, ocb), _ = b.configure_optimizers()
    a.attach_optimizers(oa, oca)
    for _ in range(2):
        ra = a.training_step(batch, 0)
        for p_ in b.parameters():
            p_.grad = None
        rb = b.training_step(batch, 0)
        rb["loss"].backward()
        b.optimizer_step_manual(ob, ocb, epoch=0)
        assert set(ra["other"]) == {"step_dist_ap", "step_dist_an", "l2_mean_centroid"}
        assert float(ra["loss"]) == float(rb["loss"])
    for (ka, va), (kb, vb) in zip(a.state_dict().items(), b.state_dict().items()):
        assert ka == kb and torch.equal(va, vb), ka
    assert len(a.losses_dict["centroid_triplet"]) == 2 and int(a.bn.num_batches_tracked) == 2


def test_dynamic_loss_scaling_skips_an_overflowing_step():
    """GradScaler semantics (the reference trains under PL native AMP, utils/misc.py:111) without host synchronisation:
    inf / NaN gradients make the optimizer kernels skip themselves (parameters and Adam moments untouched), the scale is
    halved on the device, the skipped step is taken back out of Adam's step count one step later; clean steps proceed."""
    model, batch = _tiny_model(seed=7)
    (opt, opt_c), _ = model.configure_optimizers()
    out = model.training_step(batch, 0)
    out["loss"].backward()
    scaler = model.backbone.loss_scaler
    assert scaler is not None and scaler.scale == 65536.0
    w = model.backbone.base.layer3[1].conv2.weight
    w0, c0 = w.detach().clone(), model.center_loss.centers.detach().clone()
    w.grad[0, 0, 0, 0] = float("inf")
    model.optimizer_step_manual(opt, opt_c, epoch=0)
    torch.cuda.synchronize()
    assert torch.equal(w.detach(), w0) and torch.equal(model.center_loss.centers.detach(), c0)
    assert scaler.scale == 32768.0
    assert all(float(st["exp_avg"].abs().max()) == 0 and float(st["exp_avg_sq"].abs().max()) == 0 for st in opt.state.values())
    for p_ in model.parameters():
        p_.grad = None
    out = model.training_step(batch, 0)
    out["loss"].backward()
    model.optimizer_step_manual(opt, opt_c, epoch=0)
    torch.cuda.synchronize()
    assert scaler.skipped_steps == 1 and all(int(st["step"]) == 1 for st in opt.state.values())  # the skipped step does not count
    assert not torch.equal(w.detach(), w0) and scaler.scale == 32768.0
    assert all(torch.isfinite(p_).all() for p_ in model.parameters())
    # the bias correction of this first REAL step is that of step 1: same update as a fresh torch.optim.Adam step
    g = w.grad.detach()
    expect = w0 - opt.param_groups[0]["lr"] * (g + 5e-4 * w0) / ((g + 5e-4 * w0).abs() + 1e-8)
    assert float((w.detach() - expect).abs().max()) <= 1e-6 * float(w0.abs().max()) + 1e-9


def test_eval_engine_never_serves_stale_weights():
    """ADVICE r1: the packed eval operands are a cache of the parameters; load_state_dict, an in-place parameter edit and
    an optimizer step must all be visible to the next eval forward without a manual invalidate()."""
    from ctl_b200.modelling.baseline import Baseline

    model = Baseline(_cfg()).cuda().eval()
    model.base.load_state_dict(O.make_trunk_state(seed=2))
    x = torch.randn(2, 3, 64, 32, generator=torch.Generator().manual_seed(4)).cuda()
    with torch.no_grad():
        f0 = model(x)[1].clone()
        assert torch.equal(model(x)[1], f0)
        eng = model._engine
        assert model.engine() is eng  # unchanged parameters: the pack is reused
        model.base.load_state_dict(O.make_trunk_state(seed=3))
        f1 = model(x)[1].clone()
        assert not torch.equal(f0, f1)
        model.base.layer4[2].bn3.weight.mul_(1.5)
        f2 = model(x)[1].clone()
        assert not torch.equal(f1, f2)
        model.base.load_state_dict(O.make_trunk_state(seed=2))
        assert torch.equal(model(x)[1], f0)


@pytest.mark.parametrize("seed,n_ids,n_cams", [(0, 12, 3), (1, 40, 6), (2, 7, 2), (3, 25, 9)])
def test_device_grouping_matches_the_reference_host_loop(seed, n_ids, n_cams):
    """validation_create_centroids with the grouping done on the device (sort / segments / camera-set bit masks) against
    the oracle's restatement of the reference's per-identity host loop (bases.py:179-262, pinned to the reference by
    tests/golden/centroids.npz): random identities with few rows, query cameras that do not occur in the gallery,
    identities present on one side only, single-camera identities (empty "other camera" sets) -- both camid modes."""
    from ctl_b200 import reduce as RD

    rng = np.random.default_rng(seed)
    nq, ng, d = 60, 400, 64
    labels = np.concatenate((rng.integers(0, n_ids + 3, nq), rng.integers(2, n_ids + 2, ng))) * 7 + 11   # sparse pids
    camids = rng.integers(0, n_cams, nq + ng) * 3 + 1
    camids[:nq][rng.random(nq) < 0.2] = 100                       # a query camera no gallery row has
    emb = torch.randn(nq + ng, d, generator=torch.Generator().manual_seed(seed))
    for respect in (False, True):
        e_ref, l_ref, c_ref = O.validation_create_centroids(emb, labels, camids, nq, respect_camids=respect)
        e, l, c = RD.validation_create_centroids(emb.cuda(), labels, camids, nq, respect_camids=respect)
        assert np.array_equal(l, np.asarray(l_ref))
        if respect:
            assert [list(map(int, x)) for x in c] == [list(map(int, np.atleast_1d(x))) for x in c_ref]
        else:
            assert np.array_equal(np.asarray(c), np.asarray(c_ref))
        np.testing.assert_allclose(e.cpu().numpy(), np.asarray(e_ref), rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("name,over", [("p8k4_pad_cosine", {"SOLVER__DISTANCE_FUNC": "cosine"}),
                                       ("p8k4_pad_softmargin", {"SOLVER__MARGIN": None}),
                                       ("p8k4_pad", {"SOLVER__DISTANCE_FUNC": "euclidean"})])
def test_ctl_step_triplet_variants_match_reference_training_step(name, over):
    """SOLVER.DISTANCE_FUNC = 'cosine' and MARGIN = None (SoftMarginLoss) through CTLModel.training_step_from_features
    against goldens produced by the reference's own training_step with those settings (oracle/make_golden.py::LOSS_VARIANTS);
    the third case forces the composed path on the default configuration and checks it against the fused step's golden."""
    from ctl_b200.modelling import ctl_model as M

    g = load_golden(f"loss_{name}.npz")
    base = name.replace("_cosine", "").replace("_softmargin", "")
    P, K, pad, seed, scale_f = LOSS_CASES[base]
    feats, labels, is_real = O.synth_batch(P, K, DIM, NUM_CLASSES, seed, pad, scale_f)
    hs = head_state(seed)
    torch.manual_seed(0)
    cfg = _cfg(**over)
    cfg["DATALOADER"]["NUM_INSTANCE"] = K
    model = M.CTLModel(cfg, num_classes=NUM_CLASSES, num_query=24).cuda().train()
    with torch.no_grad():
        model.center_loss.centers.copy_(hs["centers"])
        model.bn.weight.copy_(hs["bn_weight"])
        model.bn.bias.copy_(hs["bn_bias"])
        model.fc_query.weight.copy_(hs["fc_weight"])
    f = feats.cuda().requires_grad_(True)
    if name == "p8k4_pad":
        total, parts = M.ctl_losses_composed(model, f, labels.cuda(), is_real.cuda())
    else:
        out = model.training_step_from_features(f, labels.cuda(), is_real.cuda())
        total, parts = out["loss"], out["parts"]
    total.backward()
    p = parts.tolist()
    np.testing.assert_allclose(float(total), float(g["total"]), rtol=1e-4)
    for got, key in zip(p[1:8], ("xent", "triplet", "center", "ctl", "dist_ap", "dist_an", "l2_centroid")):
        np.testing.assert_allclose(got, float(g[key]), rtol=2e-4, atol=1e-6)
    np.testing.assert_allclose(f.grad.cpu().numpy(), g["grad_feats"], rtol=1e-4, atol=2e-4 * np.abs(g["grad_feats"]).max())
    np.testing.assert_allclose(model.bn.weight.grad.cpu().numpy(), g["grad_bn_weight"], rtol=1e-3,
                               atol=2e-4 * np.abs(g["grad_bn_weight"]).max())
