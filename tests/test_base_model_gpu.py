"""GPU: the base model's fused loss step (ctl_base_loss_step through BaseStepFn) and BaseModel.training_step against
the golden vectors of the UNMODIFIED reference's train_base_model.CTLModel.training_step, the float64 oracle
(oracle/base_oracle.py) and the composed drop-in losses."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import ctl_oracle as O
from oracle.base_oracle import BASE_CASES, base_step_losses
from oracle.make_golden import DIM, NUM_CLASSES, checksum, head_state
from test_base_model_cpu import variant_kwargs

pytestmark = pytest.mark.gpu
RTOL = 1e-4
PART_NAMES = ("total", "xent", "triplet", "center", "dist_ap", "dist_an")
VARIANTS = [(0.5, "euclidean"), (None, "euclidean"), (0.5, "cosine"), (None, "cosine")]


def _close(a, b, rtol=RTOL, atol=0.0):
    np.testing.assert_allclose(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64), rtol=rtol, atol=atol)


def _cfg(B, D, Cn, margin=0.5, dist="euclidean", center_weight=5e-4, xent_weight=1.0, triplet_weight=1.0):
    from ctl_b200 import _native as N

    return N.BaseLossConfig(B, D, Cn, 0.0 if margin is None else float(margin), int(margin is None),
                            int(dist == "cosine"), center_weight, xent_weight, triplet_weight, 1e-5, 0.1, 0.1)


def _fused(feats, labels, is_real, centers, bn_w, bn_b, fc_w, cfg, run_mean=None, run_var=None):
    """BaseStepFn on CUDA copies (leaves with gradients); returns (parts[6] numpy, grads, running stats)."""
    from ctl_b200.losses._fn import BaseStepFn

    f, c, bw, fw = (t.detach().float().cuda().requires_grad_(True) for t in (feats, centers, bn_w, fc_w))
    rm = torch.zeros(f.shape[1], device="cuda") if run_mean is None else run_mean
    rv = torch.ones(f.shape[1], device="cuda") if run_var is None else run_var
    total, parts = BaseStepFn.apply(f, c, bw, fw, bn_b.float().cuda(), rm, rv, labels.cuda(), is_real.cuda(), cfg)
    total.backward()
    assert float(total.detach()) == float(parts[0])
    return parts.cpu().numpy(), (f.grad.cpu(), c.grad.cpu(), bw.grad.cpu(), fw.grad.cpu()), (rm.cpu(), rv.cpu())


@pytest.mark.parametrize("name", list(BASE_CASES))
def test_base_step_matches_reference_training_step(name):
    """The six outputs within 1e-4 relative; gradients and running statistics at the tolerances of
    tests/test_losses_gpu.py::test_ctl_step_matches_reference_training_step."""
    g = load_golden(f"base_loss_{name}.npz")
    (P, K, pad, seed, scale), over = BASE_CASES[name]
    feats, labels, is_real = O.synth_batch(P, K, DIM, NUM_CLASSES, seed, pad, scale)
    _close(checksum(feats), g["in_checksum"], 1e-12)
    hs = head_state(seed)
    kw = variant_kwargs(over)
    cfg = _cfg(P * K, DIM, NUM_CLASSES, kw.get("margin", 0.5), kw.get("dist_func", "euclidean"))
    parts, (gf, gc, gbw, gfw), (rm, rv) = _fused(feats, labels, is_real, hs["centers"], hs["bn_weight"], hs["bn_bias"],
                                                 hs["fc_weight"], cfg)
    for i, key in enumerate(PART_NAMES):
        _close(parts[i], float(g[key]), RTOL)
    # the feature gradient is stored as a row sample (mock rows included) plus checksums of the whole tensor
    gscale = float(g["grad_feats_abs_max"])
    _close(gf[torch.from_numpy(g["grad_feats_rows_idx"])].numpy(), g["grad_feats_rows"], RTOL, 1e-4 * gscale)
    fcs = checksum(gf)
    assert abs(fcs[0] - g["grad_feats_checksum"][0]) < 1e-4 * gscale * gf.numel() ** 0.5  # signed sum: absolute
    _close(fcs[1], g["grad_feats_checksum"][1], 1e-3)
    rows = torch.from_numpy(g["grad_centers_rows_idx"])
    # the reference multiplies centers.grad by 1/CENTER_LOSS_WEIGHT afterwards (train_base_model.py:80-81)
    _close(gc[rows].numpy() / 5e-4, g["grad_centers_rows"], RTOL, 1e-5 * np.abs(g["grad_centers_rows"]).max())
    _close(float(gc.abs().sum()) / 5e-4, float(g["grad_centers_abs_sum"]), RTOL)
    _close(gbw.numpy(), g["grad_bn_weight"], 1e-3, 1e-4 * np.abs(g["grad_bn_weight"]).max())
    _close(gfw[rows].numpy(), g["grad_fc_rows"], 1e-3, 1e-4 * np.abs(g["grad_fc_rows"]).max())
    cs = checksum(gfw)
    assert abs(cs[0] - g["grad_fc_checksum"][0]) < 1e-3  # a sum of ~1.5M signed terms: absolute tolerance
    _close(cs[1], g["grad_fc_checksum"][1], 1e-3)
    _close(rm.numpy(), g["bn_running_mean"], RTOL, 1e-6)
    _close(rv.numpy(), g["bn_running_var"], RTOL, 1e-6)


def _ragged_batch(D, Cn, seed, scale=0.5):
    """37 rows (not a multiple of 32) in shuffled order, 10 identities with 2..6 rows each, about a fifth of them mock
    rows: a label multiset no pid-major sampler would produce, which batch-hard mining is defined for all the same."""
    g = torch.Generator().manual_seed(seed)
    counts = torch.tensor([5, 3, 4, 2, 6, 3, 4, 3, 2, 5])
    ids = torch.randperm(Cn, generator=g)[: len(counts)]
    labels = ids.repeat_interleave(counts)
    perm = torch.randperm(len(labels), generator=g)
    labels = labels[perm]
    B = len(labels)
    offset = torch.randn(Cn, D, generator=g)
    feats = scale * (torch.randn(B, D, generator=g) + 0.3 * offset[labels]) + 0.05
    is_real = torch.rand(B, generator=g) > 0.2
    is_real[0] = True
    head = dict(centers=torch.randn(Cn, D, generator=g), bn_weight=0.5 + torch.rand(D, generator=g),
                bn_bias=0.1 * torch.randn(D, generator=g), fc_weight=0.05 * torch.randn(Cn, D, generator=g))
    return feats, labels, is_real, head


@pytest.mark.parametrize("margin,dist", VARIANTS)
def test_base_step_matches_float64_oracle(margin, dist):
    """Shapes the goldens do not cover: B = 37, D = 512 (ResNet18/34 features), C = 23, every TripletLoss variant,
    a non-zero BN bias and weights other than 1, against autograd through the float64 oracle."""
    D, Cn, wc, wx, wt = 512, 23, 5e-3, 0.7, 1.3
    feats, labels, is_real, hd = _ragged_batch(D, Cn, seed=3)
    B = len(labels)
    fo, co, bwo, fwo = (t.double().requires_grad_(True) for t in (feats, hd["centers"], hd["bn_weight"], hd["fc_weight"]))
    rmo, rvo = torch.zeros(D, dtype=torch.float64), torch.ones(D, dtype=torch.float64)
    ref = base_step_losses(fo, labels, is_real, co, bwo, hd["bn_bias"].double(), fwo, margin=margin, dist_func=dist,
                           center_loss_weight=wc, query_xent_weight=wx, query_contrastive_weight=wt, running_mean=rmo,
                           running_var=rvo)
    ref["total"].backward()
    cfg = _cfg(B, D, Cn, margin, dist, wc, wx, wt)
    parts, (gf, gc, gbw, gfw), (rm, rv) = _fused(feats, labels, is_real, hd["centers"], hd["bn_weight"], hd["bn_bias"],
                                                 hd["fc_weight"], cfg)
    for i, key in enumerate(PART_NAMES):
        _close(parts[i], float(ref[key]), RTOL, 1e-7)
    for got, want in ((gf, fo.grad), (gc, co.grad), (gbw, bwo.grad), (gfw, fwo.grad)):
        _close(got.numpy(), want.numpy(), RTOL, 1e-4 * float(want.abs().max()))
    _close(rm.numpy(), rmo.numpy(), RTOL, 1e-6)
    _close(rv.numpy(), rvo.numpy(), RTOL, 1e-6)


@pytest.mark.parametrize("margin,dist", VARIANTS)
def test_base_step_matches_composed_drop_ins(margin, dist):
    """train_base_model.py:60-75 assembled from the stand-alone drop-ins (TripletLoss, CenterLoss, CrossEntropyLabelSmooth)
    and torch's BatchNorm1d + bias-free Linear on the p16k16_pad inputs: the fused step agrees within fp32
    reduction-order noise (values, every gradient, running statistics)."""
    from ctl_b200.losses.center_loss import CenterLoss
    from ctl_b200.losses.triplet_loss import CrossEntropyLabelSmooth, TripletLoss

    (P, K, pad, seed, scale), _ = BASE_CASES["p16k16_pad"]
    feats, labels, is_real = O.synth_batch(P, K, DIM, NUM_CLASSES, seed, pad, scale)
    hs = head_state(seed)
    lab, real = labels.cuda(), is_real.cuda()
    f = feats.cuda().requires_grad_(True)
    cl = CenterLoss(NUM_CLASSES, DIM).cuda()
    bn = torch.nn.BatchNorm1d(DIM).cuda().train()
    bn.bias.requires_grad_(False)
    fc = torch.nn.Linear(DIM, NUM_CLASSES, bias=False).cuda()
    with torch.no_grad():
        cl.centers.copy_(hs["centers"])
        bn.weight.copy_(hs["bn_weight"])
        fc.weight.copy_(hs["fc_weight"])
    lq, ap, an = TripletLoss(margin, dist)(f, lab, mask=real)
    center = 5e-4 * cl(f, lab)
    xent = CrossEntropyLabelSmooth(NUM_CLASSES)(fc(bn(f)), lab)
    total = center + xent + lq
    total.backward()
    want = [float(v) for v in (total, xent, lq, center, ap.mean(), an.mean())]
    parts, (gf, gc, gbw, gfw), (rm, rv) = _fused(feats, labels, is_real, hs["centers"], hs["bn_weight"], hs["bn_bias"],
                                                 hs["fc_weight"], _cfg(P * K, DIM, NUM_CLASSES, margin, dist))
    _close(parts, want, 2e-5)
    for got, ref in ((gf, f.grad), (gc, cl.centers.grad), (gbw, bn.weight.grad), (gfw, fc.weight.grad)):
        ref = ref.cpu()
        _close(got.numpy(), ref.numpy(), RTOL, 2e-5 * float(ref.abs().max()))
    _close(rm.numpy(), bn.running_mean.cpu().numpy(), 1e-5, 1e-7)
    _close(rv.numpy(), bn.running_var.cpu().numpy(), 1e-5, 1e-7)


def _raw_step(cfg, bufs, ws_bytes=None):
    from ctl_b200 import _native as N

    b = bufs
    ws_bytes = b["ws"].numel() if ws_bytes is None else ws_bytes
    return N.lib().ctl_base_loss_step(C.byref(cfg), *(b[k].data_ptr() for k in (
        "f", "lab", "real", "c", "bw", "bb", "rm", "rv", "fw", "out", "df", "dc", "dbw", "dfw", "ws")), ws_bytes,
        N.stream_ptr())


def _buffers(name, cfg):
    from ctl_b200 import _native as N

    (P, K, pad, seed, scale), _ = BASE_CASES[name]
    feats, labels, is_real = O.synth_batch(P, K, DIM, NUM_CLASSES, seed, pad, scale)
    hs = head_state(seed)
    b = dict(f=feats.cuda(), lab=labels.int().cuda(), real=is_real.to(torch.uint8).cuda(), c=hs["centers"].cuda(),
             bw=hs["bn_weight"].cuda(), bb=hs["bn_bias"].cuda(), rm=torch.zeros(DIM).cuda(), rv=torch.ones(DIM).cuda(),
             fw=hs["fc_weight"].cuda(), out=torch.zeros(6).cuda())
    b.update(df=torch.empty_like(b["f"]), dc=torch.empty_like(b["c"]), dbw=torch.empty_like(b["bw"]),
             dfw=torch.empty_like(b["fw"]))
    b["ws"] = torch.empty(N.lib().ctl_base_loss_workspace_bytes(C.byref(cfg)), dtype=torch.uint8, device="cuda")
    return b


OUT_KEYS = ("out", "df", "dc", "dbw", "dfw", "rm", "rv")


@pytest.mark.parametrize("margin,dist", [(0.5, "euclidean"), (None, "cosine")])
def test_base_step_graph_replay_and_repeat_are_bit_identical(margin, dist):
    """One enqueue, no host synchronisation, fixed-order reductions: two eager calls and the replay of a captured CUDA
    graph give identical bits (outputs, every gradient, the updated running statistics)."""
    cfg = _cfg(256, DIM, NUM_CLASSES, margin, dist)
    b = _buffers("p16k16_pad", cfg)
    runs = []
    for _ in range(2):
        b["rm"].zero_()
        b["rv"].fill_(1.0)
        assert _raw_step(cfg, b) == 0
        torch.cuda.synchronize()
        runs.append({k: b[k].clone() for k in OUT_KEYS})
    for k in ("df", "dc", "dbw", "dfw"):
        b[k].fill_(float("nan"))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        assert _raw_step(cfg, b) == 0
    b["rm"].zero_()
    b["rv"].fill_(1.0)
    graph.replay()
    torch.cuda.synchronize()
    runs.append({k: b[k].clone() for k in OUT_KEYS})
    assert torch.isfinite(runs[0]["out"]).all() and torch.isfinite(runs[0]["df"]).all()
    for other in runs[1:]:
        for k in OUT_KEYS:
            assert torch.equal(runs[0][k], other[k]), k


def test_base_step_input_errors():
    """A label outside [0, C) poisons every output (the model raises ValueError on it) without indexing the centers out
    of range; a workspace one byte short returns CTL_ERR_WORKSPACE before any device work."""
    from ctl_b200 import _native as N
    from ctl_b200.modelling.base_model import BaseModel
    from test_modules_gpu import _cfg as model_cfg

    cfg = _cfg(32, DIM, NUM_CLASSES)
    b = _buffers("p8k4_pad", cfg)
    need = b["ws"].numel()
    assert _raw_step(cfg, b, need - 1) == -2 and b"workspace too small" in N.lib().ctl_last_error()
    b["lab"][5] = NUM_CLASSES
    assert _raw_step(cfg, b) == 0
    out = b["out"].cpu()
    assert torch.isnan(out).all() and ((out.view(torch.int32) & 0x3FFFFF) == 1).all()
    model = BaseModel(model_cfg(), num_classes=16, num_query=4).cuda().train()
    feats = torch.randn(8, 2048, device="cuda")
    labels = torch.tensor([0, 0, 3, 3, 5, 5, 16, 16], device="cuda")
    with pytest.raises(ValueError, match="outside"):
        model.training_step_from_features(feats, labels, torch.ones(8, dtype=torch.bool, device="cuda"))


def _model(name):
    from ctl_b200.modelling.base_model import BaseModel
    from oracle import basic_oracle as BO
    from test_modules_gpu import _cfg as model_cfg

    torch.manual_seed(0)
    emb = 512 if name == "resnet18" else 2048
    cfg = model_cfg(MODEL__NAME=name, MODEL__BACKBONE_EMB_SIZE=emb)
    cfg["SOLVER"].update(dict(OPTIMIZER_NAME="Adam", BASE_LR=3.5e-4, WEIGHT_DECAY=5e-4, CENTER_LR=0.5,
                              LR_SCHEDULER_NAME="multistep_lr", LR_STEPS=(40, 70), GAMMA=0.1, USE_WARMUP_LR=False,
                              WARMUP_EPOCHS=10))
    model = BaseModel(cfg, num_classes=16, num_query=4).cuda().train()
    if name == "resnet18":
        sd = BO.make_trunk_state(seed=9)
        feats_of = lambda x: BO.trunk_train_fp16sim(x, sd)[0]  # noqa: E731
    else:
        sd = O.make_trunk_state(seed=9)
        feats_of = lambda x: O.trunk_train_fp16sim(x, sd)[0]  # noqa: E731
    model.backbone.base.load_state_dict(sd)
    return model, feats_of


@pytest.mark.parametrize("name", ["resnet50", "resnet18"])
def test_base_model_training_step_end_to_end(name):
    """BaseModel.training_step with optimizers attached (train_base_model.py:38-96): train-mode trunk -> fused base loss
    -> backward through the trunk -> Adam + center SGD, on 4 x 4 crops of 64x32 with one mock row.  Every parameter but
    the frozen bn.bias gets a finite gradient; the loss matches the oracle on the fp16-simulated train-mode features;
    losses_dict and the returned dict have the reference's shape; three iterations lower the loss."""
    model, feats_of = _model(name)
    (opt, opt_center), _ = model.configure_optimizers()
    model.attach_optimizers(opt, opt_center)
    P_, K_ = 4, 4
    g = torch.Generator().manual_seed(6)
    x = torch.randn(P_ * K_, 3, 64, 32, generator=g)
    labels = torch.arange(P_).repeat_interleave(K_) + 3
    is_real = torch.ones(P_ * K_, dtype=torch.bool)
    is_real[K_ - 1] = False  # last slot of the first pid is a mock image (all-zero crop, datasets/bases.py:378-391)
    x[K_ - 1] = 0
    batch = (x.cuda(), labels.cuda(), torch.zeros(P_ * K_, dtype=torch.long).cuda(), is_real.cuda())
    hs = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}  # before the optimizers move them
    out = model.training_step(batch, 0)
    assert set(out) == {"loss", "other"} and set(out["other"]) == {"step_dist_ap", "step_dist_an"}
    assert list(model.losses_dict) == ["query_xent", "query_triplet", "query_center", "centroid_triplet"]
    assert [len(v) for v in model.losses_dict.values()] == [1, 1, 1, 0]
    for pname, p in model.named_parameters():
        if pname == "bn.bias":  # frozen in the reference (bases.py:83-84)
            continue
        assert p.grad is not None and torch.isfinite(p.grad).all(), pname
    assert float(model.backbone.base.layer1[0].conv1.weight.grad.abs().max()) > 0
    ref = base_step_losses(feats_of(x).float(), labels, is_real, hs["center_loss.centers"], hs["bn.weight"],
                           hs["bn.bias"], hs["fc_query.weight"])
    np.testing.assert_allclose(float(out["loss"]), float(ref["total"]), rtol=5e-3)
    np.testing.assert_allclose(out["other"]["step_dist_ap"], float(ref["dist_ap"]), rtol=5e-3)
    np.testing.assert_allclose(out["other"]["step_dist_an"], float(ref["dist_an"]), rtol=5e-3)
    np.testing.assert_allclose(sum(model.losses_dict[k][0] for k in ("query_xent", "query_triplet", "query_center")),
                               float(out["loss"]), rtol=1e-6)
    losses = [float(out["loss"])]
    for _ in range(2):
        losses.append(float(model.training_step(batch, 0)["loss"]))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    assert all(torch.isfinite(p_).all() for p_ in model.parameters())
