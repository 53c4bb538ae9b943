"""GPU: the BasicBlock trunks (ResNet18 / ResNet34) through the eval and training handles.

Checkers: the 3x3 + 1x1 K-concatenated GEMM against float64 on the same fp16 operands (1 fp16 ulp + 1e-3); the eval
trunk against oracle.basic_oracle.trunk_forward_fp16sim (3e-3 of the feature scale) and the reference's autocast
features (tests/golden/trunk_basic.npz); the training trunk against the float64 oracle that tests/test_basic_trunk_cpu.py
pins to the reference's own float64 autograd."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden
from oracle import basic_oracle as B

pytestmark = pytest.mark.gpu

NAMES = [("r18", "resnet18"), ("r34", "resnet34")]


def _head(seed=0, d=512):
    g = torch.Generator().manual_seed(seed)
    return dict(weight=torch.rand(d, generator=g) + 0.5, bias=torch.randn(d, generator=g) * 0.1,
                running_mean=torch.randn(d, generator=g) * 0.1, running_var=torch.rand(d, generator=g) + 0.5)


def _engine(name, seed=7, last_stride=1, head=None):
    from ctl_b200.modelling.backbones.engine import TrunkEngine

    sd = B.make_trunk_state(seed=seed, layers=B.BASIC_LAYERS[name])
    eng = TrunkEngine(sd, "cuda", last_stride=last_stride, layers=B.BASIC_LAYERS[name], bn_head=head, block="basic")
    return sd, eng


@pytest.mark.parametrize("case", [
    # n, ho, wo, cin1, cin2, cout, stride2, relu
    (2, 32, 16, 128, 64, 128, 2, 1),     # layer2.0 at 256x128
    (2, 16, 8, 256, 128, 256, 2, 1),     # layer3.0
    (2, 8, 4, 512, 256, 512, 2, 1),      # layer4.0, LAST_STRIDE 2
    (2, 16, 8, 512, 256, 512, 1, 1),     # layer4.0, LAST_STRIDE 1: stride-1 shortcut
    (16, 32, 16, 128, 64, 128, 2, 0),    # many tiles per CTA, no ReLU
    (3, 10, 10, 128, 64, 128, 2, 1),     # partial tiles
    (1, 5, 3, 64, 64, 64, 1, 1),         # tiny, heavily over-covered tile
])
def test_conv3x3_dual_shortcut(case):
    """ctl_conv3x3_dual_nhwc_f16 == act(conv3x3(x1; W[:, :9 cin1]) + W[:, 9 cin1:] x2[::s, ::s] + b) in float64 on the
    same fp16 operands."""
    from ctl_b200 import _native as N

    n, ho, wo, c1, c2, cout, s2, relu = case
    g = torch.Generator().manual_seed(n * 1000 + cout + s2)
    x1 = (torch.randn(n, ho, wo, c1, generator=g) * 0.5).half()
    x2 = (torch.randn(n, ho * s2, wo * s2, c2, generator=g) * 0.5).half()
    w = (torch.randn(cout, 9 * c1 + c2, generator=g) / ((9 * c1 + c2) ** 0.5)).half()
    bias = torch.randn(cout, generator=g) * 0.1
    w3 = w[:, :9 * c1].double().reshape(cout, 3, 3, c1).permute(0, 3, 1, 2)
    ref = F.conv2d(x1.double().permute(0, 3, 1, 2), w3, None, 1, 1).permute(0, 2, 3, 1)
    ref = ref + torch.einsum("nhwc,oc->nhwo", x2[:, ::s2, ::s2].double(), w[:, 9 * c1:].double()) + bias.double()
    if relu:
        ref = ref.clamp(min=0)
    x1d, x2d, wd, bd = x1.cuda(), x2.cuda(), w.cuda(), bias.cuda()
    out = torch.full((n, ho, wo, cout), float("nan"), dtype=torch.float16, device="cuda")
    N.check(N.lib().ctl_conv3x3_dual_nhwc_f16(x1d.data_ptr(), c1, x2d.data_ptr(), ho * s2, wo * s2, c2, s2, n,
                                              wd.data_ptr(), bd.data_ptr(), out.data_ptr(), cout, relu, N.stream_ptr()))
    torch.cuda.synchronize()
    got = out.cpu().double()
    assert torch.isfinite(got).all(), "unwritten or non-finite outputs"
    err = (got - ref).abs()
    bad = err > ref.abs() * 2.0 ** -10 + 1e-3
    assert not bad.any(), f"{int(bad.sum())} / {bad.numel()} outputs off; max err {float(err.max()):.4e}"


@pytest.mark.parametrize("case", [
    # n, h, w, relu, seed: 3x3 / 1, 64 -> 64 with an identity residual (the halo-slab kernel's residual slab)
    (2, 64, 32, 1, 0),     # layer1 conv2 at 256x128
    (2, 64, 32, 0, 1),     # no ReLU (the training data gradient)
    (64, 64, 32, 1, 2),    # many tiles per CTA: the residual slab is refilled while the next tile's MMAs run
    (3, 20, 12, 1, 3),     # partial tiles in both directions
    (1, 7, 5, 1, 4),       # one heavily over-covered tile
])
def test_conv3x3_c64_residual(case):
    """ctl_conv2d_nhwc_f16 for a 64 -> 64 3x3 / 1 convolution with a residual == act(conv + residual + b) in float64 on
    the same fp16 operands, within 1 fp16 ulp + 1e-3."""
    from test_trunk_gpu import _conv_case

    n, h, w, relu, seed = case
    _conv_case(n, h, w, 64, 64, 3, 1, bool(relu), True, seed=seed)


@pytest.mark.parametrize("tag,name", NAMES)
@pytest.mark.parametrize("ls", [1, 2])
def test_basic_trunk_matches_checker_and_reference_autocast(tag, name, ls):
    """Features within 3e-3 of the fp16 checker; against the reference under fp16 autocast within 2e-3 of the feature
    scale and within 3x the reference's own autocast-vs-fp32 distance (DESIGN section 4); `emb` is the folded
    512-wide BatchNorm1d of the features."""
    g = load_golden("trunk_basic.npz")
    head = _head()
    sd, eng = _engine(name, B.EVAL_SEED, ls, head)
    x = B.eval_input()
    out = eng.forward(x.cuda(), want_emb=True)
    feat = out["global_feat"].cpu()
    assert feat.shape == (2, 512) and out["emb"].shape == (2, 512)
    with torch.no_grad():
        _, sim = B.trunk_forward_fp16sim(x, sd, last_stride=ls, layers=B.BASIC_LAYERS[name])
    amp, f32 = torch.from_numpy(g[f"{tag}_ls{ls}_eval_feat_amp"]), torch.from_numpy(g[f"{tag}_ls{ls}_eval_feat_fp32"])
    scale = float(f32.abs().max())
    e_sim = float((feat - sim).abs().max()) / float(sim.abs().max())
    e_amp = float((feat - amp).abs().max()) / scale
    e_f32 = float((feat - f32).abs().max()) / scale
    ref_own = float(g[f"{tag}_ls{ls}_amp_vs_fp32"])
    print(f"{tag} ls{ls}: vs fp16-sim {e_sim:.3e}, vs reference autocast {e_amp:.3e}, vs reference fp32 {e_f32:.3e}, "
          f"reference autocast vs its fp32 {ref_own:.3e}")
    assert e_sim <= 3e-3
    assert e_amp <= 2e-3 and e_f32 <= 3.0 * ref_own
    emb_ref = F.batch_norm(feat, head["running_mean"], head["running_var"], head["weight"], head["bias"], False, 0.1, 1e-5)
    np.testing.assert_allclose(out["emb"].cpu().numpy(), emb_ref.numpy(), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("name,ls,hw,n", [("resnet18", 1, (256, 128), 6), ("resnet34", 2, (256, 128), 3),
                                          ("resnet34", 1, (110, 62), 2)])
def test_basic_stage_calls_and_graph_match_embed_forward(name, ls, hw, n):
    """The three stage calls and a CUDA-graph replay reproduce ctl_embed_forward bit for bit, with the same launch
    count (110 x 62 takes the tensor-core stem, whose temporary spans several of the basic walk's slots)."""
    from ctl_b200 import _native as N
    from ctl_b200.modelling.backbones.engine import GraphedForward

    L = N.lib()
    _, eng = _engine(name, 5, ls, _head(1))
    x = torch.randn(n, 3, *hw, generator=torch.Generator().manual_seed(8)).cuda()
    ws = torch.empty(L.ctl_embed_workspace_bytes(eng._h, n, *hw), dtype=torch.uint8, device="cuda")
    feat, emb = torch.empty(n, 512, device="cuda"), torch.empty(n, 512, device="cuda")
    N.check(L.ctl_embed_forward(eng._h, x.data_ptr(), n, hw[0], hw[1], feat.data_ptr(), emb.data_ptr(), ws.data_ptr(),
                                ws.numel(), N.stream_ptr()))
    launches = L.ctl_embed_launches(eng._h)
    out = eng.forward(x, want_emb=True)
    assert torch.isfinite(feat).all()
    assert torch.equal(out["global_feat"], feat) and torch.equal(out["emb"], emb)
    assert launches == eng.launches_per_forward
    graphed = GraphedForward(eng, x, want_emb=True)()
    assert torch.equal(graphed["global_feat"], feat) and torch.equal(graphed["emb"], emb)


@pytest.mark.parametrize("name", ["resnet18", "resnet34"])
def test_basic_batch_invariance_at_bench_shape(name):
    """Image i of a batch of 256 at 256x128 is bit-identical to the same image in a batch of 2."""
    _, eng = _engine(name, 7, 1, _head(2))
    x = torch.randn(256, 3, 256, 128, generator=torch.Generator().manual_seed(33)).cuda()
    full = eng.forward(x, want_emb=True)
    feat, emb = full["global_feat"].clone(), full["emb"].clone()
    assert torch.isfinite(feat).all()
    for lo in (0, 127, 254):
        small = eng.forward(x[lo:lo + 2].contiguous(), want_emb=True)
        assert torch.equal(small["global_feat"], feat[lo:lo + 2]) and torch.equal(small["emb"], emb[lo:lo + 2]), lo


def _rel(a, b):
    return float((a.double() - b.double()).abs().max()) / (float(b.double().abs().max()) + 1e-30)


@pytest.mark.parametrize("name,ls", [("resnet18", 1), ("resnet34", 2)])
def test_basic_trunk_train_step_against_float64_autograd(name, ls):
    """Train-mode forward + backward vs the float64 oracle with the engine's rounding points: features and running
    statistics of the independent forward within 2e-2; gradients teacher-forced through the engine's saved activations
    within 2e-2 (max-norm relative)."""
    from ctl_b200.modelling.backbones.engine_train import TrunkTrainer

    layers = B.BASIC_LAYERS[name]
    sd = B.make_trunk_state(seed=7, layers=layers)
    g = torch.Generator().manual_seed(1)
    n, H, W = 8, 128, 64
    x = torch.randn(n, 3, H, W, generator=g)
    dfeat = torch.randn(n, 512, generator=g) * 1e-3
    feat_o, _, running_o = B.trunk_train_fp16sim(x, sd, last_stride=ls, layers=layers)
    params = {k: v.clone().cuda() for k, v in sd.items() if v.is_floating_point()}
    tr = TrunkTrainer("cuda", last_stride=ls, layers=layers, grad_scale=4096.0, block="basic")
    feat = tr.forward(x.cuda(), params)
    torch.cuda.synchronize()
    assert feat.shape == (n, 512) and _rel(feat.cpu(), feat_o) <= 2e-2
    for k, v in running_o.items():
        assert _rel(params[k].cpu(), v) <= 2e-2, k
    nchw = lambda t: t.cpu().float().permute(0, 3, 1, 2)  # noqa: E731
    saved = tr.saved_activations()
    assert len(saved) == 1 + 2 * sum(layers) + 3
    forced = [(nchw(y), nchw(z)) for y, z in saved]
    grads = tr.backward(dfeat.cuda())
    torch.cuda.synchronize()
    feat_f, grads_f, _ = B.trunk_train_fp16sim(x, sd, dfeat, last_stride=ls, layers=layers, forced=forced)
    assert _rel(feat.cpu(), feat_f) <= 1e-5
    assert set(grads.keys()) == set(grads_f.keys())
    gscale = max(float(v.abs().max()) for v in grads_f.values())
    bad = {}
    for k, go in grads_f.items():
        gk = grads[k].cpu()
        assert gk.shape == go.shape and torch.isfinite(gk).all(), k
        if float(go.abs().max()) < 1e-6 * gscale:  # stem bn1.bias: cancelled by the next batch-statistics BN
            assert float(gk.abs().max()) <= 1e-3 * gscale, k
            continue
        r = _rel(gk, go)
        if r > 2e-2:
            bad[k] = r
    assert not bad, f"gradient mismatch (max-norm relative): {sorted(bad.items(), key=lambda t: -t[1])[:8]}"


@pytest.mark.parametrize("name,shape,ls", [("resnet18", (4, 64, 32), 1), ("resnet34", (3, 96, 64), 2)])
def test_basic_trunk_train_graphs_reproduce_eager_bits(name, shape, ls):
    """Two graphs=True steps are bit-identical to eager: features, every gradient and the running statistics."""
    from ctl_b200.modelling.backbones.engine_train import TrunkTrainer

    layers = B.BASIC_LAYERS[name]
    sd = B.make_trunk_state(seed=3, layers=layers)
    n, H, W = shape
    g = torch.Generator().manual_seed(8)
    xs = [torch.randn(n, 3, H, W, generator=g).cuda() for _ in range(2)]
    dfs = [(torch.randn(n, 512, generator=g) * 1e-3).cuda() for _ in range(2)]
    outs = []
    for graphs in (False, True):
        params = {k: v.clone().cuda() for k, v in sd.items() if v.is_floating_point()}
        tr = TrunkTrainer("cuda", last_stride=ls, layers=layers, graphs=graphs, block="basic")
        res = []
        for x, df in zip(xs, dfs):
            feat = tr.forward(x, params)
            grads = tr.backward(df)
            res.append((feat.clone(), {k: v.clone() for k, v in grads.items()}))
        torch.cuda.synchronize()
        outs.append((res, {k: v.clone() for k, v in params.items() if "running" in k}))
    (eager, run_e), (graph, run_g) = outs
    for (fe, ge), (fg, gg) in zip(eager, graph):
        assert torch.isfinite(fe).all() and torch.equal(fe, fg)
        assert set(ge) == set(gg) and all(torch.equal(ge[k], gg[k]) for k in ge)
    assert all(torch.equal(run_e[k], run_g[k]) for k in run_e)


def _model(name):
    from ctl_b200.modelling.ctl_model import CTLModel
    from test_modules_gpu import _cfg

    torch.manual_seed(0)
    cfg = _cfg(MODEL__NAME=name, MODEL__BACKBONE_EMB_SIZE=512, DATALOADER__NUM_INSTANCE=16)
    cfg["SOLVER"].update(dict(OPTIMIZER_NAME="Adam", BASE_LR=3.5e-4, WEIGHT_DECAY=5e-4, CENTER_LR=0.5,
                              LR_SCHEDULER_NAME="multistep_lr", LR_STEPS=(40, 70), GAMMA=0.1, USE_WARMUP_LR=False,
                              WARMUP_EPOCHS=10))
    model = CTLModel(cfg, num_classes=32, num_query=16).cuda().train()
    model.backbone.base.load_state_dict(B.make_trunk_state(seed=11, layers=B.BASIC_LAYERS[name]))
    return model


@pytest.mark.parametrize("name", ["resnet18", "resnet34"])
def test_basic_full_training_iterations_reduce_the_loss(name):
    """CTLModel with MODEL.NAME resnet18 / resnet34 and BACKBONE_EMB_SIZE 512: three complete iterations (train-mode
    trunk -> losses -> backward -> fused Adam + center SGD) at P x K = 16 x 16, 256x128: finite, parameters move, the
    loss decreases."""
    model = _model(name)
    (opt, opt_center), _ = model.configure_optimizers()
    g = torch.Generator().manual_seed(2)
    x = torch.randn(256, 3, 256, 128, generator=g).cuda()
    labels = (torch.arange(16).repeat_interleave(16) + 1).cuda()
    batch = (x, labels, torch.zeros(256, dtype=torch.long).cuda(), torch.ones(256, dtype=torch.bool).cuda())
    w0 = model.backbone.base.layer2[0].conv2.weight.detach().clone()
    losses = []
    for _ in range(3):
        for p_ in model.parameters():
            p_.grad = None
        out = model.training_step(batch, 0)
        out["loss"].backward()
        model.optimizer_step_manual(opt, opt_center, epoch=20)
        losses.append(float(out["loss"]))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    assert not torch.equal(w0, model.backbone.base.layer2[0].conv2.weight)
    assert all(torch.isfinite(p_).all() for p_ in model.parameters())


def test_basic_validation_epoch_end_on_512d_embeddings():
    """validation_step embeds through the 512-wide head; validation_epoch_end's CMC / mAP match the reference metric
    (oracle.r1_map_compute) on the same embeddings.  The crops of one identity share a base image, so the embeddings
    carry the identity; distances computed on the device and on the host still differ in the last bits, which may swap
    near-tied gallery rows, hence the small mAP tolerance."""
    from oracle import ctl_oracle as O

    model = _model("resnet18")
    nq, n = 16, 96
    g = torch.Generator().manual_seed(5)
    pids = torch.arange(n) % 24
    cams = (torch.arange(n) // 24) % 4
    base = torch.randn(24, 3, 256, 128, generator=g)
    x = base[pids] + 0.5 * torch.randn(n, 3, 256, 128, generator=g)
    outs = [model.validation_step((x[i:i + 32].cuda(), pids[i:i + 32], cams[i:i + 32], torch.arange(i, i + 32)), 0)
            for i in range(0, n, 32)]
    emb = torch.cat([o["emb"] for o in outs]).cpu()
    assert emb.shape == (n, 512) and torch.isfinite(emb).all()
    cmc, mAP, topk = model.validation_epoch_end(outs)
    cmc_o, mAP_o, topk_o = O.r1_map_compute(emb, pids.numpy(), cams.numpy(), nq)
    assert mAP_o > 0.5
    np.testing.assert_allclose(mAP, mAP_o, atol=2e-3)
    np.testing.assert_allclose(cmc, cmc_o, atol=1.0 / nq + 1e-9)
