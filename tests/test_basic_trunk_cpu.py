"""CPU: the BasicBlock trunks (ResNet18 / ResNet34) without a GPU -- the BasicBlock oracle pinned against the
unmodified reference (tests/golden/trunk_basic.npz, written by `python -m oracle.basic_oracle`), the parameter tree's
state_dict layout, the C ABI's argument checks and workspace planning of the basic handles, and the embedding-width
check of CTLModel."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import ctl_b200  # noqa: F401
from oracle import basic_oracle as B
from oracle.make_golden import checksum, grad_sample

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "trunk_basic.npz")
NAMES = [("r18", "resnet18"), ("r34", "resnet34")]


def _gold():
    return np.load(GOLD, allow_pickle=False)


@pytest.mark.parametrize("tag,name", NAMES)
@pytest.mark.parametrize("ls", [1, 2])
def test_basic_oracle_matches_reference_eval(tag, name, ls):
    """fp32 eval features of the oracle equal the reference's ResNet(block=BasicBlock) at the bottleneck trunk's
    tolerance, and the fp16 simulation sits within 2e-3 of the feature scale of the reference's own autocast run."""
    g = _gold()
    x = B.eval_input()
    assert np.allclose(checksum(x), g["eval_in_checksum"], rtol=1e-12)
    sd = B.make_trunk_state(seed=B.EVAL_SEED, layers=B.BASIC_LAYERS[name])
    with torch.no_grad():
        feat = B.trunk_forward(x, sd, last_stride=ls, layers=B.BASIC_LAYERS[name]).mean(dim=(2, 3))
        _, sim = B.trunk_forward_fp16sim(x, sd, last_stride=ls, layers=B.BASIC_LAYERS[name])
    f32 = g[f"{tag}_ls{ls}_eval_feat_fp32"]
    np.testing.assert_allclose(feat.numpy(), f32, rtol=1e-4, atol=1e-5)
    scale = np.abs(f32).max()
    assert np.abs(sim.numpy() - g[f"{tag}_ls{ls}_eval_feat_amp"]).max() <= 2e-3 * scale
    assert np.abs(sim.numpy() - f32).max() <= 2e-3 * scale


@pytest.mark.parametrize("tag,name", NAMES)
def test_basic_train_oracle_pinned_against_reference_autograd(tag, name):
    """trunk_train_fp16sim with the storage rounding off is the reference's train-mode BasicBlock trunk in float64
    (features, sampled gradients, running statistics to 1e-7); with the rounding on it stays within fp16 distance."""
    g = _gold()
    x, dfeat = B.train_inputs()
    assert np.array_equal(g["train_in_checksum"], checksum(torch.cat((x.flatten(), dfeat.flatten()))))
    sd = B.make_trunk_state(seed=B.TRAIN_SEED, layers=B.BASIC_LAYERS[name])
    ref = g[f"{tag}_train_feat"]
    for rnd in (False, True):
        feat, grads, running = B.trunk_train_fp16sim(x, sd, dfeat, layers=B.BASIC_LAYERS[name], round_fp16=rnd)
        assert np.abs(feat.numpy() - ref).max() <= (5e-3 if rnd else 1e-7) * np.abs(ref).max()
        for k in B.TRAIN_GRAD_KEYS:
            got, exp = grad_sample(grads[k]), g[f"{tag}_train_grad_{k}"]
            if not rnd:
                assert np.abs(got[:-2] - exp[:-2]).max() <= 1e-7 * np.abs(exp[:-2]).max(), k
                assert abs(got[-1] - exp[-1]) <= 1e-7 * exp[-1], k
            else:  # ReLU masks flip under fp16 rounding: direction and size only
                cos = float(np.dot(got[:-2], exp[:-2]) / (np.linalg.norm(got[:-2]) * np.linalg.norm(exp[:-2])))
                assert cos >= 0.97 and abs(got[-1] / exp[-1] - 1) <= 1e-1, (k, cos)
        for k in B.TRAIN_RUN_KEYS:
            tol = dict(rtol=5e-3, atol=1e-5) if rnd else dict(rtol=1e-6, atol=1e-9)
            np.testing.assert_allclose(running[k].numpy(), g[f"{tag}_train_run_{k}"], **tol)


@pytest.mark.parametrize("tag,name", NAMES)
def test_basic_params_state_dict_matches_reference(tag, name):
    """ResNetParams(block="basic") has ResNet(block=BasicBlock)'s state_dict keys and shapes, so torchvision-layout
    ResNet18/34 checkpoints load through load_param; the oracle's synthetic state has them too."""
    from ctl_b200.modelling.backbones.resnet import ResNetParams

    g = _gold()
    keys = g[f"{tag}_state_keys"].tolist()
    shapes = g[f"{tag}_state_shapes"].tolist()
    sd = ResNetParams(1, B.BASIC_LAYERS[name], block="basic").state_dict()
    assert list(sd.keys()) == keys
    assert [",".join(str(d) for d in v.shape) for v in sd.values()] == shapes
    osd = B.make_trunk_state(layers=B.BASIC_LAYERS[name])
    assert sorted(osd.keys()) == sorted(keys)
    with pytest.raises(ValueError):
        ResNetParams(1, B.BASIC_LAYERS[name], ibn=True, block="basic")


def test_create_argument_errors_without_a_gpu():
    """Unknown block kinds, IBN-a BasicBlocks and a last stride of 3 are rejected by both create calls before any device
    work; feature_dim is a host query of the block kind."""
    from ctl_b200 import _native as N

    L = N.lib()
    r18 = (C.c_int32 * 4)(2, 2, 2, 2)
    cases = [
        lambda: L.ctl_trunk_create(C.byref(C.c_void_p()), 2, 0, 1, r18),                          # unknown block
        lambda: L.ctl_trunk_create(C.byref(C.c_void_p()), -1, 0, 1, r18),                         # unknown block
        lambda: L.ctl_trunk_create(C.byref(C.c_void_p()), N.CTL_BLOCK_BASIC, 1, 1, r18),           # basic + IBN
        lambda: L.ctl_trunk_create(C.byref(C.c_void_p()), N.CTL_BLOCK_BASIC, 0, 3, r18),           # LAST_STRIDE 3
        lambda: L.ctl_trainer_create(C.byref(C.c_void_p()), 2, 0, 1, 0.1, r18),                   # unknown block
        lambda: L.ctl_trainer_create(C.byref(C.c_void_p()), -1, 0, 1, 0.1, r18),                  # unknown block
        lambda: L.ctl_trainer_create(C.byref(C.c_void_p()), N.CTL_BLOCK_BASIC, 1, 1, 0.1, r18),    # basic + IBN
        lambda: L.ctl_trainer_create(C.byref(C.c_void_p()), N.CTL_BLOCK_BASIC, 0, 3, 0.1, r18),    # LAST_STRIDE 3
        lambda: L.ctl_trainer_create(C.byref(C.c_void_p()), N.CTL_BLOCK_BASIC, 0, 1, 0.0, r18),    # momentum 0
        lambda: L.ctl_conv3x3_dual_nhwc_f16(C.c_void_p(16), 64, C.c_void_p(16), 7, 8, 64, 2, 1, C.c_void_p(16),
                                            C.c_void_p(16), C.c_void_p(16), 128, 1, None),     # odd H2, stride 2
    ]
    for i, call in enumerate(cases):
        rc = call()
        assert rc == -1, (i, rc, L.ctl_last_error())
        assert len(L.ctl_last_error()) > 0
        with pytest.raises(ValueError):
            N.check(rc)
    for block, dim in ((N.CTL_BLOCK_BOTTLENECK, 2048), (N.CTL_BLOCK_BASIC, 512)):
        h, t = C.c_void_p(), C.c_void_p()
        assert L.ctl_trunk_create(C.byref(h), block, 0, 1, r18) == 0
        assert L.ctl_trainer_create(C.byref(t), block, 0, 1, 0.1, r18) == 0
        assert L.ctl_trunk_feature_dim(h) == dim and L.ctl_trainer_feature_dim(t) == dim
        L.ctl_trunk_destroy(h)
        L.ctl_trainer_destroy(t)
    assert L.ctl_trunk_feature_dim(None) == 0 and L.ctl_trainer_feature_dim(None) == 0


def test_basic_handles_plan_their_workspace_without_a_gpu():
    """Both workspace queries are host-side walks: non-zero for ResNet18 / ResNet34, growing with depth, and the eval
    workspace sized by the BasicBlock walk's own widest activation (layer1's 64 channels), not the bottleneck's 256."""
    from ctl_b200 import _native as N

    L = N.lib()
    n, H, W, hp, wp = 16, 256, 128, 64, 32
    ev, tr = {}, {}
    for name, layers in B.BASIC_LAYERS.items():
        h, t = C.c_void_p(), C.c_void_p()
        assert L.ctl_trunk_create(C.byref(h), N.CTL_BLOCK_BASIC, 0, 1, (C.c_int32 * 4)(*layers)) == 0
        assert L.ctl_trainer_create(C.byref(t), N.CTL_BLOCK_BASIC, 0, 1, 0.1, (C.c_int32 * 4)(*layers)) == 0
        ev[name], tr[name] = L.ctl_embed_workspace_bytes(h, n, H, W), L.ctl_train_workspace_bytes(t, n, H, W)
        slot = n * hp * wp * 64 * 2
        # three slots of layer1's output; the tensor-core stem's temporary [n, 128, 64, 64] starts at slot 1
        assert ev[name] == max(3 * slot, slot + n * 128 * 64 * 64 * 2)
        assert L.ctl_embed_workspace_bytes(h, n, 4 * hp, 4 * wp) == ev[name]
        assert L.ctl_train_workspace_bytes(t, 2 * n, H, W) > tr[name] > 0
        L.ctl_trunk_destroy(h)
        L.ctl_trainer_destroy(t)
    assert 0 < tr["resnet18"] < tr["resnet34"]
    assert 0 < ev["resnet18"] <= ev["resnet34"]
    hb = C.c_void_p()
    assert L.ctl_trunk_create(C.byref(hb), N.CTL_BLOCK_BOTTLENECK, 0, 1, (C.c_int32 * 4)(3, 4, 6, 3)) == 0
    assert ev["resnet34"] < L.ctl_embed_workspace_bytes(hb, n, H, W)
    L.ctl_trunk_destroy(hb)


def _cfg(name, emb):
    class Cfg(dict):
        __getattr__ = dict.__getitem__

    return Cfg(MODEL=Cfg(NAME=name, LAST_STRIDE=1, PRETRAINED=False, PRETRAIN_PATH="", BACKBONE_EMB_SIZE=emb,
                         RESUME_TRAINING=False, USE_CENTROIDS=True, KEEP_CAMID_CENTROIDS=False),
               TEST=Cfg(ONLY_TEST=False, FEAT_NORM=True), USE_MIXED_PRECISION=False,
               SOLVER=Cfg(MARGIN=0.3, DISTANCE_FUNC="euclidean", CENTER_LOSS_WEIGHT=5e-4),
               num_classes=10, num_query=4)


def test_backbone_emb_size_must_match_the_trunk_width():
    """MODEL.BACKBONE_EMB_SIZE sizes bn / fc_query / centers; the trunk's features are Baseline.in_planes wide.  A
    mismatch is refused at construction instead of computing with the wrong width."""
    from ctl_b200.modelling.baseline import Baseline
    from ctl_b200.modelling.ctl_model import CTLModel

    for name in ("resnet18", "resnet34"):
        assert Baseline(_cfg(name, 512)).in_planes == 512
        with pytest.raises(ValueError, match="BACKBONE_EMB_SIZE"):
            CTLModel(_cfg(name, 2048))
    assert Baseline(_cfg("resnet50", 2048)).in_planes == 2048
    with pytest.raises(ValueError, match="BACKBONE_EMB_SIZE"):
        CTLModel(_cfg("resnet50", 512))
    model = CTLModel(_cfg("resnet18", 512))
    assert model.bn.num_features == 512 and model.fc_query.in_features == 512
