"""CPU: host-side logic of the package (no GPU compute calls)."""
import ctypes
import os
import re

import numpy as np
import pytest

import ctl_b200
from conftest import ROOT, load_golden
from ctl_b200 import _native as N
from ctl_b200 import retrieval as R
from ctl_b200.utils.eval_reid import eval_func
from oracle import ctl_oracle as O


def test_abi_version_5_and_every_declared_symbol_exported():
    """The shared library loads, reports ABI version 5 and exports exactly what include/ctl_b200.h declares."""
    header = open(os.path.join(ROOT, "include", "ctl_b200.h")).read()
    declared = set(re.findall(r"\b(ctl_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    lib = ctypes.CDLL(N.LIB_PATH)
    missing = [n for n in sorted(declared) if not hasattr(lib, n)]
    assert not missing, f"declared in the header but not exported: {missing}"
    assert declared == set(N.SIGNATURES), declared ^ set(N.SIGNATURES)
    assert N.lib().ctl_abi_version() == 5


def test_no_cpu_fallback():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        R.build_planes(torch.zeros(4, 64))
    assert N.lib().ctl_device_check() != 0
    assert b"CUDA" in N.lib().ctl_last_error() or b"device" in N.lib().ctl_last_error()


def test_key_encoding_orders_like_distance_then_index():
    L = N.lib()
    vals = [-3.5, -0.0, 0.0, 1e-30, 1.0, 1.0000001, 7.25, float("inf")]
    keys = [L.ctl_key_encode(v, 5) for v in vals]
    assert keys == sorted(keys)
    assert L.ctl_key_encode(1.0, 3) < L.ctl_key_encode(1.0, 4) < L.ctl_key_encode(1.0000001, 0)
    d, i = ctypes.c_float(), ctypes.c_uint32()
    L.ctl_key_decode(L.ctl_key_encode(-2.75, 123456), ctypes.byref(d), ctypes.byref(i))
    assert d.value == -2.75 and i.value == 123456


@pytest.mark.parametrize("name", ["small", "ties"])
def test_eval_func_matches_reference_golden(name):
    g = load_golden(f"retrieval_{name}.npz")
    nq, ng = int(g["num_q"]), int(g["num_g"])
    _, pids, cams = O.synth_retrieval(nq, ng, int(g["num_ids"]), 2048, float(g["sigma"]), int(g["seed"]),
                                      dyadic=bool(g["dyadic"]))
    idx = O.rank_indices(g["dist"])
    cmc, mAP, topk, single = eval_func(idx, pids[:nq], pids[nq:], cams[:nq], cams[nq:], 50)
    assert np.array_equal(cmc, g["cmc"])
    np.testing.assert_allclose(mAP, float(g["mAP"]), rtol=1e-12)
    np.testing.assert_allclose(topk, g["all_topk"], rtol=1e-12)
    np.testing.assert_allclose(single[:, 2].astype(np.float64), g["ap"], rtol=1e-12)


def test_eval_func_respect_camids_matches_oracle():
    g = load_golden("centroids.npz")
    nq = int(g["num_q"])
    feats, pids, cams = O.synth_retrieval(nq, int(g["num_g"]), int(g["num_ids"]), 2048, 3.0, 11, num_cams=4)
    emb, lab, cam = O.validation_create_centroids(feats, pids, cams, nq, True)
    import torch

    f = torch.nn.functional.normalize(emb.float(), dim=1)
    idx = O.rank_indices(O.get_euclidean(f[:nq], f[nq:]).numpy())
    cmc, mAP, topk, single = eval_func(idx, lab[:nq], lab[nq:], cam[:nq], cam[nq:], 50, True)
    assert np.array_equal(cmc, g["cam_cmc"])
    np.testing.assert_allclose(mAP, float(g["cam_mAP"]), rtol=1e-12)
    np.testing.assert_allclose(single[:, 2].astype(np.float64), g["cam_ap"], rtol=1e-12)


def test_encode_identities_masks():
    qp, qc, gp, gm, max_pos = R.encode_identities([5, 9], [9, 9, 5, 7], [0, 3], [[0, 3], [1], [3], [0]], True)
    assert qp.tolist() == [0, 2] and gp.tolist() == [2, 2, 0, 1]
    assert max_pos == 2
    cams = {0: 0, 1: 1, 3: 2}
    assert gm.tolist() == [(1 << cams[0]) | (1 << cams[3]), 1 << cams[1], 1 << cams[3], 1 << cams[0]]
    assert qc.tolist() == [cams[0], cams[3]]


def test_ctl_model_under_a_lightning_like_base(monkeypatch):
    """ADVICE r1: with pytorch_lightning importable, `hparams` is a PL property (PL 1.1.4: getter + setter backed by
    `_hparams`), so assigning through `__dict__` never populated it.  A stub LightningModule with that property checks
    that CTLModel sets the hyper-parameters through the setter, saves them, builds its modules, and exposes the
    reference's manual-optimisation hooks."""
    import importlib
    import sys
    import types

    import torch.nn as nn

    class AttributeDict(dict):
        __getattr__ = dict.__getitem__
        __setattr__ = dict.__setitem__

    class LightningModule(nn.Module):
        def __init__(self):
            super().__init__()
            self._hparams = AttributeDict()
            self.trainer = None
            self.saved = None

        @property
        def hparams(self):
            return self._hparams

        @hparams.setter
        def hparams(self, hp):
            self._hparams = hp

        def save_hyperparameters(self, *args, **kw):
            self.saved = args[0] if args else None

        def optimizers(self, use_pl_optimizer=True):
            return self.trainer.optimizers

        def manual_backward(self, loss, optimizer=None):
            loss.backward()

    pl = types.ModuleType("pytorch_lightning")
    pl.LightningModule = LightningModule
    util = types.ModuleType("pytorch_lightning.utilities")
    util.AttributeDict = AttributeDict
    pl.utilities = util
    monkeypatch.setitem(sys.modules, "pytorch_lightning", pl)
    monkeypatch.setitem(sys.modules, "pytorch_lightning.utilities", util)
    import ctl_b200.modelling.ctl_model as M

    try:
        M = importlib.reload(M)
        assert M._Base is LightningModule

        class Cfg(dict):
            __getattr__ = dict.__getitem__

        cfg = Cfg(MODEL=Cfg(NAME="resnet50", LAST_STRIDE=1, PRETRAINED=False, PRETRAIN_PATH="", BACKBONE_EMB_SIZE=2048,
                            USE_CENTROIDS=False, KEEP_CAMID_CENTROIDS=True, RESUME_TRAINING=False),
                  SOLVER=Cfg(MARGIN=0.5, DISTANCE_FUNC="euclidean", CENTER_LOSS_WEIGHT=5e-4, QUERY_XENT_WEIGHT=1.0,
                             QUERY_CONTRASTIVE_WEIGHT=1.0, CENTROID_CONTRASTIVE_WEIGHT=1.0),
                  DATALOADER=Cfg(NUM_INSTANCE=4), TEST=Cfg(FEAT_NORM=True, ONLY_TEST=False, VISUALIZE="no"),
                  USE_MIXED_PRECISION=True)
        model = M.CTLModel(cfg, num_classes=17, num_query=3)
        assert isinstance(model.hparams, AttributeDict) and model.hparams.MODEL.NAME == "resnet50"
        assert model.hparams.num_classes == 17 and model.saved is model.hparams
        assert model.fc_query.weight.shape == (17, 2048) and hasattr(model.backbone, "base")
        assert model._step_optimizers() is None  # no trainer attached: training_step returns the loss only

        class _T:
            current_epoch = 3
            optimizers = ("opt", "opt_center")

        model.trainer = _T()
        assert model._step_optimizers() == ("opt", "opt_center")  # train_ctl_model.py:39 under a Trainer
    finally:
        monkeypatch.undo()
        importlib.reload(M)


def test_runtime_switches_are_the_known_ones():
    """Every environment variable the package reads.  An A/B switch left in a kernel or engine is a second code path
    nobody runs; a new read must be added here on purpose."""
    allowed = {
        ("csrc/common.h", "CTL_PDL"),  # rules out launch-overlap ordering when diagnosing a fault
        ("modelling/baseline.py", "CTL_TRAIN_GRAPHS"),
        ("modelling/baseline.py", "CTL_DYNAMIC_LOSS_SCALE"),
        ("modelling/ctl_model.py", "CTL_VALIDATE_BATCH"),
    }
    pkg = os.path.join(ROOT, "centroids-reid_b200")
    found = set()
    for dirpath, _, names in os.walk(pkg):
        for name in names:
            if not name.endswith((".py", ".cu", ".cuh", ".h")):
                continue
            path = os.path.join(dirpath, name)
            rel = os.path.relpath(path, pkg).replace(os.sep, "/")
            for line in open(path, encoding="utf-8"):
                if "getenv(" in line or "os.environ" in line:
                    m = re.search(r"(?:getenv\(|os\.environ(?:\.get\(|\[))\s*[\"'](\w+)[\"']", line)
                    found.add((rel, m.group(1) if m else line.strip()))
    assert found == allowed, found ^ allowed


def test_no_undefined_names_in_the_python_sources():
    """GPU-only branches (sharded retrieval, NCCL paths) are not executed by the CPU suite: a static scan keeps a typo in them
    from surviving until a GPU run (tools/undefined_names.py: names loaded in a function that are bound nowhere)."""
    import subprocess
    import sys
    from pathlib import Path

    root = Path(__file__).resolve().parents[1]
    files = [str(p) for p in list((root / "centroids-reid_b200").rglob("*.py")) + [root / "bench.py", root / "__graft_entry__.py"]
             + list((root / "tools").glob("*.py"))]
    r = subprocess.run([sys.executable, str(root / "tools" / "undefined_names.py")] + files, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout
