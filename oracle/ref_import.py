"""TEST INFRASTRUCTURE ONLY -- never imported by the product path.

Imports the UNMODIFIED reference (mikwieczorek/centroids-reid, mounted read-only at
/root/reference) *in place* so that its own functions can be executed on CPU to pin the
oracle restatement (``oracle/ctl_oracle.py``) and to generate the golden vectors committed
under ``tests/golden/`` (``oracle/make_golden.py``).

The reference pins pytorch_lightning==1.1.4 / yacs / mlflow, none of which is installed in
this image and none of which takes part in the arithmetic of the hot path, so they are
replaced by ~60 lines of ``sys.modules`` stubs (SURVEY.md section 8c).  Two constructor
defaults (``use_gpu=True`` with hard ``.cuda()`` calls, losses/center_loss.py:21-22,40 and
losses/triplet_loss.py:187,202) are switched to ``use_gpu=False`` -- that is the only
behavioural patch, and it does not touch any arithmetic.

Where /root/reference is absent the module imports the verbatim copy ``oracle/_ref`` made by
``oracle/vendor_ref.py`` (git-ignored); that is used only by ``bench.py --impl reference`` / the
``cpu_baseline`` legs (the reference timed on the host cores) and by ``oracle/make_golden.py``.
No test imports the reference: tests compare against tests/golden/.
"""
from __future__ import annotations

import copy
import os
import sys
import types

_VENDORED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")  # oracle/vendor_ref.py (git-ignored)


def _default_root():
    if os.path.isfile("/root/reference/train_ctl_model.py"):
        return "/root/reference"
    return _VENDORED  # the verbatim copy made by oracle/vendor_ref.py


REFERENCE_ROOT = os.environ.get("CTL_REFERENCE_ROOT") or _default_root()


def reference_available() -> bool:
    return os.path.isfile(os.path.join(REFERENCE_ROOT, "train_ctl_model.py"))


class _AttributeDict(dict):
    """pytorch_lightning.utilities.AttributeDict: a dict with attribute access."""

    def __getattr__(self, key):
        try:
            return self[key]
        except KeyError as exc:  # pragma: no cover
            raise AttributeError(key) from exc

    def __setattr__(self, key, val):
        self[key] = val


class _CfgNode(_AttributeDict):
    """yacs.config.CfgNode look-alike: nested attribute dict with the merge helpers the
    reference calls (config/defaults.py:13, train_ctl_model.py:196-198)."""

    def clone(self):
        return copy.deepcopy(self)

    def merge_from_list(self, opts):
        assert len(opts) % 2 == 0
        for key, val in zip(opts[0::2], opts[1::2]):
            node = self
            parts = key.split(".")
            for p in parts[:-1]:
                node = node[p]
            old = node[parts[-1]]
            if isinstance(val, str) and not isinstance(old, str):
                import ast

                val = ast.literal_eval(val)
            node[parts[-1]] = val

    def merge_from_file(self, path):  # pragma: no cover - not used by the oracle
        import yaml

        def _merge(dst, src):
            for k, v in src.items():
                if isinstance(v, dict):
                    _merge(dst[k], v)
                else:
                    dst[k] = v

        with open(path) as f:
            _merge(self, yaml.safe_load(f))

    def freeze(self):
        pass

    def defrost(self):
        pass


def _install_stubs():
    import torch.nn as nn

    if "pytorch_lightning" in sys.modules and getattr(
        sys.modules["pytorch_lightning"], "__ctl_stub__", False
    ):
        return

    pl = types.ModuleType("pytorch_lightning")
    pl.__ctl_stub__ = True

    class LightningModule(nn.Module):
        """nn.Module + the handful of PL 1.1.4 hooks the reference's step functions touch."""

        def __init__(self, *a, **k):
            super().__init__()
            self.trainer = None
            self._ctl_optimizers = None

        def save_hyperparameters(self, *a, **k):
            pass

        def optimizers(self, use_pl_optimizer=True):
            return self._ctl_optimizers

        def manual_backward(self, loss, optimizer=None, *a, **k):
            loss.backward()

        @property
        def current_epoch(self):
            return self.trainer.current_epoch if self.trainer is not None else 0

    class LightningDataModule:
        def __init__(self, *a, **k):
            pass

    class Callback:
        pass

    class Trainer:
        def __init__(self, *a, **k):
            self.current_epoch = 0

    pl.LightningModule = LightningModule
    pl.LightningDataModule = LightningDataModule
    pl.Trainer = Trainer
    pl.Callback = Callback

    util = types.ModuleType("pytorch_lightning.utilities")
    util.AttributeDict = _AttributeDict
    util.rank_zero_only = lambda fn: fn
    seed = types.ModuleType("pytorch_lightning.utilities.seed")
    seed.seed_everything = lambda s=None: s
    dist = types.ModuleType("pytorch_lightning.utilities.distributed")
    dist.rank_zero_only = util.rank_zero_only
    cbs = types.ModuleType("pytorch_lightning.callbacks")
    cbs.ModelCheckpoint = type("ModelCheckpoint", (Callback,), {})
    cbs.Callback = Callback
    cbs_base = types.ModuleType("pytorch_lightning.callbacks.base")
    cbs_base.Callback = Callback
    loggers = types.ModuleType("pytorch_lightning.loggers")
    loggers.MLFlowLogger = type("MLFlowLogger", (), {})
    loggers.TensorBoardLogger = type("TensorBoardLogger", (), {})
    pl.utilities = util
    pl.callbacks = cbs
    pl.loggers = loggers

    sys.modules["pytorch_lightning"] = pl
    sys.modules["pytorch_lightning.utilities"] = util
    sys.modules["pytorch_lightning.utilities.seed"] = seed
    sys.modules["pytorch_lightning.utilities.distributed"] = dist
    sys.modules["pytorch_lightning.callbacks"] = cbs
    sys.modules["pytorch_lightning.callbacks.base"] = cbs_base
    sys.modules["pytorch_lightning.loggers"] = loggers

    yacs = types.ModuleType("yacs")
    yacs_cfg = types.ModuleType("yacs.config")
    yacs_cfg.CfgNode = _CfgNode
    yacs.config = yacs_cfg
    sys.modules["yacs"] = yacs
    sys.modules["yacs.config"] = yacs_cfg

    sys.modules.setdefault("mlflow", types.ModuleType("mlflow"))


_REF = None


def load_reference():
    """Returns a namespace with the reference's own modules (imported from REFERENCE_ROOT)."""
    global _REF
    if _REF is not None:
        return _REF
    if not reference_available():
        raise RuntimeError(
            f"reference tree not found at {REFERENCE_ROOT}; the golden vectors under "
            "tests/golden/ hold what the tests compare against"
        )
    _install_stubs()
    # The reference is used as a flat source tree with its root on sys.path
    # (e.g. `from losses.center_loss import CenterLoss`, modelling/bases.py:22).
    shadowed = [m for m in ("config", "losses", "modelling", "utils", "datasets", "solver",
                            "callbacks", "inference", "train_ctl_model") if m in sys.modules]
    if shadowed:
        raise RuntimeError(f"modules {shadowed} already imported; cannot import the reference in place")
    sys.path.insert(0, REFERENCE_ROOT)
    try:
        import warnings

        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            import config as ref_config
            import losses.center_loss as ref_center_loss
            import losses.triplet_loss as ref_triplet_loss
            import modelling.backbones.resnet as ref_resnet
            import modelling.backbones.resnet_ibn_a as ref_resnet_ibn_a
            import modelling.baseline as ref_baseline
            import modelling.bases as ref_bases
            import utils.eval_reid as ref_eval_reid
            import utils.reid_metric as ref_reid_metric
            import train_ctl_model as ref_train_ctl
            import inference.inference_utils as ref_inference_utils
    finally:
        sys.path.remove(REFERENCE_ROOT)

    # behaviour-neutral patch: the reference hard-codes .cuda() unless use_gpu=False
    _cl_init = ref_center_loss.CenterLoss.__init__

    def _cl_init_cpu(self, num_classes=751, feat_dim=2048, use_gpu=False):
        _cl_init(self, num_classes=num_classes, feat_dim=feat_dim, use_gpu=False)

    ref_center_loss.CenterLoss.__init__ = _cl_init_cpu
    _xe_init = ref_triplet_loss.CrossEntropyLabelSmooth.__init__

    def _xe_init_cpu(self, num_classes, epsilon=0.1, use_gpu=False):
        _xe_init(self, num_classes=num_classes, epsilon=epsilon, use_gpu=False)

    ref_triplet_loss.CrossEntropyLabelSmooth.__init__ = _xe_init_cpu

    ns = types.SimpleNamespace(
        config=ref_config,
        center_loss=ref_center_loss,
        triplet_loss=ref_triplet_loss,
        resnet=ref_resnet,
        resnet_ibn_a=ref_resnet_ibn_a,
        baseline=ref_baseline,
        bases=ref_bases,
        eval_reid=ref_eval_reid,
        reid_metric=ref_reid_metric,
        train_ctl=ref_train_ctl,
        inference_utils=ref_inference_utils,
        CfgNode=_CfgNode,
        AttributeDict=_AttributeDict,
    )
    _REF = ns
    return ns


def default_cfg(ref=None, **overrides):
    """A deep copy of the reference's config/defaults.py tree with dotted overrides."""
    ref = ref or load_reference()
    cfg = copy.deepcopy(ref.config.cfg)
    cfg.MODEL.PRETRAINED = False  # no ImageNet weights offline (modelling/baseline.py:84-87)
    flat = []
    for k, v in overrides.items():
        flat += [k.replace("__", "."), v]
    cfg.merge_from_list(flat)
    return cfg
