"""Drop-in for modelling/baseline.py: Baseline(cfg).forward(x) -> (base_out, global_feat).

Parameters live in reference-layout modules (`self.base.*`); eval-mode forward runs the H100
engine, whose packed operands are rebuilt lazily whenever the parameters change
(`invalidate()`; call it after `opt.step()` / `load_state_dict`).  Train-mode forward runs the
training engine (batch-statistics BatchNorm, running statistics updated in place) and is differentiable:
`global_feat.backward()` fills `.grad` of every trunk parameter through the H100 backward kernels.
"""
from __future__ import annotations

import os

import torch
from torch import nn

from .backbones.engine import TrunkEngine
from .backbones.engine_train import TrunkTrainer
from .backbones.resnet import ResNetParams

# MODEL.NAME -> (blocks per stage, IBN-a, block kind); modelling/baseline.py:56-100
_LAYERS = {"resnet18": ((2, 2, 2, 2), False, "basic"), "resnet34": ((3, 4, 6, 3), False, "basic"),
           "resnet50": ((3, 4, 6, 3), False, "bottleneck"), "resnet101": ((3, 4, 23, 3), False, "bottleneck"),
           "resnet152": ((3, 8, 36, 3), False, "bottleneck"), "resnet50_ibn_a": ((3, 4, 6, 3), True, "bottleneck"),
           "resnet101_ibn_a": ((3, 4, 23, 3), True, "bottleneck")}


class _TrunkTrainFn(torch.autograd.Function):
    """global_feat = trunk(x; parameters) with the H100 training engine; backward returns the parameter gradients
    (the input crops get no gradient, like the reference's data tensors)."""

    @staticmethod
    def forward(ctx, x, trainer, scaler, names, buffers, *tensors):
        params = dict(zip(names, tensors))
        params.update(buffers)
        ctx.trainer, ctx.names, ctx.scaler = trainer, names, scaler
        return trainer.forward(x, params)

    @staticmethod
    def backward(ctx, dfeat):
        # dynamic loss scaling (the reference's PL native-AMP GradScaler, utils/misc.py:111): the fp16 backward runs on
        # (scale / trainer.grad_scale) * dfeat on top of the trainer's fixed internal scale and is un-scaled in fp32;
        # an overflow shows up as inf / NaN gradients, which CTLModel.optimizer_step_manual detects and skips
        sc = ctx.scaler if (ctx.scaler is not None and ctx.scaler.enabled) else None
        grads = ctx.trainer.backward(dfeat * sc.ratio if sc is not None else dfeat)  # ratio: a DEVICE scalar
        out = [grads.get(n) for n in ctx.names]
        if sc is not None:  # un-scale (and look for inf / NaN while the data is in flight): one multi-tensor launch
            sc.check([g for g in out if g is not None], mul_dev=sc.inv_ratio)
        return (None, None, None, None, None) + tuple(out)


class Baseline(nn.Module):
    in_planes = 2048

    def __init__(self, cfg):
        super().__init__()
        name = cfg.MODEL.NAME
        if name not in _LAYERS:
            raise NotImplementedError(f"MODEL.NAME={name!r}: the H100 trunk covers the ResNets {sorted(_LAYERS)}")
        layers, ibn, block = _LAYERS[name]
        self.in_planes = 512 if block == "basic" else 2048  # baseline.py:58-69
        self.model_name = name
        self.use_mixed_precision = cfg.USE_MIXED_PRECISION
        self.base = ResNetParams(cfg.MODEL.LAST_STRIDE, layers, ibn, block)
        if cfg.MODEL.PRETRAINED and not cfg.MODEL.RESUME_TRAINING and not cfg.TEST.ONLY_TEST:
            self.base.load_param(cfg.MODEL.PRETRAIN_PATH)  # modelling/baseline.py:84-87
            print("Loading pretrained ImageNet model......")
        self.gap = nn.AdaptiveAvgPool2d(1)
        self._engine = None
        self._engine_key = None
        self._trainer = None
        self.loss_scaler = None  # solver.build.DynamicLossScaler, created with the training engine

    def invalidate(self):
        self._engine = None

    def _param_version(self, bn_head=None):
        """Changes whenever any trunk parameter / buffer (or the BatchNorm1d head) is modified in place or replaced:
        optimizer steps, load_state_dict, load_param, EMA updates, running statistics."""
        ts = list(self.base.parameters()) + list(self.base.buffers())
        if bn_head is not None:
            ts += [bn_head.weight, bn_head.bias, bn_head.running_mean, bn_head.running_var]
        return tuple((t.data_ptr(), t._version) for t in ts)

    def engine(self, bn_head=None) -> TrunkEngine:
        dev = next(self.base.parameters()).device
        # the packed operands (folded BN, fp16 weights) are a cache of the parameters: keyed on their version counters,
        # so a stale pack can never be used after load_state_dict / an external optimizer / updated running statistics
        key = (str(dev), self._param_version(bn_head))
        if self._engine is not None and self._engine_key is not None and self._engine_key[0] == key[0] \
                and self._engine_key[1][: len(key[1])] == key[1] and bn_head is None:
            return self._engine  # a pack built WITH the head also serves calls without it (same trunk versions)
        if self._engine is None or self._engine_key != key:
            sd = {k: v for k, v in self.base.state_dict().items()}
            head = None
            if bn_head is not None:
                head = dict(weight=bn_head.weight, bias=bn_head.bias, running_mean=bn_head.running_mean,
                            running_var=bn_head.running_var)
            self._engine = TrunkEngine(sd, dev, ibn=self.base.ibn, last_stride=self.base.last_stride,
                                       layers=self.base.layers_cfg, bn_head=head, block=self.base.block)
            self._engine_key = key
        return self._engine

    def forward(self, x):
        """modelling/baseline.py:91-96.  base_out is returned in the reference's NCHW view."""
        if self.training:
            dev = next(self.base.parameters()).device
            if self._trainer is None or self._trainer.device != dev:
                from ..solver.build import DynamicLossScaler

                self._trainer = TrunkTrainer(dev, last_stride=self.base.last_stride, layers=self.base.layers_cfg,
                                             graphs=os.environ.get("CTL_TRAIN_GRAPHS", "1") == "1", ibn=self.base.ibn,
                                             block=self.base.block)
                self.loss_scaler = DynamicLossScaler(dev, base_scale=self._trainer.grad_scale,
                                                     enabled=os.environ.get("CTL_DYNAMIC_LOSS_SCALE", "1") == "1")
            names = [k for k, _ in self.base.named_parameters()]
            tensors = [v for _, v in self.base.named_parameters()]
            buffers = {k: v for k, v in self.base.named_buffers() if "running" in k}
            feat = _TrunkTrainFn.apply(x, self._trainer, self.loss_scaler, names, buffers, *tensors)
            from ..solver.build import _bump_version

            _bump_version(buffers.values())  # running statistics were updated in place by the kernels
            for k, v in self.base.named_buffers():
                if k.endswith("num_batches_tracked"):
                    v += 1
            return None, feat  # callers use only global_feat (train_ctl_model.py:55); base_out is not kept
        out = self.engine().forward(x, want_base=True)
        return out["base_out_nhwc"].permute(0, 3, 1, 2), out["global_feat"]


def embed(pl_module, x):
    """ModelBase.validation_step's arithmetic (modelling/bases.py:169-177) ==
    inference_utils._inference (inference/inference_utils.py:104-113): eval trunk -> GAP ->
    eval BatchNorm1d, fused into the engine's last kernel."""
    eng = pl_module.backbone.engine(bn_head=pl_module.bn)
    return eng.forward(x, want_emb=True)["emb"]
