"""TEST INFRASTRUCTURE ONLY -- CPU oracle of the BasicBlock trunks (ResNet18 / ResNet34) and the generator of
tests/golden/trunk_basic.npz.

The same restatement as the bottleneck functions of ``oracle/ctl_oracle.py`` (make_trunk_state, trunk_forward,
trunk_forward_fp16sim, trunk_train_fp16sim), for ResNet(block=BasicBlock) (modelling/backbones/resnet.py:19-48,
88-133; modelling/baseline.py:56-65).  ctl_oracle keeps the bottleneck trunks; the shared helpers are imported from it.

    python -m oracle.basic_oracle      runs the UNMODIFIED reference (oracle/ref_import.py) on the CPU and writes
                                       tests/golden/trunk_basic.npz, which pins this module (tests/test_basic_trunk_cpu.py)

This module stands beside oracle/ctl_oracle.py and oracle/make_golden.py instead of adding a `block=` keyword and a
`--only trunk_basic` entry to them: those two files pin the bottleneck trunks and every existing golden, and they are
kept byte-for-byte as they were.  So trunk_basic.npz is the one golden not listed in make_golden's --only set; its
recipe is `generate()` below (same seeds, checksums and grad_sample as make_golden's trunk generators).

Only tests/ and tools/ may import this module; the product never does.
"""
from __future__ import annotations

import math
import os
import sys
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ctl_oracle as O  # noqa: E402

BASIC_LAYERS = {"resnet18": (2, 2, 2, 2), "resnet34": (3, 4, 6, 3)}


def _stride0(li, last_stride):
    return 1 if li == 1 else (last_stride if li == 4 else 2)


def _blocks(layers, last_stride):
    """(prefix, planes, inplanes, stride, has_downsample) of every BasicBlock (resnet.py:103-120, expansion 1)."""
    out, inplanes = [], 64
    for li, (planes, nblk) in enumerate(zip((64, 128, 256, 512), layers), start=1):
        for b in range(nblk):
            stride = _stride0(li, last_stride) if b == 0 else 1
            # resnet.py:105; at last_stride 1 layer4.0 still has one, because it changes the width
            out.append((f"layer{li}.{b}", planes, inplanes, stride, stride != 1 or inplanes != planes))
            inplanes = planes
    return out


def make_trunk_state(seed=0, layers=BASIC_LAYERS["resnet18"], randomize_bn=True):
    """Deterministic synthetic weights with ResNet(block=BasicBlock)'s state_dict keys / shapes; conv weights
    ~ N(0, sqrt(2 / (k*k*Cout))) (resnet.py:156-164), BN affine and running statistics randomised.  The residual-branch
    BN (bn2) gets the small gain ctl_oracle gives bn3, so that the residual sum stays O(1) in fp16."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()

    def conv(name, cout, cin, k):
        sd[name + ".weight"] = torch.randn(cout, cin, k, k, generator=g) * math.sqrt(2.0 / (k * k * cout))

    def bn(name, c):
        if randomize_bn:
            gain = 0.25 if name.endswith("bn2") else 1.0
            sd[name + ".weight"] = gain * (0.5 + torch.rand(c, generator=g))
            sd[name + ".bias"] = 0.1 * torch.randn(c, generator=g)
            sd[name + ".running_mean"] = 0.1 * torch.randn(c, generator=g)
            sd[name + ".running_var"] = 0.5 + torch.rand(c, generator=g)
        else:
            sd[name + ".weight"] = torch.ones(c)
            sd[name + ".bias"] = torch.zeros(c)
            sd[name + ".running_mean"] = torch.zeros(c)
            sd[name + ".running_var"] = torch.ones(c)
        sd[name + ".num_batches_tracked"] = torch.zeros((), dtype=torch.long)

    conv("conv1", 64, 3, 7)
    bn("bn1", 64)
    for p, planes, inplanes, _, has_down in _blocks(layers, 1):
        conv(p + ".conv1", planes, inplanes, 3)
        bn(p + ".bn1", planes)
        conv(p + ".conv2", planes, planes, 3)
        bn(p + ".bn2", planes)
        if has_down:
            conv(p + ".downsample.0", planes, inplanes, 1)
            bn(p + ".downsample.1", planes)
    return sd


def trunk_forward(x, sd, last_stride=1, train=False, layers=BASIC_LAYERS["resnet18"]):
    """ResNet.forward (resnet.py:122-133, no ReLU after the stem) over BasicBlock.forward (resnet.py:31-47)
    -> base_out [B, 512, H/16, W/16] at last_stride 1."""
    x = F.conv2d(x, sd["conv1.weight"], None, 2, 3)
    x = F.max_pool2d(O._bn(x, sd, "bn1", train), 3, 2, 1)
    for p, _, _, stride, has_down in _blocks(layers, last_stride):
        out = F.relu(O._bn(F.conv2d(x, sd[p + ".conv1.weight"], None, stride, 1), sd, p + ".bn1", train))
        out = O._bn(F.conv2d(out, sd[p + ".conv2.weight"], None, 1, 1), sd, p + ".bn2", train)
        res = x
        if has_down:
            res = O._bn(F.conv2d(x, sd[p + ".downsample.0.weight"], None, stride), sd, p + ".downsample.1", train)
        x = F.relu(out + res)
    return x


def trunk_forward_fp16sim(x, sd, last_stride=1, layers=BASIC_LAYERS["resnet18"]):
    """trunk_forward(eval) with the H100 eval path's rounding points: BatchNorm folded into fp16 weights, fp32
    accumulation, every stored activation rounded to fp16.  A block with a downsample sums conv2 and the shortcut in
    one accumulator (ctl_conv3x3_dual_nhwc_f16), so its shortcut is never rounded on its own.
    Returns (base_out, global_feat)."""
    eps = 1e-5

    def fold(wname, bnname):
        sc = sd[bnname + ".weight"] / torch.sqrt(sd[bnname + ".running_var"] + eps)
        return sd[wname] * sc[:, None, None, None], sd[bnname + ".bias"] - sd[bnname + ".running_mean"] * sc

    def q(t):
        return t.half().float()

    w, b = fold("conv1.weight", "bn1")
    x = F.max_pool2d(q(F.conv2d(q(x), q(w), b, 2, 3)), 3, 2, 1)
    for p, _, _, stride, has_down in _blocks(layers, last_stride):
        w1, b1 = fold(p + ".conv1.weight", p + ".bn1")
        o1 = q(F.relu(F.conv2d(x, q(w1), b1, stride, 1)))
        w2, b2 = fold(p + ".conv2.weight", p + ".bn2")
        if has_down:
            wd, bd = fold(p + ".downsample.0.weight", p + ".downsample.1")
            x = q(F.relu(F.conv2d(o1, q(w2), b2, 1, 1) + F.conv2d(x, q(wd), bd, stride)))
        else:
            x = q(F.relu(F.conv2d(o1, q(w2), b2, 1, 1) + x))
    return x, x.mean(dim=(2, 3))


def trunk_train_fp16sim(x, sd, dfeat=None, last_stride=1, layers=BASIC_LAYERS["resnet18"], momentum=0.1, forced=None,
                        round_fp16=True):
    """Train-mode BasicBlock trunk in float64 with the H100 training path's rounding points (see
    ctl_oracle.trunk_train_fp16sim; round_fp16=False is the reference's own arithmetic in float64).  Returns
    (global_feat, grads, running).  `forced`: (y, z) NCHW tensors per conv + BatchNorm in the order the trainer saves
    them -- stem, then per block conv1, [downsample], conv2."""
    eps = 1e-5
    q = O._RoundHalfSTE.apply if round_fp16 else (lambda t: t)
    P = {k: v.detach().double().requires_grad_(True) for k, v in sd.items()
         if v.is_floating_point() and "running" not in k}
    running = {}
    it = iter(forced) if forced is not None else None

    def force(t, val):
        return t if val is None else val.double() + (t - t.detach())

    def batch_norm(y, name):
        mean = y.mean(dim=(0, 2, 3))
        var = y.var(dim=(0, 2, 3), unbiased=False)
        cnt = y.numel() / y.shape[1]
        running[name + ".running_mean"] = (1 - momentum) * sd[name + ".running_mean"].double() + momentum * mean.detach()
        running[name + ".running_var"] = ((1 - momentum) * sd[name + ".running_var"].double()
                                          + momentum * var.detach() * cnt / max(cnt - 1, 1))
        return ((y - mean[None, :, None, None]) / torch.sqrt(var + eps)[None, :, None, None]
                * P[name + ".weight"][None, :, None, None] + P[name + ".bias"][None, :, None, None])

    def conv_bn(a, conv, name, k, stride, res=None, relu=True):
        fy, fz = next(it) if it is not None else (None, None)
        y = force(q(F.conv2d(a, q(P[conv + ".weight"]), None, stride, k // 2)), fy)
        z = batch_norm(y, name)
        if res is not None:
            z = z + res
        return force(q(F.relu(z) if relu else z), fz)

    a = conv_bn(q(x.double()), "conv1", "bn1", 7, 2, relu=False)
    a = F.max_pool2d(a, 3, 2, 1)
    for p, _, _, stride, has_down in _blocks(layers, last_stride):
        o1 = conv_bn(a, p + ".conv1", p + ".bn1", 3, stride)
        res = a
        if has_down:
            res = conv_bn(a, p + ".downsample.0", p + ".downsample.1", 1, stride, relu=False)
        a = conv_bn(o1, p + ".conv2", p + ".bn2", 3, 1, res=res)
    feat = a.mean(dim=(2, 3))
    grads = None
    if dfeat is not None:
        (feat * dfeat.double()).sum().backward()
        grads = {k: v.grad for k, v in P.items()}
    return feat.detach(), grads, running


# --------------------------------------------------------------------------------------
# golden vectors: the unmodified reference on the CPU
# --------------------------------------------------------------------------------------

GOLD = os.path.join(ROOT, "tests", "golden", "trunk_basic.npz")
EVAL_SEED, TRAIN_SEED = 7, 17
TRAIN_GRAD_KEYS = ("conv1.weight", "bn1.weight", "layer1.0.conv1.weight", "layer1.0.bn1.weight", "layer2.0.conv1.weight",
                   "layer2.0.downsample.0.weight", "layer3.1.conv2.weight", "layer4.1.conv2.weight", "layer4.1.bn2.weight",
                   "layer4.1.bn2.bias")
TRAIN_RUN_KEYS = ("bn1.running_mean", "layer2.0.downsample.1.running_var", "layer4.1.bn2.running_var")


def eval_input(n=2, hw=(256, 128)):
    return torch.randn(n, 3, *hw, generator=torch.Generator().manual_seed(21))


def train_inputs():
    g = torch.Generator().manual_seed(23)
    x = torch.randn(4, 3, 64, 32, generator=g)
    return x, torch.randn(4, 512, generator=g) * 1e-2


def generate():
    from oracle.make_golden import checksum, grad_sample
    from oracle.ref_import import default_cfg, load_reference

    torch.set_num_threads(os.cpu_count())
    ref = load_reference()
    out = {}
    for name, layers in BASIC_LAYERS.items():
        tag = name.replace("resnet", "r")
        cfg = default_cfg(ref)
        cfg.MODEL.NAME = name
        base = ref.baseline.Baseline(cfg)
        ref_sd = base.base.state_dict()
        out[f"{tag}_state_keys"] = np.array(list(ref_sd.keys()))
        out[f"{tag}_state_shapes"] = np.array([",".join(str(d) for d in v.shape) for v in ref_sd.values()])
        out[f"{tag}_in_planes"] = int(base.in_planes)
        x = eval_input()
        out["eval_in_checksum"] = checksum(x)
        for ls in (1, 2):
            cfg = default_cfg(ref)
            cfg.MODEL.NAME, cfg.MODEL.LAST_STRIDE = name, ls
            base = ref.baseline.Baseline(cfg)
            sd = make_trunk_state(seed=EVAL_SEED, layers=layers)
            base.base.load_state_dict(sd, strict=True)
            base.eval()
            with torch.no_grad():
                _, f32 = base(x)
                with torch.autocast("cpu", dtype=torch.float16):
                    _, f16 = base(x)
            key = f"{tag}_ls{ls}"
            out[f"{key}_eval_feat_fp32"] = f32.float().numpy()
            out[f"{key}_eval_feat_amp"] = f16.float().numpy()
            rel = float((f16.float() - f32).abs().max() / f32.abs().max())
            out[f"{key}_amp_vs_fp32"] = rel
            print(f"{key}: feat std {float(f32.std()):.4f}, reference autocast vs fp32 {rel:.3e} of the feature scale")
        # train mode in float64 (batch statistics), LAST_STRIDE 1
        cfg = default_cfg(ref)
        cfg.MODEL.NAME = name
        base = ref.baseline.Baseline(cfg)
        sd = make_trunk_state(seed=TRAIN_SEED, layers=layers)
        base.base.load_state_dict(sd, strict=True)
        base.to(torch.float64).train()
        x, dfeat = train_inputs()
        _, feat = base(x.double())
        (feat * dfeat.double()).sum().backward()
        params, bufs = dict(base.base.named_parameters()), dict(base.base.named_buffers())
        out["train_in_checksum"] = checksum(torch.cat((x.flatten(), dfeat.flatten())))
        out[f"{tag}_train_feat"] = feat.detach().numpy()
        for k in TRAIN_GRAD_KEYS:
            out[f"{tag}_train_grad_{k}"] = grad_sample(params[k].grad)
        for k in TRAIN_RUN_KEYS:
            out[f"{tag}_train_run_{k}"] = bufs[k].numpy()
        print(f"{tag} train: feat std {float(feat.detach().std()):.4f}")
    np.savez_compressed(GOLD, **out)
    print("wrote", GOLD)


if __name__ == "__main__":
    generate()
