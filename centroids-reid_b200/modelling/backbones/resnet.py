"""Reference-layout parameter containers for the ResNet / ResNet-IBN-A trunks.

These modules exist so that `state_dict()` keys, shapes and the optimizer's named_parameters
are IDENTICAL to modelling/backbones/resnet.py:90-120 (Bottleneck or BasicBlock) and
resnet_ibn_a.py:77-124 of the reference (checkpoints load unchanged).  They carry no arithmetic: the forward pass is the
H100 engine (engine.py, engine_train.py); the layer graph is described by the C handles they
drive (csrc/trunk.cu, csrc/trunk_train.cu), not here.
"""
from __future__ import annotations

import math

import torch
from torch import nn


def _conv(cin, cout, k, stride=1):
    return nn.Conv2d(cin, cout, kernel_size=k, stride=stride, padding=k // 2 if k == 3 else (3 if k == 7 else 0), bias=False)


class IBN(nn.Module):
    """resnet_ibn_a.py:18-26: InstanceNorm2d(affine) on the first half, BatchNorm2d on the rest."""

    def __init__(self, planes):
        super().__init__()
        self.half = int(planes / 2)
        self.IN = nn.InstanceNorm2d(self.half, affine=True)
        self.BN = nn.BatchNorm2d(planes - self.half)


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None, ibn=False):
        super().__init__()
        self.conv1 = _conv(inplanes, planes, 1)
        self.bn1 = IBN(planes) if ibn else nn.BatchNorm2d(planes)
        self.conv2 = _conv(planes, planes, 3, stride)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = _conv(planes, planes * 4, 1)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.downsample = downsample
        self.stride = stride


class BasicBlock(nn.Module):
    """resnet.py:19-48: two 3x3 convolutions (the first one strided)."""

    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = _conv(inplanes, planes, 3, stride)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = _conv(planes, planes, 3)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = downsample
        self.stride = stride


class ResNetParams(nn.Module):
    """Parameter tree of ResNet(last_stride, Bottleneck | BasicBlock, layers) / ResNet_IBN(...).
    `block` is "bottleneck" or "basic"; IBN-a exists for bottlenecks only."""

    def __init__(self, last_stride=1, layers=(3, 4, 6, 3), ibn=False, block="bottleneck"):
        super().__init__()
        if block not in ("bottleneck", "basic"):
            raise ValueError(f"block={block!r}: expected 'bottleneck' or 'basic'")
        if ibn and block != "bottleneck":
            raise ValueError("IBN-a is defined for bottleneck blocks only (resnet_ibn_a.py)")
        self.ibn = ibn
        self.block = block
        self.layers_cfg = tuple(layers)
        self.last_stride = last_stride
        self.inplanes = 64
        self.conv1 = _conv(3, 64, 7, 2)
        self.bn1 = nn.BatchNorm2d(64)
        self.layer1 = self._make_layer(64, layers[0], 1)
        self.layer2 = self._make_layer(128, layers[1], 2)
        self.layer3 = self._make_layer(256, layers[2], 2)
        self.layer4 = self._make_layer(512, layers[3], last_stride)
        if ibn:  # resnet_ibn_a.py:92-93 carries an unused classifier; kept for state_dict parity
            self.fc = nn.Linear(2048, 1000)
        self.random_init()

    def _make_layer(self, planes, blocks, stride):
        if self.block == "basic":  # resnet.py:103-120 with expansion 1
            down = None
            if stride != 1 or self.inplanes != planes:
                down = nn.Sequential(_conv(self.inplanes, planes, 1, stride), nn.BatchNorm2d(planes))
            mods = [BasicBlock(self.inplanes, planes, stride, down)]
            self.inplanes = planes
            mods += [BasicBlock(planes, planes) for _ in range(1, blocks)]
            return nn.Sequential(*mods)
        down = None
        if stride != 1 or self.inplanes != planes * 4:
            down = nn.Sequential(_conv(self.inplanes, planes * 4, 1, stride), nn.BatchNorm2d(planes * 4))
        use_ibn = self.ibn and planes != 512
        mods = [Bottleneck(self.inplanes, planes, stride, down, use_ibn)]
        self.inplanes = planes * 4
        for _ in range(1, blocks):
            mods.append(Bottleneck(self.inplanes, planes, ibn=use_ibn))
        return nn.Sequential(*mods)

    def random_init(self):
        """resnet.py:156-164 / resnet_ibn_a.py:95-105."""
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2.0 / n))
            elif isinstance(m, (nn.BatchNorm2d, nn.InstanceNorm2d)):
                m.weight.data.fill_(1)
                m.bias.data.zero_()

    def load_param(self, model_path):
        """resnet.py:135-154: strips `backbone.base.` / `base.` prefixes, skips classifier heads."""
        param_dict = torch.load(model_path, map_location="cpu")
        if "state_dict" in param_dict:
            param_dict = param_dict["state_dict"]
        own = self.state_dict()
        for name, val in param_dict.items():
            if any(t in name for t in ("fc", "bottleneck", "classifier", "transformer", "reduce_embeddings.weight")):
                continue
            if "backbone" in name:
                key = name[14:]
            elif "base" in name:
                key = name[5:]
            else:
                key = name
            own[key].copy_(val)
