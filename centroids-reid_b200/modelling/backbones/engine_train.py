"""Train-mode ResNet trunk (bottleneck or BasicBlock) on the H100 kernels: forward with batch-statistics BatchNorm and the full backward
(what autograd does through modelling/backbones/resnet.py:67-87,122-133 + baseline.py:91-96 in the reference).

The layer walk is the ctl_trainer handle's (csrc/trunk_train.cu, the C ABI a non-Python host binds): per conv+BN of
the forward, conv (wgmma implicit GEMM, raw fp16 output y) -> batch statistics -> z = [relu](gamma * xhat + beta
[+ shortcut]) (fp16); the backward walks the blocks in reverse (BN/ReLU backward, weight gradient, data gradient
through the transposed convolution, shortcut gradients folded into conv1's data gradient).  Activations and
activation gradients are fp16, every reduction and all parameter gradients fp32.  TrunkTrainer binds the parameters,
owns the workspace and the gradient buffers, and can replay both passes from CUDA graphs.

Gradients are computed on `grad_scale * dfeat` (a fixed loss scale against fp16 underflow, the role of the AMP
GradScaler in the reference's PL trainer) and un-scaled in fp32.  `ibn=True` runs the IBN-a variant
(resnet_ibn_a.py): ReLU after the stem, and bn1 of layer1-3 = InstanceNorm on the first half of the channels
(per-image statistics) + batch-statistics BatchNorm on the rest, both through channel-slice (row pitch) kernels.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Tuple

import torch

from ... import _native as N
from .engine import BLOCKS, R50_LAYERS


def _named(tensors: Dict[str, torch.Tensor]):
    arr = (N.NamedTensor * len(tensors))()  # ctl_named_buffer has the same layout (writable data pointer)
    for i, (k, v) in enumerate(tensors.items()):
        arr[i].name, arr[i].data, arr[i].numel = k.encode(), v.data_ptr(), v.numel()
    return arr


class TrunkTrainer:
    """`params`: name -> tensor with the reference's `base.*`-stripped names (conv weights [Cout, Cin, k, k], BN
    weight / bias fp32 on the device; BN running_mean / running_var are updated in place).  `block` is "bottleneck"
    (feature_dim 2048) or "basic" (ResNet18/34, feature_dim 512)."""

    def __init__(self, device, last_stride: int = 1, layers=R50_LAYERS, grad_scale: float = 1024.0,
                 momentum: float = 0.1, graphs: bool = False, ibn: bool = False, block: str = "bottleneck"):
        if block not in BLOCKS:
            raise ValueError(f"block={block!r}: expected one of {sorted(BLOCKS)}")
        self.device = torch.device(device)
        self.ibn = ibn  # resnet_ibn_a.py: ReLU after the stem, IBN (InstanceNorm half + BatchNorm half) as bn1 of layer1-3
        self.block = block
        self.last_stride, self.layers, self.grad_scale, self.momentum = last_stride, tuple(layers), float(grad_scale), momentum
        self._h = C.c_void_p()
        N.check(N.lib().ctl_trainer_create(C.byref(self._h), BLOCKS[block], int(ibn), int(last_stride), float(momentum),
                                           (C.c_int32 * 4)(*self.layers)))
        self.feature_dim = N.lib().ctl_trainer_feature_dim(self._h)
        self._bound = None  # (name, data_ptr) of the bound parameters
        self._ws = None
        self._x = None  # the backward's stem im2col reads the input again
        # graphs=True: forward and backward are captured once per (input shape, parameter storage) into two CUDA
        # graphs and replayed (the ~540 launches of a step cost more CPU time than the GPU needs to run them)
        self.graphs = graphs
        self._graph = None

    def _bind(self, params: Dict[str, torch.Tensor]):
        # the trunk's own tensors only (resnet_ibn_a.py keeps an unused ImageNet `fc` in its state_dict)
        params = {k: v for k, v in params.items() if v.is_floating_point() and not k.startswith("fc.")}
        key = tuple((k, v.data_ptr()) for k, v in params.items())
        if key == self._bound:
            return
        dev = torch.device("cuda", torch.cuda.current_device() if self.device.index is None else self.device.index)
        for k, v in params.items():
            if v.dtype != torch.float32 or not v.is_contiguous() or v.device != dev:
                raise TypeError(f"{k} must be a contiguous fp32 tensor on {dev}")
        self._bound = None
        self._params = params
        self.grads = {k: torch.empty_like(v) for k, v in params.items() if "running" not in k}
        with torch.cuda.device(self.device):  # a synchronous copy of the pack table: never inside a capture
            N.check(N.lib().ctl_trainer_bind(self._h, _named(params), len(params), _named(self.grads), len(self.grads)))
        self._bound = key

    def _workspace(self, n, H, W):
        need = N.lib().ctl_train_workspace_bytes(self._h, n, H, W)
        if need == 0:
            raise ValueError(f"unsupported input shape {(n, 3, H, W)}")
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)

    def _forward(self, x: torch.Tensor) -> torch.Tensor:
        self._x = x.float().contiguous()
        n, _, H, W = self._x.shape
        self._workspace(n, H, W)
        feat = torch.empty(n, self.feature_dim, device=self.device)
        with torch.cuda.device(self.device):
            N.check(N.lib().ctl_train_forward(self._h, self._x.data_ptr(), n, H, W, feat.data_ptr(), self._ws.data_ptr(),
                                              self._ws.numel(), N.stream_ptr()))
        return feat

    def _backward(self, dfeat: torch.Tensor) -> Dict[str, torch.Tensor]:
        dfeat = dfeat.float().contiguous()
        with torch.cuda.device(self.device):
            N.check(N.lib().ctl_train_backward(self._h, dfeat.data_ptr(), self.grad_scale, N.ptr(self._ws),
                                               0 if self._ws is None else self._ws.numel(), N.stream_ptr()))
        return self.grads

    def forward(self, x: torch.Tensor, params: Dict[str, torch.Tensor]) -> torch.Tensor:
        """x: [B, 3, H, W] fp32 NCHW on the device -> global_feat [B, feature_dim] fp32; keeps what backward needs."""
        N.require_cuda(x)
        if not self.graphs:
            self._bind(params)
            return self._forward(x)
        key = (tuple(x.shape), tuple(sorted((k, v.data_ptr()) for k, v in params.items())))
        g = self._graph
        if g is None or g["key"] != key:  # same key: the same storage is bound already
            self._bind(params)
            g = self._capture(x, key)
        g["x"].copy_(x)
        g["fwd"].replay()
        return g["feat"].clone()

    def backward(self, dfeat: torch.Tensor) -> Dict[str, torch.Tensor]:
        """dfeat: [B, feature_dim] fp32 = dLoss/dglobal_feat -> {param name: fp32 gradient in the reference's layout}.
        Copies: the next backward overwrites the bound gradient buffers, and autograd may keep these as `.grad`."""
        g = self._graph
        if g is None:
            grads = self._backward(dfeat)
        else:
            g["dfeat"].copy_(dfeat)
            g["bwd"].replay()
            grads = self.grads
        return {k: v.clone() for k, v in grads.items()}

    def _capture(self, x, key):
        self._graph = None
        sx = x.detach().float().contiguous().clone()
        n, _, H, W = sx.shape
        self._workspace(n, H, W)  # outside the capture: the graphs keep its address
        running = {k: v.clone() for k, v in self._params.items() if "running" in k}
        sdf = torch.zeros(n, self.feature_dim, device=self.device)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):  # eager warm-up: function attributes, allocator pools
            self._forward(sx)
            self._backward(sdf)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        fwd, bwd = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(fwd):
            feat = self._forward(sx)
        with torch.cuda.graph(bwd, pool=fwd.pool()):
            self._backward(sdf)
        for k, v in running.items():  # the warm-up and capture passes must not count as training steps
            self._params[k].copy_(v)
        self._graph = {"key": key, "x": sx, "dfeat": sdf, "fwd": fwd, "bwd": bwd, "feat": feat}
        return self._graph

    def saved_activations(self) -> List[Tuple[torch.Tensor, torch.Tensor]]:
        """(y, z) of the last forward as NHWC fp16 views into the workspace: the stem's raw conv output and its
        normalised output first, then every conv + BatchNorm in forward order (conv1, conv2, [downsample], conv3 per
        bottleneck; conv1, [downsample], conv2 per BasicBlock) -- the order the oracles' `forced=` takes."""
        y, z, shape = C.c_void_p(), C.c_void_p(), (C.c_int32 * 4)()
        base = N.ptr(self._ws)

        def view(p):
            off = p - base
            numel = shape[0] * shape[1] * shape[2] * shape[3]
            return self._ws[off:off + 2 * numel].view(torch.float16).view(*shape)

        out = []
        if self.block == "basic":  # stem + two convs per block + the downsamples of layer2-4
            count = 1 + 2 * sum(self.layers) + 3
        else:  # stem + three convs per block + one downsample per stage
            count = 1 + 3 * sum(self.layers) + 4
        for i in range(count):
            N.check(N.lib().ctl_train_saved(self._h, i, C.byref(y), C.byref(z), shape))
            out.append((view(y.value), view(z.value)))
        return out

    def __del__(self):
        try:
            if self._h:
                N.lib().ctl_trainer_destroy(self._h)
                self._h = None
        except Exception:  # noqa: BLE001 - interpreter shutdown
            pass
