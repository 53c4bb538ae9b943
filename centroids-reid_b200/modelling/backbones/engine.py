"""H100 inference engine of the ResNet trunks: bottleneck (ResNet50/101/152, -IBN-A) and BasicBlock (ResNet18/34).

TrunkEngine is the ctypes form of the ctl_trunk handle (csrc/trunk.cu, the C ABI a non-Python host binds): the handle
packs a reference-layout state_dict (keys of modelling/backbones/resnet.py:90-120 / resnet_ibn_a.py:77-124) into kernel
operands -- NHWC / [Cout][kh][kw][Cin] fp16 weights with the eval-mode BatchNorm folded in, fp32 biases -- and walks the
layer graph as a sequence of fused conv+BN(+residual)(+ReLU) wgmma launches (csrc/conv.cu).

Forward semantics follow ResNet.forward (resnet.py:122-133: NO ReLU after the stem) and
ResNet_IBN.forward (resnet_ibn_a.py:126-141: ReLU after the stem; IBN as bn1 of layer1-3),
Baseline.forward (baseline.py:91-96: global average pool) and the eval embedding
bn(backbone(x)) of modelling/bases.py:169-177.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from ... import _native as N

R50_LAYERS = (3, 4, 6, 3)
BLOCKS = {"bottleneck": N.CTL_BLOCK_BOTTLENECK, "basic": N.CTL_BLOCK_BASIC}


def pack_stem_fused(w_folded: torch.Tensor) -> torch.Tensor:
    """[64, 3, 7, 7] folded stem weights -> the fused stem's operand [28][64][8] fp16 (include/ctl_b200.h,
    ctl_stem_pool_fused): chunk c = r * 4 + s // 2, element e = (s % 2) * 4 + ch; ch == 3 and s == 7 are zero."""
    wk = torch.zeros(64, 7, 8, 4, device=w_folded.device)            # [o][r][s][ch]
    wk[:, :, :7, :3] = w_folded.float().permute(0, 2, 3, 1)
    return wk.reshape(64, 28, 8).permute(1, 0, 2).contiguous().half()  # [c = r*4 + s//2][o][e = (s%2)*4 + ch]


class TrunkEngine:
    """Packed weights + forward.  `state` is the `base.*`-stripped trunk state_dict on any
    device; `bn_head` optionally the BatchNorm1d(feature_dim) of ModelBase (bases.py:83) for `embed`.  `block` is
    "bottleneck" (feature_dim 2048) or "basic" (ResNet18/34, feature_dim 512)."""

    def __init__(self, state: Dict[str, torch.Tensor], device, ibn: bool = False, last_stride: int = 1,
                 layers=R50_LAYERS, bn_head: Optional[Dict[str, torch.Tensor]] = None, block: str = "bottleneck"):
        if block not in BLOCKS:
            raise ValueError(f"block={block!r}: expected one of {sorted(BLOCKS)}")
        self.device = torch.device(device)
        self.ibn, self.last_stride, self.block = ibn, last_stride, block
        self.launches_per_forward = 0  # kernels launched by the last forward / forward_u8
        self._h = C.c_void_p()
        N.check(N.lib().ctl_trunk_create(C.byref(self._h), BLOCKS[block], int(ibn), int(last_stride),
                                         (C.c_int32 * 4)(*layers)))
        self.feature_dim = N.lib().ctl_trunk_feature_dim(self._h)
        self.pack(state, bn_head)

    def pack(self, state: Dict[str, torch.Tensor], bn_head: Optional[Dict[str, torch.Tensor]] = None):
        """(Re-)folds the parameters into the handle's operands, e.g. after they changed."""
        tensors = {k: v.detach().to(self.device, torch.float32).contiguous() for k, v in state.items() if v.is_floating_point()}
        if bn_head is not None:
            for k in ("weight", "bias", "running_mean", "running_var"):
                tensors["bn_head." + k] = bn_head[k].detach().to(self.device, torch.float32).contiguous()
        arr = (N.NamedTensor * len(tensors))()
        for i, (k, v) in enumerate(tensors.items()):
            arr[i].name, arr[i].data, arr[i].numel = k.encode(), v.data_ptr(), v.numel()
        with torch.cuda.device(self.device):
            N.check(N.lib().ctl_weights_pack(self._h, arr, len(tensors), N.stream_ptr()))
            torch.cuda.current_stream().synchronize()  # the fp32 sources may be freed once the pack kernels have run
        self.has_head = bn_head is not None

    def _workspace(self, n, H, W):
        # per call, like every activation: eager calls reuse the caching allocator's blocks in stream order, and a
        # captured graph keeps its own
        return torch.empty(N.lib().ctl_embed_workspace_bytes(self._h, n, H, W), dtype=torch.uint8, device=self.device)

    def _launched(self):
        return N.lib().ctl_embed_launches(self._h)

    def forward(self, x: torch.Tensor, want_base: bool = False, want_emb: bool = False):
        """x: [B, 3, H, W] fp32 NCHW on the device -> dict(global_feat [B, C] fp32,
        base_out NHWC fp16 (if want_base), emb (if want_emb and a head was given))."""
        N.require_cuda(x)
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"expected [B, 3, H, W], got {tuple(x.shape)}")
        x = x.float().contiguous()
        with torch.cuda.device(self.device):
            return self._run(self.stem(x), want_base, want_emb)

    def forward_u8(self, images_u8: torch.Tensor, want_base: bool = False, want_emb: bool = False,
                   pixel_mean=(0.485, 0.456, 0.406), pixel_std=(0.229, 0.224, 0.225)):
        """images_u8: [B, H, W, 3] uint8 crops on the device (what a validation loader ships after `T.Resize`) -> the same
        dict as forward(normalize_batch(images_u8)), bit for bit: ToTensor + Normalize (datasets/transforms/build.py:29-33)
        are folded into the fused stem's input packing, the fp32 NCHW tensor is never written.  Shapes the fused stem does
        not take (W > 128, H % 4 != 0) go through normalize_batch."""
        N.require_cuda(images_u8)
        if images_u8.dim() != 4 or images_u8.shape[3] != 3 or images_u8.dtype != torch.uint8:
            raise ValueError(f"expected uint8 [B, H, W, 3], got {images_u8.dtype} {tuple(images_u8.shape)}")
        n, H, W, _ = images_u8.shape
        if not (H % 4 == 0 and W % 2 == 0 and W <= 128):
            from ...datasets.transforms import normalize_batch

            return self.forward(normalize_batch(images_u8, pixel_mean, pixel_std), want_base, want_emb)
        images_u8 = images_u8.contiguous()
        with torch.cuda.device(self.device):
            return self._run(self.stem(images_u8, u8_norm=(pixel_mean, pixel_std)), want_base, want_emb)

    def _run(self, stem_out, want_base, want_emb):
        a, n, h, w = stem_out
        launches = self._launched()
        a, h, w = self.bottlenecks(a, n, h, w)
        launches += self._launched()
        out = self.tail(a, n, h, w, want_base, want_emb)
        self.launches_per_forward = launches + self._launched()
        return out

    # The three segments of the forward (bench.py captures each as its own CUDA graph to attribute the graph-mode step
    # time to the convolution kernels without leaving graph / PDL mode).
    def stem(self, x: torch.Tensor, u8_norm=None):
        """conv1 7x7/2 + bn1 (+ReLU for IBN-a) + maxpool 3x3/2 -> NHWC fp16 [n, hp, wp, 64].  `u8_norm` = (mean, std):
        x is a uint8 [n, H, W, 3] batch, normalised inside the fused stem's packing kernel (forward_u8)."""
        if u8_norm is not None:
            n, H, W, _ = x.shape
            mean = (C.c_float * 3)(*[float(v) for v in u8_norm[0]])
            std = (C.c_float * 3)(*[float(v) for v in u8_norm[1]])
        else:
            n, _, H, W = x.shape
            mean = std = None
        h, w = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
        hp, wp = (h + 2 - 3) // 2 + 1, (w + 2 - 3) // 2 + 1
        a = torch.empty(n, hp, wp, 64, dtype=torch.float16, device=self.device)
        ws = self._workspace(n, H, W)
        N.check(N.lib().ctl_embed_stem(self._h, x.data_ptr(), n, H, W, mean, std, a.data_ptr(), ws.data_ptr(), ws.numel(),
                                       N.stream_ptr()))
        return a, n, hp, wp

    def bottlenecks(self, a, n, h, w):
        """[n, h, w, 64] stem output -> [n, h', w', feature_dim] trunk output; `a` is only read."""
        ho, wo = h, w
        for s in (2, 2, self.last_stride):  # first blocks of layer2, layer3, layer4: 3x3 / s, pad 1
            ho, wo = (ho + 2 - 3) // s + 1, (wo + 2 - 3) // s + 1
        out = torch.empty(n, ho, wo, self.feature_dim, dtype=torch.float16, device=self.device)
        ws = self._workspace(n, 4 * h, 4 * w)  # a 4h x 4w image has this stem output and no larger stem temporary
        N.check(N.lib().ctl_embed_blocks(self._h, a.data_ptr(), n, h, w, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                         N.stream_ptr()))
        return out, ho, wo

    def tail(self, a, n, h, w, want_base=False, want_emb=False):
        """global average pool (+ the folded eval BatchNorm1d head)."""
        feat = torch.empty(n, self.feature_dim, dtype=torch.float32, device=self.device)
        emb = torch.empty(n, self.feature_dim, dtype=torch.float32, device=self.device) if (want_emb and self.has_head) else None
        N.check(N.lib().ctl_embed_head(self._h, a.data_ptr(), n, h * w, feat.data_ptr(), N.ptr(emb), N.stream_ptr()))
        out = {"global_feat": feat}
        if want_base:
            out["base_out_nhwc"] = a
        if emb is not None:
            out["emb"] = emb
        return out

    def __del__(self):
        try:
            if self._h:
                N.lib().ctl_trunk_destroy(self._h)
                self._h = None
        except Exception:  # noqa: BLE001 - interpreter shutdown
            pass


class GraphedCall:
    """A CUDA graph of any launch sequence `fn()` on static buffers (two eager warm-ups on a side stream, then capture)."""

    def __init__(self, fn, device):
        cur = torch.cuda.current_stream(device)
        side = torch.cuda.Stream(device=device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            for _ in range(2):
                fn()
        cur.wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = fn()

    def __call__(self):
        self.graph.replay()
        return self.out


class GraphedForward:
    """One CUDA graph of TrunkEngine.forward on a fixed input buffer: its launches (45 for ResNet50 at 256x128) replayed
    with a single cudaGraphLaunch (no per-launch host work, no tensor-map re-encoding).  `x` is read in
    place at every replay; outputs are static tensors overwritten by each replay."""

    def __init__(self, engine: "TrunkEngine", x: torch.Tensor, want_emb: bool = True):
        self.engine, self.x = engine, x
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream(device=x.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):  # warm-up outside capture (function attributes, allocator pools)
            for _ in range(2):
                engine.forward(x, want_emb=want_emb)
        cur.wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = engine.forward(x, want_emb=want_emb)
        self.launches = engine.launches_per_forward

    def __call__(self):
        self.graph.replay()
        return self.out
