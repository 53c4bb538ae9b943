"""H100 inference engine of the ResNet50(-IBN-A) trunk.

Packs a reference-layout state_dict (keys of modelling/backbones/resnet.py:90-120 /
resnet_ibn_a.py:77-124) into kernel operands -- NHWC / [Cout][kh][kw][Cin] fp16 weights with the
eval-mode BatchNorm folded in, fp32 biases -- and runs the forward as a sequence of fused
conv+BN(+residual)(+ReLU) wgmma launches (csrc/conv.cu) through the C ABI.

Forward semantics follow ResNet.forward (resnet.py:122-133: NO ReLU after the stem) and
ResNet_IBN.forward (resnet_ibn_a.py:126-141: ReLU after the stem; IBN as bn1 of layer1-3),
Baseline.forward (baseline.py:91-96: global average pool) and the eval embedding
bn(backbone(x)) of modelling/bases.py:169-177.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from ... import _native as N

R50_LAYERS = (3, 4, 6, 3)
BN_EPS = 1e-5


def _fold(w: torch.Tensor, bn: Dict[str, torch.Tensor], eps: float = BN_EPS):
    scale = bn["weight"].float() / torch.sqrt(bn["running_var"].float() + eps)
    bias = bn["bias"].float() - bn["running_mean"].float() * scale
    return w.float() * scale[:, None, None, None], bias


def _bn(sd, prefix):
    return {k: sd[f"{prefix}.{k}"] for k in ("weight", "bias", "running_mean", "running_var")}


class _Conv:
    __slots__ = ("w", "b", "cin", "cout", "k", "stride", "relu", "relu_from")

    def __init__(self, w_folded, bias, stride, relu, relu_from=0):
        cout, cin, k, _ = w_folded.shape
        self.w = w_folded.permute(0, 2, 3, 1).contiguous().half()  # [Cout][kh][kw][Cin]
        self.b = bias.float().contiguous()
        self.cin, self.cout, self.k, self.stride, self.relu, self.relu_from = cin, cout, k, stride, relu, relu_from


def pack_stem_fused(w_folded: torch.Tensor) -> torch.Tensor:
    """[64, 3, 7, 7] folded stem weights -> the fused stem's operand [28][64][8] fp16 (include/ctl_b200.h,
    ctl_stem_pool_fused): chunk c = r * 4 + s // 2, element e = (s % 2) * 4 + ch; ch == 3 and s == 7 are zero."""
    wk = torch.zeros(64, 7, 8, 4, device=w_folded.device)            # [o][r][s][ch]
    wk[:, :, :7, :3] = w_folded.float().permute(0, 2, 3, 1)
    return wk.reshape(64, 28, 8).permute(1, 0, 2).contiguous().half()  # [c = r*4 + s//2][o][e = (s%2)*4 + ch]


class TrunkEngine:
    """Packed weights + forward.  `state` is the `base.*`-stripped trunk state_dict on any
    device; `bn_head` optionally the BatchNorm1d(2048) of ModelBase (bases.py:83) for `embed`."""

    def __init__(self, state: Dict[str, torch.Tensor], device, ibn: bool = False, last_stride: int = 1,
                 layers=R50_LAYERS, bn_head: Optional[Dict[str, torch.Tensor]] = None):
        self.device = torch.device(device)
        self.ibn = ibn
        sd = {k: v.detach().to(self.device) for k, v in state.items() if v.is_floating_point()}
        w, b = _fold(sd["conv1.weight"], _bn(sd, "bn1"))
        # stem weights for the tensor-core stem: [64][192] fp16, k = (c*7 + r)*8 + s; s = 7 and k >= 168 zero
        wk = torch.zeros(64, 21, 8, device=self.device)
        wk[:, :, :7] = w.reshape(64, 21, 7)
        self.stem_w = torch.cat((wk.reshape(64, 168), torch.zeros(64, 24, device=self.device)), 1).half().contiguous()
        self.stem_b = b.contiguous()
        self.stem_w3 = pack_stem_fused(w)
        self._stem_pad = {}  # (n, H, W) -> zero-bordered NHWC4 staging buffer of the fused stem
        self.blocks = []
        for li, (planes, nblk) in enumerate(zip((64, 128, 256, 512), layers), start=1):
            stride0 = 1 if li == 1 else (last_stride if li == 4 else 2)
            for bi in range(nblk):
                p = f"layer{li}.{bi}"
                stride = stride0 if bi == 0 else 1
                blk = {}
                if ibn and planes != 512:  # resnet_ibn_a.py:116-119
                    half = planes // 2
                    wbn, bbn = _fold(sd[p + ".conv1.weight"][half:], _bn(sd, p + ".bn1.BN"))
                    w1 = torch.cat((sd[p + ".conv1.weight"][:half].float(), wbn), 0)
                    b1 = torch.cat((torch.zeros(half, device=self.device), bbn), 0)
                    blk["conv1"] = _Conv(w1, b1, 1, True, relu_from=half)
                    blk["in"] = (half, sd[p + ".bn1.IN.weight"].float().contiguous(),
                                 sd[p + ".bn1.IN.bias"].float().contiguous())
                else:
                    blk["conv1"] = _Conv(*_fold(sd[p + ".conv1.weight"], _bn(sd, p + ".bn1")), 1, True)
                blk["conv2"] = _Conv(*_fold(sd[p + ".conv2.weight"], _bn(sd, p + ".bn2")), stride, True)
                blk["conv3"] = _Conv(*_fold(sd[p + ".conv3.weight"], _bn(sd, p + ".bn3")), 1, True)
                if bi == 0:
                    blk["down"] = _Conv(*_fold(sd[p + ".downsample.0.weight"], _bn(sd, p + ".downsample.1")),
                                        stride, False)
                    # conv3 + shortcut as ONE GEMM over the concatenated K dimension (ctl_conv1x1_dual_nhwc_f16):
                    # [W3 | Wd] fp16 (each folded matrix rounded exactly as in the two-launch form), bias3 + bias_d
                    c3, cd = blk["conv3"], blk["down"]
                    blk["dual_w"] = torch.cat((c3.w.reshape(c3.cout, c3.cin), cd.w.reshape(cd.cout, cd.cin)), 1).contiguous()
                    blk["dual_b"] = (c3.b + cd.b).contiguous()
                self.blocks.append(blk)
        self.out_channels = self.blocks[-1]["conv3"].cout
        self.profile = None  # set to a list to record (kernel, flops, bytes, start_evt, end_evt) per launch
        self.launches_per_forward = 0
        self.head = None
        if bn_head is not None:
            # folded on the DEVICE like the trunk's BatchNorms (fp32 add / sqrt / div / mul / sub, each correctly rounded):
            # torch's vectorised CPU kernels round some of these differently, and the C-ABI pack (csrc/trunk.cu) must
            # produce the same bits
            hb = {k: bn_head[k].detach().to(self.device, torch.float32) for k in ("weight", "bias", "running_mean", "running_var")}
            scale = hb["weight"] / torch.sqrt(hb["running_var"] + BN_EPS)
            shift = hb["bias"] - hb["running_mean"] * scale
            self.head = (scale.contiguous(), shift.contiguous())

    # -- single ops --------------------------------------------------------------------------
    def _conv(self, x, n, h, w, c: _Conv, residual=None):
        pad = 1 if c.k == 3 else 0
        ho, wo = (h + 2 * pad - c.k) // c.stride + 1, (w + 2 * pad - c.k) // c.stride + 1
        out = torch.empty(n, ho, wo, c.cout, dtype=torch.float16, device=self.device)
        m = n * ho * wo
        flops = 2.0 * m * c.cout * c.cin * c.k * c.k
        # algorithmic bytes: input read once (a strided 1x1 only touches its sampled pixels), output
        # written once, residual read once, weights once -- fp16
        in_px = m if (c.k == 1) else n * h * w
        nbytes = 2.0 * (in_px * c.cin + m * c.cout * (2 if residual is not None else 1) + c.cout * c.cin * c.k * c.k)
        with self._timed("conv_gemm", flops, nbytes):
            N.check(N.lib().ctl_conv2d_nhwc_f16(x.data_ptr(), n, h, w, c.cin, c.w.data_ptr(), c.b.data_ptr(),
                                                N.ptr(residual), out.data_ptr(), c.cout, c.k, c.stride, int(c.relu),
                                                c.relu_from, N.stream_ptr()))
        return out, ho, wo

    def _dual(self, o2, a, n, h, w, h2, w2, blk):
        """relu(bn3(conv3(o2)) + bn_d(downsample(a))) in one launch; the shortcut tensor never exists."""
        c3, cd = blk["conv3"], blk["down"]
        out = torch.empty(n, h2, w2, c3.cout, dtype=torch.float16, device=self.device)
        m = n * h2 * w2
        flops = 2.0 * m * c3.cout * (c3.cin + cd.cin)
        nbytes = 2.0 * (m * (c3.cin + cd.cin) + m * c3.cout + c3.cout * (c3.cin + cd.cin))
        with self._timed("conv_gemm", flops, nbytes):
            N.check(N.lib().ctl_conv1x1_dual_nhwc_f16(o2.data_ptr(), c3.cin, a.data_ptr(), h, w, cd.cin, cd.stride, n,
                                                      blk["dual_w"].data_ptr(), blk["dual_b"].data_ptr(),
                                                      out.data_ptr(), c3.cout, 1, N.stream_ptr()))
        return out, h2, w2

    def _timed(self, name, flops=0.0, nbytes=0.0):
        return _Timed(self, name, flops, nbytes)

    def forward(self, x: torch.Tensor, want_base: bool = False, want_emb: bool = False):
        """x: [B, 3, H, W] fp32 NCHW on the device -> dict(global_feat [B, C] fp32,
        base_out NHWC fp16 (if want_base), emb (if want_emb and a head was given))."""
        N.require_cuda(x)
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"expected [B, 3, H, W], got {tuple(x.shape)}")
        x = x.float().contiguous()
        self.launches_per_forward = 0
        with torch.cuda.device(self.device):
            a, n, h, w = self.stem(x)
            a, h, w = self.bottlenecks(a, n, h, w)
            return self.tail(a, n, h, w, want_base, want_emb)

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
        self.launches_per_forward = 0
        with torch.cuda.device(self.device):
            a, n, h, w = self.stem(images_u8, u8_norm=(pixel_mean, pixel_std))
            a, h, w = self.bottlenecks(a, n, h, w)
            return self.tail(a, n, h, w, want_base, want_emb)

    # The three segments of the forward (bench.py captures each as its own CUDA graph to attribute the graph-mode step
    # time to the convolution kernels without leaving graph / PDL mode).
    def stem(self, x: torch.Tensor, u8_norm=None):
        """conv1 7x7/2 + bn1 (+ReLU for IBN-a) + maxpool 3x3/2 -> NHWC fp16 [n, hp, wp, 64].  `u8_norm` = (mean, std):
        x is a uint8 [n, H, W, 3] batch, normalised inside the fused stem's packing kernel (forward_u8)."""
        if u8_norm is not None:
            n, H, W, _ = x.shape
        else:
            n, _, H, W = x.shape
        L = N.lib()
        h, w = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
        hp, wp = (h + 2 - 3) // 2 + 1, (w + 2 - 3) // 2 + 1
        a = torch.empty(n, hp, wp, 64, dtype=torch.float16, device=self.device)
        if H % 4 == 0 and W % 2 == 0 and W <= 128:
            # conv1 + bn1 (+ReLU) + maxpool in one pass; only the pooled tensor is written
            pad = self._stem_pad.get((n, H, W))
            if pad is None:
                pad = torch.zeros(L.ctl_stem_pad_bytes(n, H, W), dtype=torch.uint8, device=self.device)
                self._stem_pad[(n, H, W)] = pad
            with self._timed("stem_pool", 2.0 * n * h * w * 64 * 147, n * (3.0 * H * W * 4 + hp * wp * 64 * 2)):
                if u8_norm is not None:
                    import ctypes as C

                    mean = (C.c_float * 3)(*[float(v) for v in u8_norm[0]])
                    std = (C.c_float * 3)(*[float(v) for v in u8_norm[1]])
                    N.check(L.ctl_stem_pool_fused_u8(x.data_ptr(), n, H, W, mean, std, pad.data_ptr(), self.stem_w3.data_ptr(),
                                                     self.stem_b.data_ptr(), int(self.ibn), a.data_ptr(), N.stream_ptr()))
                else:
                    N.check(L.ctl_stem_pool_fused(x.data_ptr(), n, H, W, pad.data_ptr(), self.stem_w3.data_ptr(),
                                                  self.stem_b.data_ptr(), int(self.ibn), a.data_ptr(), N.stream_ptr()))
            self.launches_per_forward += 1  # pack + conv/pool kernels
        else:
            s = torch.empty(n, h, w, 64, dtype=torch.float16, device=self.device)
            with self._timed("stem_conv", 2.0 * n * h * w * 64 * 147, n * (3.0 * H * W * 4 + h * w * 64 * 2)):
                N.check(L.ctl_stem_conv7x7_tc(x.data_ptr(), n, H, W, self.stem_w.data_ptr(), self.stem_b.data_ptr(),
                                              int(self.ibn), s.data_ptr(), N.stream_ptr()))
            with self._timed("maxpool", 0.0, n * 64 * 2.0 * (h * w + hp * wp)):
                N.check(L.ctl_maxpool3x3s2_nhwc_f16(s.data_ptr(), n, h, w, 64, a.data_ptr(), N.stream_ptr()))
        return a, n, hp, wp

    def _chain(self, o2, a, res, n, h, w, h2, w2, blk, nxt: _Conv):
        """The block's last convolution (dual form when `res` is None and the block has a shortcut branch, else conv3 +
        residual) and the next block's conv1 in one launch (ctl_conv1x1_chain_nhwc_f16) -> (out, next conv1 output)."""
        c3 = blk["conv3"]
        dual = res is None and "down" in blk
        out = torch.empty(n, h2, w2, c3.cout, dtype=torch.float16, device=self.device)
        o1 = torch.empty(n, h2, w2, nxt.cout, dtype=torch.float16, device=self.device)
        m = n * h2 * w2
        k1 = c3.cin + (blk["down"].cin if dual else 0)
        flops = 2.0 * m * c3.cout * k1 + 2.0 * m * nxt.cout * nxt.cin
        # the block output is written once and never re-read; the next conv1's output is written once
        nbytes = 2.0 * (m * k1 + m * c3.cout * (1 if dual else 2) + c3.cout * k1 + m * nxt.cout + nxt.cout * nxt.cin)
        L = N.lib()
        with self._timed("conv_chain", flops, nbytes):
            if dual:
                cd = blk["down"]
                rc = L.ctl_conv1x1_chain_nhwc_f16(o2.data_ptr(), c3.cin, a.data_ptr(), h, w, cd.cin, cd.stride, n,
                                                  blk["dual_w"].data_ptr(), blk["dual_b"].data_ptr(), None, out.data_ptr(),
                                                  c3.cout, nxt.w.data_ptr(), nxt.b.data_ptr(), nxt.cout, nxt.relu_from,
                                                  o1.data_ptr(), N.stream_ptr())
            else:
                rc = L.ctl_conv1x1_chain_nhwc_f16(o2.data_ptr(), c3.cin, None, h2, w2, 0, 1, n, c3.w.data_ptr(),
                                                  c3.b.data_ptr(), res.data_ptr(), out.data_ptr(), c3.cout, nxt.w.data_ptr(),
                                                  nxt.b.data_ptr(), nxt.cout, nxt.relu_from, o1.data_ptr(), N.stream_ptr())
            N.check(rc)
        return out, o1

    def bottlenecks(self, a, n, h, w):
        L = N.lib()
        o1 = None  # the block's conv1 output when the previous block's last launch computed it
        for i, blk in enumerate(self.blocks):
            if o1 is None:
                o1, h1, w1 = self._conv(a, n, h, w, blk["conv1"])
            else:
                h1, w1 = h, w
            if "in" in blk:
                half, g, b = blk["in"]
                with self._timed("instnorm_relu", 0.0, 2.0 * 2 * n * h1 * w1 * half):
                    N.check(L.ctl_instnorm_relu_nhwc_f16(o1.data_ptr(), n, h1 * w1, blk["conv1"].cout, half,
                                                         g.data_ptr(), b.data_ptr(), BN_EPS, N.stream_ptr()))
            o2, h2, w2 = self._conv(o1, n, h1, w1, blk["conv2"])
            dual = "down" in blk and h % blk["down"].stride == 0 and w % blk["down"].stride == 0
            res = None if dual else a
            if "down" in blk and not dual:
                res, _, _ = self._conv(a, n, h, w, blk["down"])
            nxt = self.blocks[i + 1]["conv1"] if i + 1 < len(self.blocks) else None
            o1 = None
            if nxt is not None and L.ctl_conv1x1_chain_supported(blk["conv3"].cout, nxt.cout):
                a, o1 = self._chain(o2, a, res, n, h, w, h2, w2, blk, nxt)
            elif dual:
                a, _, _ = self._dual(o2, a, n, h, w, h2, w2, blk)
            else:
                a, _, _ = self._conv(o2, n, h2, w2, blk["conv3"], residual=res)
            h, w = h2, w2
        return a, h, w

    def tail(self, a, n, h, w, want_base=False, want_emb=False):
        """global average pool (+ the folded eval BatchNorm1d head)."""
        c = self.out_channels
        feat = torch.empty(n, c, dtype=torch.float32, device=self.device)
        emb = torch.empty(n, c, dtype=torch.float32, device=self.device) if (want_emb and self.head) else None
        sc, sh = self.head if self.head else (None, None)
        with self._timed("gap_bn", 0.0, n * c * (2.0 * h * w + 8)):
            N.check(N.lib().ctl_gap_bn_nhwc_f16(a.data_ptr(), n, h * w, c, N.ptr(sc), N.ptr(sh), feat.data_ptr(),
                                                N.ptr(emb), N.stream_ptr()))
        out = {"global_feat": feat}
        if want_base:
            out["base_out_nhwc"] = a
        if emb is not None:
            out["emb"] = emb
        return out


class NativeTrunk:
    """The same embedding path with the LAYER GRAPH behind the C ABI (ctl_trunk_create / ctl_weights_pack /
    ctl_embed_forward, csrc/trunk.cu): what a non-Python host binds.  Packs on the device from the fp32 state_dict;
    bit-identical to TrunkEngine (tests/test_trunk_gpu.py::test_native_trunk_handle_matches_engine)."""

    def __init__(self, state: Dict[str, torch.Tensor], device, ibn: bool = False, last_stride: int = 1,
                 bn_head: Optional[Dict[str, torch.Tensor]] = None):
        import ctypes as C

        self.device = torch.device(device)
        self._h = C.c_void_p()
        N.check(N.lib().ctl_trunk_create(C.byref(self._h), int(ibn), int(last_stride)))
        self._ws = None
        self.pack(state, bn_head)

    def pack(self, state, bn_head=None):
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

    def forward(self, x: torch.Tensor, want_emb: bool = False):
        N.require_cuda(x)
        x = x.float().contiguous()
        n, _, H, W = x.shape
        L = N.lib()
        need = L.ctl_embed_workspace_bytes(self._h, n, H, W)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        feat = torch.empty(n, 2048, device=self.device)
        emb = torch.empty(n, 2048, device=self.device) if (want_emb and self.has_head) else None
        with torch.cuda.device(self.device):
            N.check(L.ctl_embed_forward(self._h, x.data_ptr(), n, H, W, feat.data_ptr(), N.ptr(emb), self._ws.data_ptr(),
                                        self._ws.numel(), N.stream_ptr()))
        out = {"global_feat": feat}
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
    """One CUDA graph of TrunkEngine.forward on a fixed input buffer: 51 launches replayed with a
    single cudaGraphLaunch (no per-launch host work, no tensor-map re-encoding).  `x` is read in
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


class _Timed:
    """Counts launches; in profile mode brackets the launch with CUDA events on the current
    stream (the stream the kernel is enqueued on)."""

    def __init__(self, eng, name, flops, nbytes):
        self.eng, self.name, self.flops, self.nbytes = eng, name, flops, nbytes

    def __enter__(self):
        self.eng.launches_per_forward += 1
        if self.eng.profile is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if self.eng.profile is not None:
            self.e1.record()
            self.eng.profile.append((self.name, self.flops, self.nbytes, self.e0, self.e1))
        return False
