"""Device-side transforms: the arithmetic of ReidTransforms.build_transforms (datasets/transforms/build.py:15-33) for a
whole batch -- the loaders' JPEG decode (pack_jpegs -> decode_batch, bit for bit Pillow's
`Image.open(p).convert("RGB")`), `T.Resize` of native-size images packed in a RaggedImages (pack_images -> resize_batch,
bit for bit PIL's BILINEAR resize), then the training chain after it in one kernel (augment_batch) or the eval chain
(normalize_batch, or TrunkEngine.forward_u8, which folds it into the stem).  This module alone knows the ragged layout.

The reference draws its random numbers per image inside torchvision / `random` (flip: torch.rand(1) < p;
crop: torch.randint; erasing: random.uniform / random.randint with up to 100 attempts, random_erasing.py:30-55).
`sample_params` draws the same distributions from one numpy Generator (the stream of numbers differs -- the
reference's own stream depends on DataLoader worker scheduling); `augment_batch` is then a deterministic function of
(images, params) and is what the parity test pins against the oracle.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from .. import _native as N


def sample_params(batch: int, h: int, w: int, prob_flip=0.5, pad=10, re_prob=0.5, is_real=None, rng=None,
                  sl=0.02, sh=0.4, r1=0.3) -> np.ndarray:
    """int32 [batch, 8] = {flip, crop_top, crop_left, erase_row, erase_col, erase_h, erase_w, is_real}."""
    rng = rng if rng is not None else np.random.default_rng()
    out = np.zeros((batch, 8), dtype=np.int32)
    out[:, 7] = 1 if is_real is None else np.asarray(is_real, dtype=np.int32)
    for b in range(batch):
        out[b, 0] = rng.random() < prob_flip                       # T.RandomHorizontalFlip
        out[b, 1] = rng.integers(0, 2 * pad + 1)                   # T.RandomCrop on the padded image
        out[b, 2] = rng.integers(0, 2 * pad + 1)
        if rng.uniform(0, 1) >= re_prob:                           # random_erasing.py:32
            continue
        for _ in range(100):
            target_area = rng.uniform(sl, sh) * h * w
            aspect = rng.uniform(r1, 1 / r1)
            eh, ew = int(round(math.sqrt(target_area * aspect))), int(round(math.sqrt(target_area / aspect)))
            if ew < w and eh < h:
                out[b, 3] = rng.integers(0, h - eh + 1)            # random.randint is inclusive
                out[b, 4] = rng.integers(0, w - ew + 1)
                out[b, 5], out[b, 6] = eh, ew
                break
    return out


def augment_batch(images_u8: torch.Tensor, params, pixel_mean=(0.485, 0.456, 0.406), pixel_std=(0.229, 0.224, 0.225),
                  pad: int = 10) -> torch.Tensor:
    """images_u8: uint8 [B, H, W, 3] on the device (resized crops); params: int32 [B, 8] (numpy or tensor).
    Returns the normalised fp32 NCHW batch [B, 3, H, W]."""
    N.require_cuda(images_u8)
    if images_u8.dtype != torch.uint8 or images_u8.dim() != 4 or images_u8.shape[-1] != 3:
        raise ValueError(f"expected uint8 [B, H, W, 3], got {images_u8.dtype} {tuple(images_u8.shape)}")
    images_u8 = images_u8.contiguous()
    b, h, w, _ = images_u8.shape
    p = torch.as_tensor(np.asarray(params, dtype=np.int32) if not torch.is_tensor(params) else params)
    if tuple(p.shape) != (b, 8):
        raise ValueError(f"params must be [B, 8], got {tuple(p.shape)}")
    p = p.to(device=images_u8.device, dtype=torch.int32).contiguous()
    out = torch.empty(b, 3, h, w, dtype=torch.float32, device=images_u8.device)
    mean = (C.c_float * 3)(*[float(v) for v in pixel_mean])
    std = (C.c_float * 3)(*[float(v) for v in pixel_std])
    N.check(N.lib().ctl_augment_batch_u8(images_u8.data_ptr(), b, h, w, int(pad), p.data_ptr(), mean, std, out.data_ptr(),
                                         N.stream_ptr()))
    return out


def normalize_batch(images_u8: torch.Tensor, pixel_mean=(0.485, 0.456, 0.406), pixel_std=(0.229, 0.224, 0.225)) -> torch.Tensor:
    """The eval transform after `T.Resize` (datasets/transforms/build.py:29-33: ToTensor + Normalize) on the device:
    uint8 [B, H, W, 3] -> normalised fp32 NCHW [B, 3, H, W] (no flip / crop / erasing).  A validation loader that ships
    uint8 crops moves 4x fewer bytes over PCIe than one that normalises on the host."""
    b = images_u8.shape[0]
    key = (b, images_u8.device)
    p = _NEUTRAL.get(key)
    if p is None:
        p = torch.zeros(b, 8, dtype=torch.int32, device=images_u8.device)
        p[:, 7] = 1  # is_real
        _NEUTRAL[key] = p
    return augment_batch(images_u8, p, pixel_mean, pixel_std, pad=0)


_NEUTRAL = {}


class RaggedImages:
    """A batch of native-size HWC RGB uint8 images of any sizes, packed back to back (no padding, any byte alignment)
    in one uint8 buffer `data`, with `table` int64 [n, 3] = {byte offset, h, w} per image (struct ctl_resize_entry);
    h = w = 0 is a mock row (the A0 batch contract's padded rows), which resizes to zeros.  `rows` is the sum of the
    real images' heights, the row count of resize_batch's intermediate.  Built by pack_images; `resize_batch` turns it
    into the `T.Resize` output."""

    def __init__(self, data: torch.Tensor, table: torch.Tensor, rows: int):
        self.data, self.table, self.rows = data, table, int(rows)

    def __len__(self):
        return self.table.shape[0]

    @property
    def device(self):
        return self.data.device

    def to(self, device, non_blocking: bool = True) -> "RaggedImages":
        """The same batch on `device`; from pinned host buffers the copies do not block the host."""
        return RaggedImages(self.data.to(device, non_blocking=non_blocking),
                            self.table.to(device, non_blocking=non_blocking), self.rows)


def pack_images(images, pin: bool = True) -> RaggedImages:
    """HWC uint8 arrays [h, w, 3] or PIL RGB images (the reference's loaders decode with `.convert("RGB")`,
    datasets/bases.py:32-33), with `None` for a mock row -> one host RaggedImages (pinned when `pin`)."""
    arrays = []
    for i, im in enumerate(images):
        if im is None:
            arrays.append(None)
            continue
        if hasattr(im, "mode") and hasattr(im, "size"):  # PIL image
            if im.mode != "RGB":
                raise ValueError(f"image {i}: PIL mode {im.mode!r}, expected 'RGB'")
            im = np.asarray(im)
        a = np.asarray(im)
        if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or a.shape[0] < 1 or a.shape[1] < 1:
            raise ValueError(f"image {i}: expected uint8 [h >= 1, w >= 1, 3], got {a.dtype} {a.shape}")
        arrays.append(np.ascontiguousarray(a))
    if not arrays:
        raise ValueError("pack_images: no images")
    table = np.zeros((len(arrays), 3), dtype=np.int64)
    off = 0
    for i, a in enumerate(arrays):
        if a is not None:
            table[i] = off, a.shape[0], a.shape[1]
            off += a.nbytes
    data = torch.empty(max(off, 1), dtype=torch.uint8, pin_memory=pin)
    flat = data.numpy()
    for (o, _, _), a in zip(table, arrays):
        if a is not None:
            flat[o: o + a.nbytes] = a.reshape(-1)
    t = torch.from_numpy(table)
    return RaggedImages(data, t.pin_memory() if pin else t, int(table[:, 1].sum()))


class JpegBatch:
    """A batch of image files packed back to back (any byte alignment) in one uint8 buffer `data`, for decode_batch.
    `entries` uint8 [n, 88] holds one struct ctl_jpeg_entry per image: a JPEG with the descriptor ctl_jpeg_parse read
    from its header, raw HWC RGB bytes (a file the device decode does not cover, decoded by Pillow in pack_jpegs), or a
    mock row.  `out_table` int64 [n, 3] = {byte offset, h, w} is the table of the RaggedImages decode_batch returns,
    `out_bytes` its buffer size, `rows` the sum of its heights; `workspace_bytes` is ctl_jpeg_decode_workspace_bytes of
    the entries; `fallback` lists the indices decoded on the host, with the parser's reason for each."""

    def __init__(self, data, entries, out_table, out_bytes, rows, workspace_bytes, fallback=()):
        self.data, self.entries, self.out_table = data, entries, out_table
        self.out_bytes, self.rows, self.workspace_bytes = int(out_bytes), int(rows), int(workspace_bytes)
        self.fallback = list(fallback)

    def __len__(self):
        return self.entries.shape[0]

    @property
    def device(self):
        return self.data.device

    def to(self, device, non_blocking: bool = True) -> "JpegBatch":
        """The same batch on `device`; from pinned host buffers the copies do not block the host."""
        return JpegBatch(self.data.to(device, non_blocking=non_blocking),
                         self.entries.to(device, non_blocking=non_blocking),
                         self.out_table.to(device, non_blocking=non_blocking), self.out_bytes, self.rows,
                         self.workspace_bytes, self.fallback)


def parse_jpeg(data):
    """ctl_jpeg_parse of one file's bytes -> (struct ctl_jpeg_desc, None), or (None, the reason the device decode
    does not cover it)."""
    buf = bytes(data)
    desc = N.JpegDesc()
    rc = N.lib().ctl_jpeg_parse(buf, len(buf), C.byref(desc), None, None)
    if rc != 0:
        return None, N.lib().ctl_last_error().decode("utf-8", "replace")
    return desc, None


def _read_item(i, item):
    if isinstance(item, (bytes, bytearray, memoryview)):
        return bytes(item)
    if isinstance(item, (str, bytes)) or hasattr(item, "__fspath__"):
        with open(item, "rb") as f:
            return f.read()
    raise ValueError(f"item {i}: expected file bytes, a path or None, got {type(item).__name__}")


def pack_jpegs(items, pin: bool = True) -> JpegBatch:
    """Image files -- bytes, or paths read here, with `None` for a mock row -> one host JpegBatch (pinned when `pin`).
    A file ctl_jpeg_parse rejects (progressive, CMYK, PNG, ...) is decoded here with `Image.open(...).convert("RGB")`,
    as the reference's loaders do (datasets/bases.py:32-33), and stored as raw RGB bytes, so a mixed dataset still
    gives one batch whose decode equals the reference's.  Meant for loader workers: the collate of file bytes."""
    import io

    from PIL import Image

    blobs, descs, fallback = [], [], []
    for i, item in enumerate(items):
        if item is None:
            blobs.append(None)
            descs.append(None)
            continue
        raw = _read_item(i, item)
        desc, why = parse_jpeg(raw)
        if desc is None:
            try:
                with Image.open(io.BytesIO(raw)) as im:
                    rgb = np.ascontiguousarray(np.asarray(im.convert("RGB")))
            except Exception as exc:  # noqa: BLE001 -- any Pillow failure means the item is not an image
                raise ValueError(f"item {i}: neither a JPEG this decode covers ({why}) nor an image Pillow "
                                 f"reads ({exc})") from exc
            fallback.append((i, why))
            blobs.append(rgb)
        else:
            blobs.append(raw)
        descs.append(desc)
    n = len(blobs)
    if n == 0:
        raise ValueError("pack_jpegs: no items")
    entries = (N.JpegEntry * n)()
    out_table = np.zeros((n, 3), dtype=np.int64)
    off = out_off = 0
    for i, (blob, desc) in enumerate(zip(blobs, descs)):
        e = entries[i]
        if blob is None:
            e.kind = N.CTL_JPEG_ENTRY_MOCK
            continue
        if isinstance(blob, np.ndarray):
            e.kind = N.CTL_JPEG_ENTRY_RAW
            e.desc.h, e.desc.w = blob.shape[0], blob.shape[1]
            nbytes = blob.nbytes
        else:
            e.kind = N.CTL_JPEG_ENTRY_JPEG
            e.desc = desc
            nbytes = len(blob)
        e.offset, e.nbytes = off, nbytes
        out_table[i] = out_off, e.desc.h, e.desc.w
        off += nbytes
        out_off += e.desc.h * e.desc.w * 3
    data = torch.empty(max(off, 1), dtype=torch.uint8, pin_memory=pin)
    flat = data.numpy()
    for i, blob in enumerate(blobs):
        if blob is not None:
            o = entries[i].offset
            flat[o: o + entries[i].nbytes] = np.frombuffer(blob, dtype=np.uint8) if isinstance(blob, bytes) \
                else blob.reshape(-1)
    ws = N.lib().ctl_jpeg_decode_workspace_bytes(C.addressof(entries), n)
    ent = torch.from_numpy(np.frombuffer(entries, dtype=np.uint8).reshape(n, C.sizeof(N.JpegEntry)).copy())
    tab = torch.from_numpy(out_table)
    if pin:
        ent, tab = ent.pin_memory(), tab.pin_memory()
    return JpegBatch(data, ent, tab, out_off, int(out_table[:, 1].sum()), ws, fallback)


def _decode_enqueue(batch: JpegBatch, out: torch.Tensor, status: torch.Tensor, workspace: torch.Tensor):
    """ctl_jpeg_decode (enqueue only, capturable in a CUDA graph); the caller reads `status` back."""
    N.check(N.lib().ctl_jpeg_decode(batch.data.data_ptr(), batch.data.numel(), batch.entries.data_ptr(), len(batch),
                                    batch.out_table.data_ptr(), out.data_ptr(), batch.out_bytes, status.data_ptr(),
                                    workspace.data_ptr(), workspace.numel(), N.stream_ptr()))


def decode_batch(batch: JpegBatch) -> RaggedImages:
    """`Image.open(p).convert("RGB")` of every image of a device JpegBatch -> a device RaggedImages (the input of
    resize_batch), bit for bit Pillow's output; mock rows stay mock rows.  Reads the per-image status back (one
    synchronisation) and raises ValueError naming the images whose data is corrupt or whose entry does not fit; their
    output is zeros."""
    N.require_cuda(batch.data, batch.entries, batch.out_table)
    if batch.data.dtype != torch.uint8 or batch.entries.dtype != torch.uint8 or batch.out_table.dtype != torch.int64:
        raise ValueError("decode_batch: expected a JpegBatch from pack_jpegs")
    dev = batch.device
    with torch.cuda.device(dev):
        out = torch.empty(max(batch.out_bytes, 1), dtype=torch.uint8, device=dev)
        status = torch.empty(len(batch), dtype=torch.int32, device=dev)
        ws = torch.empty(max(batch.workspace_bytes, 1), dtype=torch.uint8, device=dev)
        _decode_enqueue(batch, out, status, ws)
        st = status.cpu().numpy()
    bad = np.flatnonzero(st)
    if bad.size:
        what = {1: "corrupt or truncated entropy-coded data", 2: "entry outside the data buffer",
                4: "output entry does not fit", 8: "workspace too short"}
        detail = ", ".join(f"{i}: " + " / ".join(v for k, v in what.items() if st[i] & k) for i in bad[:16])
        raise ValueError(f"decode_batch: {bad.size} image(s) failed ({detail}{', ...' if bad.size > 16 else ''}); "
                         "their output is zeros")
    return RaggedImages(out, batch.out_table, batch.rows)


def _resize_size(size):
    if isinstance(size, (int, np.integer)) or len(size) != 2:
        raise ValueError(f"size must be (h, w) as in T.Resize((h, w)) / INPUT.SIZE_TEST, got {size!r}")
    return int(size[0]), int(size[1])


def resize_workspace_bytes(ragged: RaggedImages, size) -> int:
    """Bytes of the uint8 intermediate [ragged.rows, w, 3] (ctl_resize_bilinear_u8_workspace_bytes)."""
    h, w = _resize_size(size)
    n = N.lib().ctl_resize_bilinear_u8_workspace_bytes(ragged.rows, h, w)
    if n == 0:
        raise ValueError(f"resize to {size!r}: unsupported output size")
    return n


def _resize_enqueue(ragged: RaggedImages, out: torch.Tensor, status: torch.Tensor, workspace: torch.Tensor):
    """ctl_resize_bilinear_u8 (enqueue only, capturable in a CUDA graph); the caller reads `status` back."""
    N.check(N.lib().ctl_resize_bilinear_u8(ragged.data.data_ptr(), ragged.data.numel(), ragged.table.data_ptr(),
                                           len(ragged), out.shape[1], out.shape[2], out.data_ptr(), status.data_ptr(),
                                           workspace.data_ptr(), workspace.numel(), N.stream_ptr()))


def resize_batch(ragged: RaggedImages, size) -> torch.Tensor:
    """`T.Resize((h, w))` (datasets/transforms/build.py:19,29: PIL `Image.resize((w, h), BILINEAR)`) of every image of a
    device RaggedImages -> uint8 [B, h, w, 3] on the device, bit for bit PIL's output; mock rows are zeros.  The input
    of augment_batch, normalize_batch and TrunkEngine.forward_u8.  Reads the device status word back (one
    synchronisation) and raises ValueError when a table entry does not fit in the data buffer."""
    N.require_cuda(ragged.data, ragged.table)
    if ragged.data.dtype != torch.uint8 or ragged.table.dtype != torch.int64 or ragged.table.dim() != 2 \
            or ragged.table.shape[1] != 3 or not ragged.table.is_contiguous():
        raise ValueError("resize_batch: expected a RaggedImages from pack_images")
    h, w = _resize_size(size)
    dev = ragged.device
    with torch.cuda.device(dev):
        out = torch.empty(len(ragged), h, w, 3, dtype=torch.uint8, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        ws = torch.empty(resize_workspace_bytes(ragged, (h, w)), dtype=torch.uint8, device=dev)
        _resize_enqueue(ragged, out, status, ws)
        st = int(status.item())
    if st:
        raise ValueError(f"resize_batch: status {st}: a table entry lies outside the image buffer"
                         f"{' or the intermediate' if st & 2 else ''}; its output is zeros")
    return out
