"""Host restatement of PIL's BILINEAR `Image.resize` on RGB images, the `T.Resize((h, w))` of the reference's transforms
(datasets/transforms/build.py:19,29), in float64 and integers: the checker of `ctl_resize_bilinear_u8`.

Each axis is resampled separately, the width first, then the height of the width pass's output clipped to uint8.  The
weights of output index o along an axis of `n_in` -> `n_out` pixels are computed with Python floats (IEEE double, one
rounding per operation, no contraction) in PIL's order; the pixel sums are exact integers.
"""
from __future__ import annotations

import functools

import numpy as np

PRECISION_BITS = 22


@functools.lru_cache(maxsize=None)
def axis_coeffs(n_in: int, n_out: int):
    """-> (xmin int64 [n_out], k int64 [n_out, taps]): the fixed-point weights of each output index, zero-padded."""
    scale = n_in / n_out
    support = max(scale, 1.0)  # the triangle's support (1.0) times the filter scale
    ss = 1.0 / support
    rows, xmins = [], []
    for o in range(n_out):
        center = (o + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)  # int() truncates toward zero, like the C cast
        taps = min(int(center + support + 0.5), n_in) - xmin
        w = []
        for x in range(taps):
            t = abs((x + xmin - center + 0.5) * ss)
            w.append(1.0 - t if t < 1.0 else 0.0)
        ww = 0.0
        for v in w:
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        rows.append([int(0.5 + v * (1 << PRECISION_BITS)) for v in w])  # never negative: truncation == C cast
        xmins.append(xmin)
    k = np.zeros((n_out, max(len(r) for r in rows)), dtype=np.int64)
    for o, r in enumerate(rows):
        k[o, : len(r)] = r
    return np.array(xmins, dtype=np.int64), k


def resample_axis0(a: np.ndarray, n_out: int) -> np.ndarray:
    """uint8 [n_in, ...] -> uint8 [n_out, ...] along axis 0."""
    n_in = a.shape[0]
    xmin, k = axis_coeffs(n_in, n_out)
    idx = np.minimum(xmin[:, None] + np.arange(k.shape[1])[None, :], n_in - 1)  # padded taps carry weight 0
    acc = np.full((n_out,) + a.shape[1:], 1 << (PRECISION_BITS - 1), dtype=np.int64)
    for t in range(k.shape[1]):
        kt = k[:, t].reshape((n_out,) + (1,) * (a.ndim - 1))
        acc += a[idx[:, t]].astype(np.int64) * kt
    return np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)


def resize_bilinear(img: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """uint8 HWC [h, w, 3] -> uint8 [out_h, out_w, 3] == np.asarray(Image.fromarray(img).resize((out_w, out_h),
    Image.BILINEAR)).  A pass whose size does not change is skipped, as in PIL."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    h, w = img.shape[:2]
    out = img
    if out_w != w:
        out = resample_axis0(out.transpose(1, 0, 2), out_w).transpose(1, 0, 2)
    if out_h != h:
        out = resample_axis0(out, out_h)
    return np.ascontiguousarray(out)
