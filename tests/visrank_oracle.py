"""Host restatement of visualize_ranked_results (utils/visrank.py:23-244 of the reference) for image data, in numpy
integers: the checker of ctl_resize_linear_cv_u8, ctl_visrank_compose, ctl_visrank_select and utils/visrank.py.

`cv_resize` is cv2.resize(img, (w, h)) with INTER_LINEAR on uint8 3-channel images; `grid` is one ranked-result PNG
in RGB; `ranked` is the loop of visrank.py:192-232 over (distance, index) order; `galleries` makes the centroid-mode
representative picks of visrank.py:60-121 with the same random.choice calls.
"""
from __future__ import annotations

import os
import random
from collections import defaultdict

import numpy as np

BW, SPACING, QUERY_EXTRA = 3, 2, 8  # visrank.py:16-18
BLACK, GREEN, RED = (0, 0, 0), (0, 255, 0), (255, 0, 0)  # RGB


def _axis(n_in: int, n_out: int, clamp_weights: bool):
    d = np.arange(n_out, dtype=np.float64)
    f = ((d + 0.5) * (n_in / n_out) - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp_weights:
        lo, hi = s < 0, s >= n_in - 1
        s[lo], f[lo] = 0, 0
        s[hi], f[hi] = n_in - 1, 0
    a0 = np.rint((np.float32(1) - f).astype(np.float32) * np.float32(2048)).astype(np.int64)
    return np.clip(s, 0, n_in - 1), np.clip(s + 1, 0, n_in - 1), a0, 2048 - a0


def cv_resize(src: np.ndarray, h: int, w: int) -> np.ndarray:
    """cv2.resize(src, (w, h)) (INTER_LINEAR) of a uint8 [H, W, 3] image."""
    x0, x1, a0, a1 = _axis(src.shape[1], w, True)
    y0, y1, b0, b1 = _axis(src.shape[0], h, False)
    s = src.astype(np.int64)
    hrow = s[:, x0] * a0[None, :, None] + s[:, x1] * a1[None, :, None]
    out = (((b0[:, None, None] * (hrow[y0] >> 4)) >> 16) + ((b1[:, None, None] * (hrow[y1] >> 4)) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


def border(img: np.ndarray, colour) -> np.ndarray:
    """cv2.copyMakeBorder(img, 3, 3, 3, 3, BORDER_CONSTANT, value=colour)."""
    out = np.empty((img.shape[0] + 2 * BW, img.shape[1] + 2 * BW, 3), dtype=np.uint8)
    out[:] = np.asarray(colour, dtype=np.uint8)
    out[BW:-BW, BW:-BW] = img
    return out


def cell(img: np.ndarray, h: int, w: int, colour) -> np.ndarray:
    """visrank.py:168-174 / 206-211: resize, border, resize again."""
    return cv_resize(border(cv_resize(img, h, w), colour), h, w)


def grid_width(w: int, topk: int) -> int:
    return (topk + 1) * w + topk * SPACING + QUERY_EXTRA


def cell_x(col: int, w: int) -> int:
    return 0 if col == 0 else col * w + col * SPACING + QUERY_EXTRA


def grid(query_img, ranked_imgs, h: int, w: int, topk: int) -> np.ndarray:
    """One grid: ranked_imgs is a list of (image, matched) in rank order, at most topk."""
    out = np.full((h, grid_width(w, topk), 3), 255, dtype=np.uint8)
    out[:, :w] = cell(query_img, h, w, BLACK)
    for c, (img, matched) in enumerate(ranked_imgs, start=1):
        x = cell_x(c, w)
        out[:, x: x + w] = cell(img, h, w, GREEN if matched else RED)
    return out


def galleries(dataset, num_q: int, use_centroids: bool, keep_camid_centroids: bool):
    """visrank.py:55-121 -> (query samples, gallery samples, respect_camids).  Samples are (path, pid, camid, ...)
    tuples; a centroid's camid is the tuple of cameras it was built from.  The picks use a private random.Random(0)
    with the reference's calls in its order, including its indexing of `camids` (query + gallery rows) with gallery
    positions."""
    query = list(dataset[:num_q])
    respect = bool(use_centroids and keep_camid_centroids)
    if not use_centroids:
        return query, list(dataset[num_q:]), respect
    gallery_list = list(dataset[num_q:])
    labels_gallery = [int(s[1]) for s in gallery_list]
    camids = np.asarray([int(s[2]) for s in [*query, *gallery_list]])
    labels_query = [int(s[1]) for s in query]
    rng = random.Random(0)
    labels2idx, labels2idx_q = defaultdict(list), defaultdict(list)
    for i, lab in enumerate(labels_gallery):
        labels2idx[lab].append(i)
    for i, lab in enumerate(labels_query):
        labels2idx_q[lab].append(i)
    centroids = []
    for label in sorted(np.unique(list(labels2idx.keys()))):
        combos = set()
        inds, inds_q = labels2idx[label], labels2idx_q[label]
        if respect:
            cams_g = camids[inds]
            for cur in sorted(np.unique(camids[inds_q])):
                sel = np.where(cams_g != cur)[0]
                if sel.shape[0] == 0:
                    continue
                used = tuple(sorted(np.unique([c for c in cams_g if c != cur]).tolist()))
                if used not in combos:
                    combos.add(used)
                    pick = rng.choice([gallery_list[inds[j]] for j in sel])
                    centroids.append((pick[0], int(pick[1]), used) + tuple(pick[3:]))
    return query, centroids, respect


def is_junk(q, g, respect: bool) -> bool:
    if respect:
        return int(g[1]) == int(q[1]) and int(q[2]) in g[2]
    return q[1] == g[1] and q[2] == g[2]


def ranked(dist_row: np.ndarray, q, gallery, respect: bool, topk: int):
    """visrank.py:192-232: the first topk non-junk gallery rows in (distance, index) order -> [(g_idx, matched)]."""
    out = []
    for g_idx in np.argsort(dist_row, kind="stable"):
        g = gallery[g_idx]
        if not is_junk(q, g, respect):
            out.append((int(g_idx), int(g[1]) == int(q[1])))
            if len(out) >= topk:
                break
    return out


def visualize(distmat, dataset, load, use_centroids: bool, keep_camid_centroids: bool, max_number: int, topk: int,
              h: int, w: int) -> dict:
    """The PNGs visualize_ranked_results writes, as {file name: RGB grid}; `load(path)` gives an image's RGB pixels."""
    num_q, num_g = distmat.shape
    query, gallery, respect = galleries(dataset, num_q, use_centroids, keep_camid_centroids)
    assert num_g == len(gallery)
    out = {}
    for q_idx in range(min(num_q, int(max_number) + 1)):
        q = query[q_idx]
        ranks = ranked(distmat[q_idx], q, gallery, respect, topk)
        name = os.path.basename(os.path.splitext(q[0])[0]) + ".png"
        out[name] = grid(load(q[0]), [(load(gallery[g][0]), m) for g, m in ranks], h, w, topk)
    return out


def load_case(g, root: str) -> dict:
    """A tests/golden/visrank_*.npz case (tools/make_visrank_golden.py) with its image files written under `root`:
    cfg, samples (absolute paths), feats, pids, camids, distmat, and expected {name: grid} or error."""
    import json

    offs = g["file_offsets"]
    for i, name in enumerate(g["file_names"]):
        path = os.path.join(root, str(name))
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as f:
            f.write(g["file_data"][offs[i]: offs[i + 1]].tobytes())
    case = dict(cfg=json.loads(str(g["cfg"])), feats=g["feats"], pids=json.loads(str(g["pids"])),
                camids=json.loads(str(g["camids"])), distmat=g["distmat"],
                samples=[(os.path.join(root, s[0]), s[1], s[2], s[3]) for s in json.loads(str(g["samples"]))])
    case["error"] = str(g["error"]) if "error" in g.files else None
    case["expected"] = {} if case["error"] else {str(n): g["grids"][i] for i, n in enumerate(g["names"])}
    return case


def load_rgb(path: str) -> np.ndarray:
    """Image.open(path).convert("RGB"): cv2.imread's pixels, in RGB order."""
    from PIL import Image

    with Image.open(path) as im:
        return np.asarray(im.convert("RGB"))


def read_pngs(directory: str) -> dict:
    return {n: load_rgb(os.path.join(directory, n)) for n in sorted(os.listdir(directory))}
