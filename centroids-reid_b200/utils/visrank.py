"""Drop-in for utils/visrank.py of the reference (visualize_ranked_results) on the H100: one ranked-result PNG per
query, pixel for pixel the reference's.

The reference reads 1 + topk images per query with cv2.imread, resizes each twice around a 3-px border and writes the
grid with cv2.imwrite, one query at a time.  Here the queries are rendered in chunks under a device-memory budget:
  ranking   the first topk non-junk gallery rows per query (ctl_visrank_select) from a (distance, index) top-k wide
            enough to hold every junk row: of the distance matrix (sorted key rows) or, from R1_mAP.compute's planes,
            the streamed top-k, which builds no [Q, G] matrix;
  images    file bytes read on host threads, decoded on the device once per chunk (pack_jpegs -> decode_batch, which
            is Pillow's decode, i.e. cv2.imread's pixels in RGB order), resized with cv2's INTER_LINEAR
            (ctl_resize_linear_cv_u8) and composed with their borders into white grids (ctl_visrank_compose);
  PNGs      copied into pinned memory and written as RGB PNGs (zlib) by a host thread pool while the next chunk runs.
The files' pixels equal the reference's; their bytes need not (another PNG encoder).
"""
from __future__ import annotations

import os
import random
import struct
import zlib
from collections import defaultdict
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from .. import _native as N
from .. import retrieval as _R
from ..datasets import transforms as _T

BW, GRID_SPACING, QUERY_EXTRA_SPACING = 3, 2, 8  # visrank.py:16-18
BLACK, GREEN, RED = 0x000000, 0x00FF00, 0xFF0000  # RGB
SORT_WIDTH = 16384  # widest key row ctl_sort_key_rows sorts


def _galleries(dataset, num_q: int, use_centroids: bool, keep_camid_centroids: bool):
    """visrank.py:55-121 -> (query samples, gallery samples, respect_camids).  In centroid mode with
    KEEP_CAMID_CENTROIDS each centroid is represented by one gallery image picked with random.choice; the picks use a
    private random.Random(0) with the reference's calls in its order (the caller's global random state is left alone),
    including its indexing of `camids` (query + gallery rows) with gallery positions.  Without KEEP_CAMID_CENTROIDS the
    reference builds no centroid, and its assert on the gallery length fails."""
    query = list(dataset[:num_q])
    respect = bool(use_centroids and keep_camid_centroids)
    if not use_centroids:
        return query, list(dataset[num_q:]), respect
    gallery_list = list(dataset[num_q:])
    camids = np.asarray([int(s[2]) for s in [*query, *gallery_list]])
    labels2idx, labels2idx_q = defaultdict(list), defaultdict(list)
    for i, s in enumerate(gallery_list):
        labels2idx[int(s[1])].append(i)
    for i, s in enumerate(query):
        labels2idx_q[int(s[1])].append(i)
    rng = random.Random(0)
    centroids = []
    for label in sorted(np.unique(list(labels2idx.keys()))):
        if not respect:
            continue
        combos = set()
        inds, inds_q = labels2idx[label], labels2idx_q[label]
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


def _ids(query, gallery, respect: bool, topk: int, dev):
    """Device identity arrays (retrieval.EncodedIds layout, caller order) and the top-k width that holds each query's
    topk non-junk rows: topk + the largest junk count of any query, at most the gallery size."""
    qp, qc, gp, gm, _ = _R.encode_identities([s[1] for s in query], [s[1] for s in gallery], [s[2] for s in query],
                                             [s[2] for s in gallery], respect)
    n_p = int(max(qp.max(initial=0), gp.max(initial=0))) + 1
    junk = np.zeros(len(query), dtype=np.int64)
    for c in np.unique(qc):
        seen = ((gm >> np.uint64(c)) & np.uint64(1)).astype(bool)
        sel = qc == c
        junk[sel] = np.bincount(gp[seen], minlength=n_p)[qp[sel]]
    k = int(min(len(gallery), topk + int(junk.max(initial=0))))

    def to_dev(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(dev)

    return (to_dev(qp), to_dev(qc), to_dev(gp), to_dev(gm.view(np.int64))), k


def _rank_dense(d: torch.Tensor, k: int, budget: int) -> torch.Tensor:
    """idx int64 [n, k]: the k smallest of every row of a float32 [n, G] device matrix in (distance, index) order --
    ctl_sort_key_rows over column blocks of at most SORT_WIDTH, each block's k best merged into the running k best."""
    n, ng = d.shape
    if ng > SORT_WIDTH and 2 * k > SORT_WIDTH:
        raise NotImplementedError(f"top-{k} of a {ng}-column distance matrix: at most {SORT_WIDTH // 2} past "
                                  f"{SORT_WIDTH} columns")
    out = torch.empty(n, k, dtype=torch.int64, device=d.device)
    rows = max(1, budget // (16 * min(ng, SORT_WIDTH)))
    for r0 in range(0, n, rows):
        blk = d[r0: r0 + rows]
        best = None
        for c0 in range(0, ng, SORT_WIDTH):
            part = blk[:, c0: c0 + SORT_WIDTH]
            col = torch.arange(c0, c0 + part.shape[1], device=d.device).expand(part.shape[0], -1)
            idx, dst = _R.merge_topk_keys(_R.pack_keys(part, col), min(k, part.shape[1]))
            if best is not None:
                idx, dst = _R.merge_topk_keys(_R.pack_keys(torch.cat([best[1], dst], 1), torch.cat([best[0], idx], 1)),
                                              min(k, best[0].shape[1] + idx.shape[1]))
            best = (idx, dst)
        out[r0: r0 + rows] = best[0]
    return out


def _rank_planes(qp: _R.Planes, gp: _R.Planes, k: int) -> torch.Tensor:
    """idx int64 [qp.n, k] in the caller's query and gallery indexing: the streamed top-k (no distance matrix)."""
    ex = _R.ShardExchange(None)
    try:
        idx, _ = _R._streamed(ex, qp, gp, None, k, None, gp.n, 0, 0, tile_lists=True)
    except OverflowError:  # more rows than a candidate list holds passed the subset threshold: the exact one
        idx, _ = _R._streamed(ex, qp, gp, None, k, None, gp.n, 0, 0, tile_lists=False)
    inv = _R._query_inverse(qp)[0]
    return idx if inv is None else idx.index_select(0, inv)


def ranked_lists(topk_idx: torch.Tensor, ids, ng: int, topk: int):
    """ctl_visrank_select: (idx int64 [n, topk], matched int8 [n, topk]) on the device, -1 / 0 past a query's last
    non-junk row.  topk_idx: int64 [n, k] in (distance, index) order; ids: (q_pid, q_cam, g_pid, g_mask) device arrays."""
    N.require_cuda(topk_idx)
    topk_idx = topk_idx.contiguous()
    n, k = topk_idx.shape
    dev = topk_idx.device
    out = torch.empty(n, topk, dtype=torch.int64, device=dev)
    matched = torch.empty(n, topk, dtype=torch.int8, device=dev)
    status = torch.empty(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        N.check(N.lib().ctl_visrank_select(topk_idx.data_ptr(), n, k, *[t.data_ptr() for t in ids], ng, topk,
                                           out.data_ptr(), matched.data_ptr(), status.data_ptr(), N.stream_ptr()))
    return out, matched, status


def resize_linear_cv(ragged: "_T.RaggedImages", size) -> torch.Tensor:
    """cv2.resize(img, (w, h)) (INTER_LINEAR) of every image of a device RaggedImages -> uint8 [B, h, w, 3], bit for
    bit; mock rows are zeros.  Reads the per-entry status back and raises ValueError naming the entries that do not
    fit in the data buffer (their output is zeros)."""
    out, status = _resize_linear_cv_enqueue(ragged, size)
    bad = np.flatnonzero(status.cpu().numpy())
    if bad.size:
        raise ValueError(f"resize_linear_cv: entries {bad[:16].tolist()} lie outside the image buffer; their output "
                         "is zeros")
    return out


def _resize_linear_cv_enqueue(ragged, size):
    N.require_cuda(ragged.data, ragged.table)
    if ragged.data.dtype != torch.uint8 or ragged.table.dtype != torch.int64 or ragged.table.dim() != 2 \
            or ragged.table.shape[1] != 3 or not ragged.table.is_contiguous():
        raise ValueError("resize_linear_cv: expected a RaggedImages")
    h, w = int(size[0]), int(size[1])
    dev = ragged.device
    with torch.cuda.device(dev):
        out = torch.empty(len(ragged), h, w, 3, dtype=torch.uint8, device=dev)
        status = torch.empty(len(ragged), dtype=torch.int32, device=dev)
        N.check(N.lib().ctl_resize_linear_cv_u8(ragged.data.data_ptr(), ragged.data.numel(), ragged.table.data_ptr(),
                                                len(ragged), h, w, out.data_ptr(), status.data_ptr(), N.stream_ptr()))
    return out, status


def grid_width(width: int, topk: int) -> int:
    return (topk + 1) * width + topk * GRID_SPACING + QUERY_EXTRA_SPACING


def compose(resized: torch.Tensor, cells, n_grids: int, topk: int):
    """ctl_visrank_compose: uint8 [n_grids, h, grid_width, 3] white grids with the cells {row of `resized`, grid,
    column, 0xRRGGBB border} pasted in (the status word is 1 when a cell was out of range)."""
    N.require_cuda(resized)
    resized = resized.contiguous()
    n_rows, h, w, _ = resized.shape
    dev = resized.device
    cells = torch.as_tensor(cells, dtype=torch.int32).reshape(-1, 4).to(dev).contiguous()
    with torch.cuda.device(dev):
        out = torch.empty(n_grids, h, grid_width(w, topk), 3, dtype=torch.uint8, device=dev)
        status = torch.empty(1, dtype=torch.int32, device=dev)
        N.check(N.lib().ctl_visrank_compose(resized.data_ptr(), n_rows, h, w, N.ptr(cells) if len(cells) else None,
                                            cells.shape[0], n_grids, topk, out.data_ptr(), status.data_ptr(),
                                            N.stream_ptr()))
    return out, status


def png_bytes(rgb: np.ndarray, level: int = 1) -> bytes:
    """An 8-bit RGB PNG of a uint8 [h, w, 3] array (filter type 0 on every row)."""
    h, w, _ = rgb.shape
    raw = np.zeros((h, 1 + 3 * w), dtype=np.uint8)
    raw[:, 1:] = rgb.reshape(h, 3 * w)

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data))

    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0))
            + chunk(b"IDAT", zlib.compress(raw.tobytes(), level)) + chunk(b"IEND", b""))


def _write_pngs(event, grids_host, paths):
    event.synchronize()
    arr = grids_host.numpy()
    for i, p in enumerate(paths):
        with open(p, "wb") as f:
            f.write(png_bytes(arr[i]))


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def _progress(lo, hi, num_q):
    """visrank.py:238-239 for queries lo .. hi - 1; returns hi."""
    for q in range(lo, hi):
        if (q + 1) % 100 == 0:
            print("- done {}/{}".format(q + 1, num_q))
    return hi


def _render(query, gallery, idx, matched, width, height, save_dir, topk, num_q, dev, memory_budget, pool):
    """Grids of queries 0 .. len(query) - 1 (idx / matched: host [n, topk]), chunked so that each chunk's device
    buffers stay under memory_budget bytes (one grid at least)."""
    names = [os.path.basename(os.path.splitext(str(q[0]))[0]) for q in query]
    last = {n: i for i, n in enumerate(names)}  # a later query of the same name overwrites an earlier one's file
    todo = [i for i in range(len(query)) if last[names[i]] == i]
    gw = grid_width(width, topk)
    cell_bytes, grid_bytes = height * width * 3, height * gw * 3
    per_grid = grid_bytes + (topk + 1) * cell_bytes
    pending, done = [], 0
    step = max(1, memory_budget // per_grid)
    stack = [todo[i: i + step] for i in range(0, len(todo), step)][::-1]  # popped in query order; a chunk whose
    # decoded images do not fit is split in two halves, pushed back in order
    while stack:
        chunk = stack.pop()
        paths, rows, cells = [], {}, []
        for g, qi in enumerate(chunk):
            items = [(str(query[qi][0]), 0, BLACK)] + [(str(gallery[j][0]), c, GREEN if m else RED)
                                                      for c, (j, m) in enumerate(zip(idx[qi], matched[qi]), 1) if j >= 0]
            for p, col, colour in items:
                if p not in rows:
                    rows[p] = len(paths)
                    paths.append(p)
                cells.append((rows[p], g, col, colour))
        batch = _T.pack_jpegs(list(pool.map(_read, paths)))
        need = batch.out_bytes + batch.workspace_bytes + batch.data.numel() + len(chunk) * grid_bytes \
            + len(paths) * cell_bytes
        if need > memory_budget and len(chunk) > 1:
            stack += [chunk[len(chunk) // 2:], chunk[: len(chunk) // 2]]
            continue
        with torch.cuda.device(dev):
            ragged = _T.decode_batch(batch.to(dev))
            resized, st_resize = _resize_linear_cv_enqueue(ragged, (height, width))
            grids, st_compose = compose(resized, cells, len(chunk), topk)
            host = torch.empty(grids.shape, dtype=torch.uint8, pin_memory=True)
            host.copy_(grids, non_blocking=True)
            event = torch.cuda.Event()
            event.record()
            if st_resize.any().item() or st_compose.item():
                raise RuntimeError("visrank: an image or a grid cell was out of range")
        pending.append(pool.submit(_write_pngs, event, host, [os.path.join(save_dir, names[qi] + ".png") for qi in chunk]))
        done = _progress(done, chunk[-1] + 1, num_q)
    _progress(done, len(query), num_q)
    for f in pending:
        f.result()


def _visualize(rank, num_q, num_g, dataset, cfg, width, height, save_dir, topk, dev, memory_budget):
    os.makedirs(save_dir, exist_ok=True)
    query, gallery, respect = _galleries(dataset, num_q, bool(cfg.MODEL.USE_CENTROIDS),
                                         bool(cfg.MODEL.KEEP_CAMID_CENTROIDS))
    assert num_q == len(query)
    assert num_g == len(gallery)
    n_vis = min(num_q, int(cfg.TEST.VISUALIZE_MAX_NUMBER) + 1)  # visrank.py:241: the break comes after the write
    query = query[:n_vis]
    topk = int(topk)
    ids, k = _ids(query, gallery, respect, topk, dev)
    idx, matched, status = ranked_lists(rank(n_vis, k), ids, num_g, topk)
    if status.item():
        raise RuntimeError("visrank: a top-k index lies outside the gallery")
    with ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 4)) as pool:
        _render(query, gallery, idx.cpu().numpy(), matched.cpu().numpy(), int(width), int(height), save_dir, topk,
                num_q, dev, memory_budget, pool)
    print('Done. Images have been saved to "{}" ...'.format(save_dir))


def visualize_ranked_results(distmat, dataset, data_type, cfg, width=128, height=256, save_dir="", topk=10,
                             memory_budget=1 << 30):
    """utils/visrank.py:23-244 for image re-id.  distmat: numpy or tensor [num_query, num_gallery], ranked on the
    device in (distance, index) order (float32; a float64 matrix must hold float32 values); dataset: the (path, pid,
    camid, index) samples of the queries, then the gallery.  Writes save_dir/<query file name>.png for queries
    0 .. cfg.TEST.VISUALIZE_MAX_NUMBER.  memory_budget: device bytes of one chunk of grids."""
    if data_type != "image":
        raise NotImplementedError("visualize_ranked_results renders image re-id only (R1_mAP passes 'image')")
    d = torch.as_tensor(distmat)
    if d.dim() != 2:
        raise ValueError(f"distmat must be [num_query, num_gallery], got {tuple(d.shape)}")
    if d.dtype != torch.float32:
        d32 = d.float()
        if not torch.equal(d32.to(d.dtype), d):
            raise ValueError(f"distmat of {d.dtype} ranks in float32: its values must be float32 values")
        d = d32
    dev = d.device if d.is_cuda else torch.device("cuda", torch.cuda.current_device())
    num_q, num_g = d.shape

    def rank(n, k):
        return _rank_dense(d[:n].to(dev).contiguous(), k, memory_budget)

    _visualize(rank, num_q, num_g, dataset, cfg, width, height, save_dir, topk, dev, memory_budget)


def visualize_ranked_planes(qp: _R.Planes, gp: _R.Planes, dataset, cfg, width=128, height=256, save_dir="", topk=10,
                            memory_budget=1 << 30):
    """visualize_ranked_results from the query and gallery planes R1_mAP.compute builds (any row order): the ranking
    is the streamed top-k, so no [num_query, num_gallery] matrix exists at any point."""

    def rank(n, k):
        return _rank_planes(qp, gp, k)[:n]

    _visualize(rank, qp.n, gp.n, dataset, cfg, width, height, save_dir, topk, qp.buf.device, memory_budget)
