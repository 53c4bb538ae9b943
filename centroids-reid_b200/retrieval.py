"""Query x gallery retrieval engine: distance planes, full matrices, streamed top-k and
streamed CMC / mAP, single GPU or gallery-sharded over ranks.

Host-side mirror of the reference's retrieval path (utils/reid_metric.py:112-136,
utils/eval_reid.py:25-92, inference/get_similar.py:104-128) on top of the C ABI in
include/ctl_b200.h.  torch is used for device memory, streams and torch.distributed only.
"""
from __future__ import annotations

from dataclasses import dataclass, replace
from typing import Optional, Sequence

import numpy as np
import torch

from . import _native as N

K_LIST = (1, 5, 10, 20, 50)  # utils/eval_reid.py:15


@dataclass
class Planes:
    """Opaque operand buffer of the distance kernel (see ctl_planes_build)."""

    buf: torch.Tensor
    n: int
    d: int
    flags: int
    # rows stored in another order than the caller's (build_planes(order=)): stored row i == caller's row order[i].
    # Results are always reported in the CALLER's indexing (gallery: ctl_pass_desc.g_index_map; queries: un-permuted).
    order: Optional[torch.Tensor] = None        # int32 on the device
    order_host: Optional[np.ndarray] = None

    @property
    def ptr(self):
        return self.buf.data_ptr()


def _flags(dist: str, normalize: bool) -> int:
    if dist not in ("euclidean", "cosine", "euclidean_sqrt"):
        raise KeyError(dist)
    f = N.CTL_DIST_COSINE if dist == "cosine" else N.CTL_DIST_EUCLIDEAN
    if dist == "euclidean_sqrt":
        f |= N.CTL_DIST_SQRT
    if normalize:
        f |= N.CTL_FLAG_NORMALIZE
    return f


def pid_order(pids) -> np.ndarray:
    """Stable order that sorts rows by identity.  With BOTH operands stored in this order almost every 128 x 128 tile
    of the distance GEMM pairs rows of disjoint identity ranges: such a tile holds no positive, so the pass that collects
    the positives (and the top-k threshold, which any subset of the gallery bounds) does not run it
    (ctl_pass_desc.tile_list) -- the results (indices, distances, ranks, AP) are bit-identical to the unsorted run."""
    return np.argsort(np.asarray(pids), kind="stable")


def pid_order_pays(nq: int, ng: int) -> bool:
    """topk_and_eval: identity-ordered planes trade a cheaper pass 1 (tile list: ~30 % of the matrix) for a lumpier pass 2
    (the positives and nearest rows of a query tile sit in a few gallery tiles, and the looser subset threshold lengthens
    the candidate lists); the threshold is where sorting paid off in earlier measurements of this kernel pair and has
    not been re-measured on the H100 build."""
    return int(nq) * int(ng) >= 150_000_000


def build_planes(x: torch.Tensor, dist: str = "euclidean", normalize: bool = False, order=None) -> Planes:
    """`order` (optional, a permutation of the rows, e.g. pid_order(pids)): the planes hold x[order]."""
    N.require_cuda(x)
    if x.dim() != 2:
        raise ValueError(f"expected [n, d] features, got {tuple(x.shape)}")
    x = x.detach().float()
    order_dev = order_host = None
    if order is not None:
        order_host = np.ascontiguousarray(np.asarray(order, dtype=np.int64))
        if order_host.shape != (x.shape[0],):
            raise ValueError("order must be a permutation of the rows")
        o64 = torch.from_numpy(order_host).to(x.device, non_blocking=True)
        x = x.index_select(0, o64)
        order_dev = o64.to(torch.int32)
    x = x.contiguous()
    n, d = x.shape
    flags = _flags(dist, normalize)
    L = N.lib()
    buf = torch.empty(L.ctl_planes_bytes(n, d), dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        N.check(L.ctl_planes_build(x.data_ptr(), n, d, flags, buf.data_ptr(), N.stream_ptr()))
    return Planes(buf, n, d, flags, order_dev, order_host)


class PlaneCache:
    """Operand planes of feature matrices that do not change between evaluations (a fixed gallery of `embeddings.npy`
    searched by many query batches, inference/get_similar.py:104-128; or one validation set evaluated under several
    settings): keyed on the tensor's storage pointer, shape, in-place version counter and the distance flags, so a
    modified tensor is re-packed.  Holds at most `capacity` plane buffers."""

    def __init__(self, capacity: int = 4):
        self.capacity = capacity
        self._items = {}

    def get(self, x: torch.Tensor, dist: str = "euclidean", normalize: bool = False, order=None) -> Planes:
        okey = None if order is None else hash(np.ascontiguousarray(np.asarray(order, dtype=np.int64)).tobytes())
        key = (x.data_ptr(), tuple(x.shape), x._version, str(x.device), dist, normalize, okey)
        p = self._items.get(key)
        if p is None:
            if len(self._items) >= self.capacity:
                self._items.pop(next(iter(self._items)))
            p = self._items[key] = build_planes(x, dist, normalize, order)
        return p


def dist_matrix(x: torch.Tensor, y: torch.Tensor, dist: str = "euclidean", normalize: bool = False) -> torch.Tensor:
    """get_euclidean / get_cosine (utils/reid_metric.py:25-59): the full [m, n] matrix."""
    qp, gp = build_planes(x, dist, normalize), build_planes(y, dist, normalize)
    if qp.d != gp.d:
        raise ValueError("feature dims differ")
    out = torch.empty(qp.n, gp.n, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        N.check(N.lib().ctl_dist_matrix(qp.ptr, qp.n, gp.ptr, gp.n, qp.d, qp.flags, out.data_ptr(), gp.n, N.stream_ptr()))
    return out


def topk(qp: Planes, gp: Planes, k: int, g_index_offset: int = 0, exact_threshold_pass: bool = False):
    """k nearest gallery rows per query in ascending (distance, index) order: the top-k-only passes of _streamed_enqueue,
    enqueued without a read-back.  Results report gallery row + g_index_offset.
    Returns (idx int64 [nq, k], dist float32 [nq, k], overflow flag) on the device.  The threshold pass runs every s-th
    gallery tile only (any subset of the gallery bounds the k-th distance from above; ctl_dist_subset_stride) unless
    `exact_threshold_pass`: identical results, the subset only trades longer candidate lists for ~2/3 of that pass."""
    if qp.order is not None or gp.order is not None:
        raise ValueError("topk() takes planes in the caller's row order (use topk_and_eval for pid-sorted planes)")
    with torch.cuda.device(qp.buf.device):
        out = _streamed_enqueue(ShardExchange(None), qp, gp, None, int(min(k, gp.n)), not exact_threshold_pass,
                                g_index_offset)
    return out["rows"] + (out["ovf"],)


def topk_dense(q: torch.Tensor, g: torch.Tensor, k: int, dist: str = "euclidean", normalize: bool = False,
               chunk_bytes: int = 1 << 30):
    """The k smallest distances per query from MATERIALISED rows of the distance matrix (the reference's own
    dist + argsort + `[:, :topk]`, inference/get_similar.py:104-128), chunked over queries so the matrix slice stays under
    `chunk_bytes`: the general path for every (gallery size, k) the streamed kernel's plan does not cover and for
    degenerate inputs (hundreds of exact ties at the k-th distance).  Same canonical ascending (distance, index) order:
    rows of packed integer keys are sorted."""
    nq, ng = q.shape[0], g.shape[0]
    k = int(min(k, ng))
    gp = build_planes(g, dist, normalize)
    rows = max(1, int(chunk_bytes // (12 * ng)))
    col = torch.arange(ng, device=q.device, dtype=torch.int64)[None, :]
    idx = torch.empty(nq, k, dtype=torch.int64, device=q.device)
    dst = torch.empty(nq, k, dtype=torch.float32, device=q.device)
    flip = -(1 << 63)  # unsigned key order == signed order of key ^ 2^63
    for lo in range(0, nq, rows):
        qp = build_planes(q[lo:lo + rows], dist, normalize)
        d = torch.empty(qp.n, ng, dtype=torch.float32, device=q.device)
        with torch.cuda.device(q.device):
            N.check(N.lib().ctl_dist_matrix(qp.ptr, qp.n, gp.ptr, ng, qp.d, qp.flags, d.data_ptr(), ng, N.stream_ptr()))
        keys = (pack_keys(d, col.expand(qp.n, ng)) ^ flip).topk(k, dim=1, largest=False, sorted=True).values ^ flip
        idx[lo:lo + rows] = keys & 0xFFFFFFFF
        dst[lo:lo + rows] = torch.gather(d, 1, idx[lo:lo + rows])
    return idx, dst


def topk_similar(q: torch.Tensor, g: torch.Tensor, k: int = 100, dist: str = "euclidean", normalize: bool = False):
    """inference/get_similar.py:104-128 without the distance matrix: (indices, distances).  The reference's
    `argsort[:, :topk]` works for every topk; so does this: the streamed two-pass kernel where its plan applies
    (ctl_topk_plan: k <= ceil(ng / 16) merged column groups, candidate capacity <= 16384), otherwise -- and when more rows
    than the candidate capacity tie at the threshold -- the materialised path `topk_dense`."""
    import ctypes as C

    k = int(min(k, g.shape[0]))
    a, b, c, d_ = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    rc = N.lib().ctl_topk_plan(g.shape[0], k, C.byref(a), C.byref(b), C.byref(c), C.byref(d_))
    if rc == 0:
        qp, gp = build_planes(q, dist, normalize), build_planes(g, dist, normalize)
        for exact in (False, True):  # a candidate overflow of the bounded threshold pass: once more with the exact one
            idx, dst, ovf = topk(qp, gp, k, exact_threshold_pass=exact)
            if int(ovf.item()) == 0:
                return idx, dst
    return topk_dense(q, g, k, dist, normalize)


# ----------------------------------------------------------------------------------------
# identities -> dense int32 pids / camera indices / camera bit masks
# ----------------------------------------------------------------------------------------


def encode_identities(q_pids, g_pids, q_camids, g_camids, respect_camids: bool):
    """Host-side re-labelling for the eval kernels (utils/eval_reid.py:52-59): pids -> dense
    int32; cameras -> dense index < 64; gallery cameras -> bit mask (one bit, or -- with
    respect_camids -- the set of cameras a centroid was built from)."""
    q_pids = np.asarray(q_pids)
    g_pids = np.asarray(g_pids)
    uniq, inv = np.unique(np.concatenate([q_pids, g_pids]), return_inverse=True)
    qp = inv[: len(q_pids)].astype(np.int32)
    gp = inv[len(q_pids):].astype(np.int32)
    n_g = len(g_pids)
    if respect_camids:
        q_cam_vals = [c[0] if isinstance(c, (list, tuple, np.ndarray)) else c for c in q_camids]
        g_sets = [list(np.atleast_1d(c)) for c in list(g_camids)[:n_g]]
        cams = sorted(set(q_cam_vals) | {c for s in g_sets for c in s})
        if len(cams) > 64:
            raise NotImplementedError(f"{len(cams)} distinct cameras; the junk filter packs camera sets into 64 bits")
        cam_index = {c: i for i, c in enumerate(cams)}
        qc = np.asarray([cam_index[c] for c in q_cam_vals], dtype=np.int32)
        gm = np.zeros(n_g, dtype=np.uint64)
        for i, s in enumerate(g_sets):
            m = 0
            for c in s:
                m |= 1 << cam_index[c]
            gm[i] = m
    else:
        q_cam = np.asarray(q_camids)
        g_cam = np.asarray(g_camids)[:n_g]  # may be over-long (bases.py:255-260 quirk)
        cams, inv_c = np.unique(np.concatenate([q_cam, g_cam]), return_inverse=True)
        if len(cams) > 64:
            raise NotImplementedError(f"{len(cams)} distinct cameras; the junk filter packs camera sets into 64 bits")
        qc = inv_c[: len(q_cam)].astype(np.int32)
        gm = np.uint64(1) << inv_c[len(q_cam):].astype(np.uint64)
    # upper bound of positives per query: the largest pid group in the gallery
    max_pos = int(np.bincount(gp).max()) if n_g else 1
    return qp, qc, gp, gm, max(1, max_pos)


@dataclass
class EncodedIds:
    """Device-resident identity arrays of one (query set, gallery set): encode once per validation set
    (identities do not change between epochs) and pass as `ids=` to skip the host re-labelling."""

    q_pid: torch.Tensor
    q_cam: torch.Tensor
    g_pid: torch.Tensor
    g_mask: torch.Tensor
    max_pos: int


def encode_ids(q_pids, g_pids, q_camids, g_camids, respect_camids: bool, device, global_labels: bool = False,
               q_order=None, g_order=None) -> EncodedIds:
    """`q_order` / `g_order`: the row orders of the planes these identities go with (Planes.order_host); the inputs are in
    the caller's order."""
    if global_labels:
        arrs = _encode_identities_global(q_pids, g_pids, q_camids, g_camids)
    else:
        arrs = encode_identities(q_pids, g_pids, q_camids, g_camids, respect_camids)
    if q_order is not None:
        arrs = (arrs[0][q_order], arrs[1][q_order]) + tuple(arrs[2:])
    if g_order is not None:
        arrs = tuple(arrs[:2]) + (arrs[2][g_order], arrs[3][g_order], arrs[4])

    def to_dev(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(device, non_blocking=True)

    return EncodedIds(to_dev(arrs[0]), to_dev(arrs[1]), to_dev(arrs[2]), to_dev(arrs[3].view(np.int64)), arrs[4])


class EvalResult:
    """eval_func's outputs (utils/eval_reid.py:86-92).  `cmc`, `mAP`, `all_topk` are reduced from ONE packed read-back
    of (AP, first hit rank, positive count) per query; `single_performance` is assembled and the full `ranks` matrix
    ([nq, max_pos] 1-based kept ranks of every positive, -1 padded) is copied from the device on first access."""

    def __init__(self, cmc, mAP, all_topk, valid_idx, aps, q_pids, ranks_dev):
        self.cmc = cmc                    # float32 [max_rank]
        self.mAP = mAP
        self.all_topk = all_topk          # float64 [5]
        self._valid_idx, self._aps, self._q_pids, self._ranks_dev = valid_idx, aps, q_pids, ranks_dev
        self._ranks = None

    @property
    def single_performance(self) -> np.ndarray:  # [n_valid, 3] (q_idx, q_pid, AP)
        q = self._valid_idx
        return np.column_stack((q.astype(np.float64), np.asarray(self._q_pids)[q].astype(np.float64), self._aps))

    @property
    def ranks(self) -> np.ndarray:
        if self._ranks is None:
            r = self._ranks_dev
            self._ranks = r.cpu().numpy() if torch.is_tensor(r) else np.asarray(r)
        return self._ranks


def _aggregate(ranks, ap: np.ndarray, n_pos: np.ndarray, q_pids, num_g: int, max_rank: int, first=None) -> EvalResult:
    """The reductions at the end of eval_func (utils/eval_reid.py:86-92) from per-query results: O(nq) on the host
    (a histogram of the first-hit ranks gives the whole CMC curve), bit-identical to the reference's float32 / float64
    reductions.  `ranks` may stay on the device (only `first` = ranks[:, 0] is needed here)."""
    max_rank = min(max_rank, num_g)
    valid = n_pos > 0
    if not valid.any():
        raise RuntimeError("no valid query: no query identity appears in the gallery")
    if first is None:
        first = np.asarray(ranks)[:, 0]
    first = first[valid].astype(np.int64)  # ranks are sorted ascending -> the first hit
    num_valid = int(valid.sum())
    hist = np.bincount(np.minimum(first, max_rank + 1), minlength=max_rank + 2)[1: max_rank + 1]
    hits = np.cumsum(hist)                                     # queries whose first hit is at rank <= r
    cmc = hits.astype(np.float32) / np.float32(num_valid)      # float32 sum of 0/1 rows / count, as the reference
    topk = np.asarray([float(hits[k - 1]) if k <= max_rank else float(num_valid) for k in K_LIST]) / float(num_valid)
    aps = ap[valid]
    return EvalResult(cmc, float(np.mean(aps)), topk, np.nonzero(valid)[0], aps, q_pids, ranks)


def _finalize(buckets, count, nq, max_pos, ovf):
    """ctl_eval_finalize_packed (enqueue only): ranks [nq, max_pos] and the packed per-query results [nq + 1, 3] float64
    (AP, first-hit rank, #positives; last row: overflow flag) on the device."""
    dev = buckets.device
    ranks = torch.empty(nq, max_pos, dtype=torch.int32, device=dev)
    ap = torch.empty(nq, dtype=torch.float64, device=dev)
    pack = torch.empty(nq + 1, 3, dtype=torch.float64, device=dev)
    N.check(N.lib().ctl_eval_finalize_packed(buckets.data_ptr(), count.data_ptr(), nq, max_pos, ranks.data_ptr(), ap.data_ptr(),
                                             pack.data_ptr(), ovf.data_ptr(), N.stream_ptr()))
    return ranks, pack


_OVF_POS = "positives list overflowed (max_pos too small)"
_OVF_TOPK = "a device-side list overflowed (exact ties at the k-th distance, or max_pos)"


def _eval_result(ranks, pack, q_pids, num_g: int, max_rank: int, msg: str = _OVF_POS, qp: Optional[Planes] = None,
                 rows=()) -> tuple:
    """The host end of every evaluation, from _finalize's (ranks, pack): ONE device->host copy of `pack` (unless it is
    already a host array), the overflow check, the caller's query order (when `qp` stores its rows in another order;
    `ranks` and the device tensors `rows` are re-ordered) and eval_func's final reductions.  Returns rows + (EvalResult,).
    float64 is exact for the packed integers."""
    h = pack if isinstance(pack, np.ndarray) else pack.cpu().numpy()
    nq = h.shape[0] - 1
    ap, first, cnt = h[:nq, 0], h[:nq, 1].astype(np.int64), h[:nq, 2].astype(np.int32)
    if h[nq, 0]:
        raise OverflowError(msg)
    inv_d, inv_h = _query_inverse(qp) if qp is not None else (None, None)
    if inv_h is not None:  # back to the caller's query order
        rows = tuple(t.index_select(0, inv_d) for t in rows)
        ranks, ap, first, cnt = ranks.index_select(0, inv_d), ap[inv_h], first[inv_h], cnt[inv_h]
    return tuple(rows) + (_aggregate(ranks, ap, cnt, np.asarray(q_pids), num_g, max_rank, first=first),)


def _tile_lists_enabled(qp: Planes, gp: Planes) -> bool:
    """Tile lists (ctl_pass_desc.tile_list) pay off when BOTH operands are stored in identity order (then few tiles can
    hold a positive)."""
    return qp.order is not None and gp.order is not None


def _tile_list(qp: Planes, gp: Planes, ids: "Optional[EncodedIds]", keep_stride: int) -> Optional[torch.Tensor]:
    """ctl_dist_worklist: the tiles that can hold a positive (none when `ids` is None) + every keep_stride-th gallery
    tile for the threshold.  None when the problem is beyond the list builder (the pass then runs every tile)."""
    L = N.lib()
    if ((qp.n + 127) // 128) * ((gp.n + 127) // 128) > (1 << 20) or (qp.n + 127) // 128 + (gp.n + 127) // 128 > 5632:
        return None
    work = torch.empty(L.ctl_dist_worklist_bytes(qp.n, gp.n) // 4, dtype=torch.int32, device=qp.buf.device)
    q_pid, g_pid = (None, None) if ids is None else (ids.q_pid, ids.g_pid)
    N.check(L.ctl_dist_worklist(N.ptr(q_pid), qp.n, N.ptr(g_pid), gp.n, int(keep_stride), work.data_ptr(), N.stream_ptr()))
    return work


def _g_index_map(gp: Planes, g_index_offset: int) -> Optional[torch.Tensor]:
    """int32 map stored gallery row -> index reported in the results (None: row + g_index_offset)."""
    if gp.order is None:
        return None
    if g_index_offset + gp.n >= (1 << 31):
        raise NotImplementedError("re-ordered gallery planes report int32 indices")
    return gp.order if g_index_offset == 0 else (gp.order + int(g_index_offset)).to(torch.int32)


def _query_inverse(qp: Planes):
    """(device int64, host) inverse of the query row order: results[inv] are in the caller's order."""
    if qp.order is None:
        return None, None
    inv = getattr(qp, "_inv", None)
    if inv is None:
        inv_h = np.empty(qp.n, dtype=np.int64)
        inv_h[qp.order_host] = np.arange(qp.n)
        inv = qp._inv = (torch.from_numpy(inv_h).to(qp.buf.device), inv_h)
    return inv


def evaluate_streamed(
    qp: Planes,
    gp: Planes,
    q_pids,
    g_pids,
    q_camids,
    g_camids,
    max_rank: int = 50,
    respect_camids: bool = False,
    g_index_offset: int = 0,
    group=None,
    total_gallery: Optional[int] = None,
    ids: "Optional[EncodedIds]" = None,
) -> EvalResult:
    """eval_func semantics (utils/eval_reid.py:25-92) straight from the features: two tensor-
    core passes (collect the positives' distances; count kept rows before each positive),
    no distance matrix, no argsort.  With `group` (torch.distributed), `gp` is this rank's
    gallery shard and g_* its identities, and the passes exchange as topk_and_eval_sharded's do.  The merged threshold
    list then holds world x (the largest per-shard max_pos of any rank, MAX-reduced here even when `ids` is given), so
    the `ranks` matrix may carry more -1 padding columns than an unsharded run's; every column up to a query's positive
    count is the same.
    Identities are given in the caller's row order even when the planes were built with `order=`; a precomputed `ids`
    must have been encoded with the planes' orders (encode_ids(q_order=, g_order=))."""
    ex = ShardExchange(group)
    dev = qp.buf.device
    if ids is None:
        if ex.world > 1 and not np.issubdtype(np.asarray(q_pids).dtype, np.integer):
            raise ValueError("sharded evaluation needs integer pids")
        # sharded: dense re-labelling must agree across ranks -> identity map instead of np.unique
        ids = encode_ids(q_pids, g_pids, q_camids, g_camids, respect_camids, dev, global_labels=ex.world > 1,
                         q_order=qp.order_host, g_order=gp.order_host)
    if ex.world > 1:
        ids = replace(ids, max_pos=_max_over_ranks(ex, ids.max_pos, dev))
    num_g = total_gallery if total_gallery is not None else gp.n
    return _streamed(ex, qp, gp, ids, None, q_pids, num_g, max_rank, g_index_offset)[0]


def _encode_identities_global(q_pids, g_pids, q_camids, g_camids):
    q_pid = np.asarray(q_pids).astype(np.int32)
    g_pid = np.asarray(g_pids).astype(np.int32)
    q_cam = np.asarray(q_camids).astype(np.int32)
    g_cam = np.asarray(g_camids).astype(np.int64)[: len(g_pid)]
    if q_cam.max(initial=0) >= 64 or g_cam.max(initial=0) >= 64 or min(q_cam.min(initial=0), g_cam.min(initial=0)) < 0:
        raise NotImplementedError("sharded evaluation expects camera ids in [0, 64)")
    g_mask = (np.uint64(1) << g_cam.astype(np.uint64)).astype(np.uint64)
    max_pos = int(np.bincount(g_pid - g_pid.min()).max()) if len(g_pid) else 1
    return q_pid, q_cam, g_pid, g_mask, max(1, max_pos)


def pack_keys(dst: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """(distance fp32, index) -> the kernels' uint64 key (carried as int64): orderable(fp32) << 32 | index, whose
    UNSIGNED integer order is the canonical ascending (distance, index) order (ctl_key_encode)."""
    b = dst.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    o = torch.where(b >= 0x80000000, b ^ 0xFFFFFFFF, b | 0x80000000)  # sign-magnitude float bits -> unsigned order
    return (o << 32) | (idx.to(torch.int64) & 0xFFFFFFFF)


def merge_topk_keys(keys: torch.Tensor, k: int):
    """keys: int64 [nq, m] packed (distance, index) keys in any order (m >= k) -> the k smallest per row as
    (idx int64 [nq, k], dist float32 [nq, k]): ctl_sort_key_rows + ctl_topk_emit."""
    L = N.lib()
    keys = keys.contiguous()
    nq, m = keys.shape
    dev = keys.device
    counts = torch.full((nq,), m, dtype=torch.int32, device=dev)
    idx = torch.empty(nq, k, dtype=torch.int64, device=dev)
    dst = torch.empty(nq, k, dtype=torch.float32, device=dev)
    ovf = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        N.check(L.ctl_sort_key_rows(keys.data_ptr(), counts.data_ptr(), nq, m, N.stream_ptr()))
        N.check(L.ctl_topk_emit(keys.data_ptr(), counts.data_ptr(), nq, m, k, idx.data_ptr(), dst.data_ptr(),
                                ovf.data_ptr(), N.stream_ptr()))
    return idx, dst


def topk_sharded(q_local: torch.Tensor, g_local: torch.Tensor, k: int, g_index_offset: int, group,
                 dist: str = "euclidean", normalize: bool = False):
    """BASELINE config 5: queries sharded by rank (the same number on every rank) are all-gathered once, the gallery
    stays sharded; every rank returns the merged global top-k of ALL queries -- the top-k-only passes of
    _streamed_enqueue, whose exchange merges every rank's k best keys.  `group=None` is torch.distributed's default
    group."""
    ex = ShardExchange.default() if group is None else ShardExchange(group)
    q = ex.rows(q_local, [q_local.shape[0]] * ex.world)
    qp, gp = build_planes(q, dist, normalize), build_planes(g_local, dist, normalize)
    return _streamed(ex, qp, gp, None, k, None, gp.n, 0, g_index_offset, tile_lists=True)


def topk_and_eval(qp: Planes, gp: Planes, k: int, q_pids, g_pids, q_camids, g_camids, max_rank: int = 50,
                  respect_camids: bool = False, ids: "Optional[EncodedIds]" = None, tile_lists: Optional[bool] = None):
    """BASELINE config 3 in TWO tensor-core passes: per-query top-k (ascending (distance, index))
    AND eval_func's CMC / mAP, neither materialising the distance matrix.
      pass 1: 16-column group minima (-> tau) + the positives' distances
      pass 2: candidates <= tau + kept rows before each positive
    Pass 1 does not need the whole matrix: the positives sit in the tiles whose query / gallery identity ranges
    intersect, and the k-th smallest group minimum of ANY subset of the gallery bounds the k-th distance from above.
    With both operands stored in pid order (build_planes(order=pid_order(pids))) pass 1 therefore runs a tile list
    (ctl_dist_worklist: the few tiles that can hold a positive + every s-th gallery tile, ~30 % of the matrix); the
    looser tau only lengthens the candidate lists of the exact pass 2, so indices, distances, ranks and AP are
    bit-identical to the full run (`tile_lists=False`).
    Identities are given in the caller's row order; a precomputed `ids` must carry the planes' orders
    (encode_ids(q_order=qp.order_host, g_order=gp.order_host)).
    Returns (idx [nq,k] int64, dist [nq,k] float32 on the device, EvalResult), all in the caller's indexing."""
    if ids is None:
        ids = encode_ids(q_pids, g_pids, q_camids, g_camids, respect_camids, qp.buf.device, q_order=qp.order_host,
                         g_order=gp.order_host)
    return _streamed(ShardExchange(None), qp, gp, ids, k, q_pids, gp.n, max_rank, 0, tile_lists)


class ShardExchange:
    """The exchanges of the sharded paths (the streamed passes of topk_sharded / evaluate_streamed /
    topk_and_eval_sharded and the row-blocked re-ranking), over the ranks of a torch.distributed group (None: one rank,
    nothing is exchanged).  Every rank calls each method in the same order.  Tests substitute stand-ins with the same
    methods."""

    def __init__(self, group=None):
        import torch.distributed as dist

        self.dist, self.group = dist, group
        self.world = 1 if group is None else dist.get_world_size(group)
        self.rank = 0 if group is None else dist.get_rank(group)

    @classmethod
    def default(cls) -> "ShardExchange":
        """The ranks of torch.distributed's default group (the meaning torch.distributed gives `group=None`)."""
        import torch.distributed as dist

        if not dist.is_initialized():
            raise ValueError("torch.distributed's default process group has not been initialized")
        return cls(dist.group.WORLD)

    def objects(self, obj) -> list:
        """Every rank's picklable `obj`, in rank order."""
        if self.group is None:
            return [obj]
        out = [None] * self.world
        self.dist.all_gather_object(out, obj, group=self.group)
        return out

    def rows(self, t: torch.Tensor, counts: Sequence[int]) -> torch.Tensor:
        """The concatenation over ranks of each rank's `t` (counts[j] rows on rank j): one all-gather, of shards padded
        to the largest when the counts differ, then trimmed."""
        if self.group is None:
            return t
        m = max(counts)
        even = all(c == m for c in counts)
        part = t.contiguous()
        if not even:
            part = t.new_zeros((m,) + tuple(t.shape[1:]))
            part[: t.shape[0]] = t
        out = t.new_empty((self.world * m,) + tuple(t.shape[1:]))
        self.dist.all_gather_into_tensor(out, part, group=self.group)
        if even:
            return out
        return torch.cat([out[j * m: j * m + c] for j, c in enumerate(counts)])

    def max_(self, t: torch.Tensor) -> torch.Tensor:
        """In place: the element-wise maximum over ranks."""
        if self.group is not None:
            self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX, group=self.group)
        return t

    def sum_(self, t: torch.Tensor) -> torch.Tensor:
        """In place: the element-wise sum over ranks."""
        if self.group is not None:
            self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM, group=self.group)
        return t


def _max_over_ranks(ex, v: int, device) -> int:
    return int(ex.max_(torch.tensor([v], device=device, dtype=torch.int64)).item())


def _gather_keys(ex, pos_keys: torch.Tensor, pos_count: torch.Tensor):
    """Exchange 1 of the sharded passes, up to the row sort: every rank's positives' keys of a query side by side in rank
    order, [nq, world * max_pos], with unused slots set to the largest key so that ONE sort of the whole row packs and
    orders them (ctl_sort_key_rows); and the total count per query."""
    nq, mp_l = pos_keys.shape
    col = torch.arange(mp_l, device=pos_keys.device)[None, :]
    masked = torch.where(col < pos_count[:, None].clamp(max=mp_l), pos_keys, torch.full_like(pos_keys, -1))
    keys = ex.rows(masked, [nq] * ex.world).view(ex.world, nq, mp_l).permute(1, 0, 2).reshape(nq, ex.world * mp_l)
    count = ex.rows(pos_count.contiguous(), [nq] * ex.world).view(ex.world, nq).sum(0, dtype=torch.int32)
    return keys, count


def _streamed_enqueue(ex, qp: Planes, gp: Planes, ids: "Optional[EncodedIds]", k: Optional[int], tile_lists: bool,
                      g_index_offset: int = 0) -> dict:
    """The launch sequence of the streamed passes over this rank's gallery `gp` (the whole gallery at world 1), with the
    exchanges of `ex` (ShardExchange or a stand-in) between them:
      pass 1: the positives' keys (+ the 16-column group minima -> tau)
      exchange 1 (world > 1): every rank's positives (_gather_keys); then one row sort gives the threshold list
      pass 2: kept rows before each positive (+ the candidates <= tau, sorted)
      exchange 2 (world > 1): sum of the bucket counts, MAX of the overflow flag, every rank's k best keys merged by
                              integer key order; at world 1 the top-k is emitted from the candidates
      finalize
    k=None evaluates only: no minima, threshold or candidates.  ids=None is the top-k only: no positives, counts or
    finalize, and no pass 1 for a small gallery (tau = +inf).  `tile_lists`: pass 1 runs a tile list (topk_and_eval; with
    ids=None the list of every s-th gallery tile, ctl_dist_subset_stride, for a threshold from a subset of the gallery).
    At world 1 nothing is exchanged and nothing waits for the host (capturable in a CUDA graph).  Returns the device
    tensors {rows: (idx, dst) or (), ovf, ranks, pack} in the planes' query order; no ranks or pack with ids=None."""
    import ctypes as C

    L = N.lib()
    dev = qp.buf.device
    nq, ng, world = qp.n, gp.n, ex.world
    if ids is not None:
        mp_l = ids.max_pos  # capacity of one rank's positives (the same on every rank)
        mp = mp_l * world   # capacity of the merged threshold list
    i32 = dict(dtype=torch.int32, device=dev)
    s = N.stream_ptr
    keep = []
    if k is None:
        emit_all = True
        pos_keys = torch.zeros(nq, mp_l, dtype=torch.int64, device=dev)
        pos_count, ovf = torch.zeros(nq, **i32), torch.zeros(1, **i32)
        buckets = None
    else:
        k_loc = int(min(k, ng))
        plan = [C.c_int32() for _ in range(4)]
        N.check(L.ctl_topk_plan(ng, k_loc, *[C.byref(x) for x in plan]))
        emit_all, n_groups, merge, cap = [x.value for x in plan]
        gmin = torch.empty(nq, n_groups, dtype=torch.float32, device=dev)
        tau = torch.empty(nq, dtype=torch.float32, device=dev)
        cand = torch.empty(nq, cap, dtype=torch.int64, device=dev)
        zeros = torch.zeros(2 * nq + 1, **i32)
        cand_count, pos_count, ovf = zeros[:nq], zeros[nq: 2 * nq], zeros[2 * nq:]
        keep += [gmin, tau, cand, zeros]
        if ids is not None:
            pos_keys = torch.empty(nq, mp_l, dtype=torch.int64, device=dev)
            buckets = torch.zeros(nq, mp + 1, **i32)
    gmap = _g_index_map(gp, g_index_offset)  # keys carry the caller's gallery row (sharded: the GLOBAL row)
    idp = dict(overflow=ovf.data_ptr(), g_index_offset=g_index_offset, g_index_map=N.ptr(gmap))
    p1 = N.PassDesc()
    if ids is not None:
        idp.update(q_pid=ids.q_pid.data_ptr(), q_cam=ids.q_cam.data_ptr(), g_pid=ids.g_pid.data_ptr(),
                   g_cammask=ids.g_mask.data_ptr())
        p1 = N.PassDesc(pos_keys=pos_keys.data_ptr(), pos_count=pos_count.data_ptr(), max_pos=mp_l, **idp)
    if not emit_all:
        p1.gmin = gmin.data_ptr()
    work = None
    if tile_lists:  # (no threshold, or tau = +inf for a small gallery: stride 0, just the tiles that can hold a positive)
        stride = 0 if emit_all else L.ctl_dist_subset_stride(ng, k_loc)
        if stride > 1 or (emit_all and ids is not None):
            work = _tile_list(qp, gp, ids, stride)
    if work is not None:
        p1.tile_list = work.data_ptr()
        if not emit_all:
            N.check(L.ctl_fill_f32(gmin.data_ptr(), gmin.numel(), float("inf"), s()))  # groups of tiles not run
    if ids is not None or not emit_all:
        N.check(L.ctl_dist_pass(qp.ptr, nq, gp.ptr, ng, qp.d, qp.flags, C.byref(p1), s()))
    if k is not None and emit_all:
        N.check(L.ctl_fill_f32(tau.data_ptr(), nq, float("inf"), s()))
    elif k is not None:
        N.check(L.ctl_select_tau(gmin.data_ptr(), nq, n_groups, merge, k_loc, tau.data_ptr(), s()))
    if ids is None:
        p2 = N.PassDesc(**idp)
    else:
        thr, thr_count, sort_count = pos_keys, pos_count, pos_count
        if world > 1:
            thr, thr_count = _gather_keys(ex, pos_keys, pos_count)
            sort_count = torch.full((nq,), mp, **i32)
        N.check(L.ctl_sort_key_rows(thr.data_ptr(), sort_count.data_ptr(), nq, mp, s()))
        if buckets is None:
            buckets = torch.zeros(nq, mp + 1, **i32)
        p2 = N.PassDesc(thr_keys=thr.data_ptr(), thr_count=thr_count.data_ptr(), buckets=buckets.data_ptr(), max_pos=mp,
                        **idp)
        keep += [pos_keys, thr, sort_count, buckets]
    if k is not None:
        p2.tau, p2.cand_keys, p2.cand_count, p2.cand_cap = tau.data_ptr(), cand.data_ptr(), cand_count.data_ptr(), cap
    N.check(L.ctl_dist_pass(qp.ptr, nq, gp.ptr, ng, qp.d, qp.flags, C.byref(p2), s()))
    rows = ()
    if k is not None:
        N.check(L.ctl_sort_key_rows(cand.data_ptr(), cand_count.data_ptr(), nq, cap, s()))
    if world > 1:
        if ids is not None:
            ex.sum_(buckets)
        ex.max_(ovf)
        if k is not None:
            best = ex.rows(cand[:, :k_loc].contiguous(), [nq] * world)
            rows = merge_topk_keys(best.view(world, nq, k_loc).permute(1, 0, 2).reshape(nq, world * k_loc),
                                   int(min(k, world * k_loc)))
    elif k is not None:
        idx = torch.empty(nq, k_loc, dtype=torch.int64, device=dev)
        dst = torch.empty(nq, k_loc, dtype=torch.float32, device=dev)
        N.check(L.ctl_topk_emit(cand.data_ptr(), cand_count.data_ptr(), nq, cap, k_loc, idx.data_ptr(), dst.data_ptr(),
                                ovf.data_ptr(), s()))
        rows = (idx, dst)
    out = {"rows": rows, "ovf": ovf, "keep": keep + [work, gmap]}
    if ids is not None:
        out["ranks"], out["pack"] = _finalize(buckets, thr_count, nq, mp, ovf)
    return out


def _streamed(ex, qp: Planes, gp: Planes, ids: "Optional[EncodedIds]", k: Optional[int], q_pids, num_g: int,
              max_rank: int, g_index_offset: int = 0, tile_lists: Optional[bool] = None) -> tuple:
    """_streamed_enqueue, ONE read-back and _eval_result: (idx, dist, EvalResult) in the caller's query order, or
    (EvalResult,) when k is None, or (idx, dist) when ids is None (the top-k only, whose read-back is the overflow flag:
    OverflowError when it is set).  `tile_lists` defaults to both planes being stored in identity order.  When the looser
    threshold of a tile-list pass 1 lets more rows through than a candidate list holds, an evaluation runs once more with
    the threshold from every tile; the overflow flag is MAX-reduced and `tile_lists` is the caller's, so every rank
    retries together."""
    if tile_lists is None:
        tile_lists = _tile_lists_enabled(qp, gp)
    with torch.cuda.device(qp.buf.device):
        out = _streamed_enqueue(ex, qp, gp, ids, k, tile_lists, g_index_offset)
        if ids is None:
            if int(out["ovf"].item()):
                raise OverflowError("top-k candidate capacity exceeded on some rank")
            return out["rows"]
        h = out["pack"].cpu().numpy()
        if h[qp.n, 0] and tile_lists and k is not None:
            return _streamed(ex, qp, gp, ids, k, q_pids, num_g, max_rank, g_index_offset, tile_lists=False)
        msg = (_OVF_POS if k is None else _OVF_TOPK) + (" on some rank" if ex.world > 1 else "")
        return _eval_result(out["ranks"], h, q_pids, num_g, max_rank, msg, qp, out["rows"])


class TopkEvalSession:
    """topk_and_eval for ONE validation set evaluated again and again (a resident gallery searched by successive query
    batches, inference/get_similar.py:104-128; the per-epoch validation of train_ctl_model.py): the ~12 launches of the step
    (query planes, both tensor-core passes, selection, sorts, emit, finalize, the packed device->host copy) are captured
    ONCE in a CUDA graph over static buffers and replayed -- no per-step allocation, descriptor encoding or launch gaps.
    Results are those of topk_and_eval, bit for bit (tests/test_retrieval_gpu.py)."""

    def __init__(self, gallery: torch.Tensor, num_query: int, k: int, q_pids, g_pids, q_camids, g_camids, max_rank: int = 50,
                 respect_camids: bool = False, dist: str = "euclidean", normalize: bool = False):
        N.require_cuda(gallery)
        dev = gallery.device
        self.dev, self.k, self.max_rank, self.q_pids = dev, int(k), max_rank, q_pids
        self.gp = build_planes(gallery, dist, normalize)
        self.ids = encode_ids(q_pids, g_pids, q_camids, g_camids, respect_camids, dev)
        self.q = torch.empty(num_query, gallery.shape[1], dtype=torch.float32, device=dev)  # static input of the graph
        self.host = torch.empty(num_query + 1, 3, dtype=torch.float64).pin_memory()
        self.done = torch.cuda.Event()
        one = ShardExchange(None)

        def enqueue():
            qp = build_planes(self.q, dist, normalize)
            out = _streamed_enqueue(one, qp, self.gp, self.ids, self.k, False)
            self.host.copy_(out["pack"], non_blocking=True)
            out["qp"] = qp
            return out

        with torch.cuda.device(dev):
            cur = torch.cuda.current_stream(dev)
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(cur)
            with torch.cuda.stream(side):  # eager warm-up: function attributes, allocator pools
                self.q.zero_()
                for _ in range(2):
                    enqueue()
            cur.wait_stream(side)
            torch.cuda.synchronize(dev)
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self.out = enqueue()

    def __call__(self, q: torch.Tensor):
        """q: [num_query, d] features on the device -> (idx, dist, EvalResult) like topk_and_eval.  The returned device
        tensors are the graph's static outputs: valid until the next call."""
        N.require_cuda(q)
        with torch.cuda.device(self.dev):
            self.q.copy_(q, non_blocking=True)
            self.graph.replay()
            self.done.record()
            self.done.synchronize()
        out = self.out
        return _eval_result(out["ranks"], self.host.numpy(), self.q_pids, self.gp.n, self.max_rank, _OVF_TOPK, out["qp"],
                            out["rows"])


def encode_ids_sharded(q_pids, g_pids_local, q_camids, g_camids_local, device, group, q_order=None,
                       g_order=None) -> EncodedIds:
    """Identity arrays of (all queries, THIS rank's gallery shard) for topk_and_eval_sharded: raw integer pids (every
    rank must agree on the labelling, so no np.unique), camera ids in [0, 64); `max_pos` = the largest number of
    same-pid rows of any shard (one MAX all-reduce, done once per validation set)."""
    ids = encode_ids(q_pids, g_pids_local, q_camids, g_camids_local, False, device, global_labels=True, q_order=q_order,
                     g_order=g_order)
    ids.max_pos = _max_over_ranks(ShardExchange(group), ids.max_pos, device)
    return ids


def topk_and_eval_sharded(qp: Planes, gp_local: Planes, k: int, ids: EncodedIds, q_pids, g_index_offset: int,
                          total_gallery: int, group, max_rank: int = 50, tile_lists: Optional[bool] = None):
    """BASELINE config 5: topk_and_eval with the GALLERY AXIS SHARDED over the ranks of `group` (queries replicated:
    all-gather them once before building `qp`).  Every rank runs the two tensor-core passes over its own shard, with
    the exchanges of _streamed_enqueue between them (utils/reid_metric.py:112-136 + utils/eval_reid.py:25-92 semantics,
    bit-identical to one GPU):
      after pass 1: all-gather of the positives' (distance, index) keys [nq, max_pos] -> one sorted threshold list
      after pass 2: all-reduce(sum) of the integer bucket counts; all-gather of each rank's k best packed keys and a
                    k-way merge by integer key order (world-size independent).
    `ids` comes from encode_ids_sharded, so max_pos is the same on every rank; every shard must hold at least k rows.
    Returns (idx [nq, k] global gallery rows, dist [nq, k], EvalResult) on every rank."""
    return _streamed(ShardExchange(group), qp, gp_local, ids, k, q_pids, total_gallery, max_rank, g_index_offset,
                     tile_lists)


# ----------------------------------------------------------------------------------------
# CMC / mAP from a materialised matrix; k-reciprocal re-ranking
# ----------------------------------------------------------------------------------------


def evaluate_matrix(distmat: torch.Tensor, q_pids, g_pids, q_camids, g_camids, max_rank: int = 50,
                    respect_camids: bool = False) -> EvalResult:
    """eval_func semantics (utils/eval_reid.py:25-92) for a [nq, ng] fp32 distance matrix already on the device (re-ranked
    distances, or any distance the caller computed): the collect and count passes of evaluate_streamed read the matrix
    instead of forming it (ctl_eval_matrix_collect / _count), then the same row sort, finalize and ONE packed read-back.
    Ties are ordered by gallery index, as everywhere in this package."""
    N.require_cuda(distmat)
    if distmat.dim() != 2 or distmat.dtype != torch.float32 or distmat.stride(1) != 1:
        raise ValueError("expected a [nq, ng] float32 matrix with unit column stride")
    dev = distmat.device
    nq, ng = distmat.shape
    ev = _eval_buffers(encode_ids(q_pids, g_pids, q_camids, g_camids, respect_camids, dev), nq, dev)
    with torch.cuda.device(dev):
        _eval_matrix_rows(distmat, 0, nq, ng, distmat.stride(0), ev)
        ranks, pack = _finalize(ev["buckets"], ev["pos_count"], nq, ev["ids"].max_pos, ev["ovf"])
        return _eval_result(ranks, pack, q_pids, ng, max_rank)[0]


def _eval_buffers(ids: "EncodedIds", nq: int, dev) -> dict:
    """The zeroed buffers of the collect / sort / count steps over a materialised matrix (_eval_matrix_rows,
    ctl_rerank_topk)."""
    pos_keys = torch.zeros(nq, ids.max_pos, dtype=torch.int64, device=dev)
    zeros = torch.zeros(nq + 1, dtype=torch.int32, device=dev)
    return {"ids": ids, "pos_keys": pos_keys, "pos_count": zeros[:nq], "ovf": zeros[nq:],
            "buckets": torch.zeros(nq, ids.max_pos + 1, dtype=torch.int32, device=dev)}


def _eval_matrix_rows(d: torch.Tensor, q0: int, rows: int, ng: int, ld: int, ev: dict):
    """The collect, row sort and count of eval_func over the distances `d` ([rows, ng], row stride ld) of queries
    [q0, q0 + rows), into the rows of `ev` (_eval_buffers over all queries)."""
    L = N.lib()
    s = N.stream_ptr()
    ids, mp = ev["ids"], ev["ids"].max_pos
    idp = (ids.q_pid.data_ptr() + 4 * q0, ids.q_cam.data_ptr() + 4 * q0, ids.g_pid.data_ptr(), ids.g_mask.data_ptr(), mp)
    pk, pc = ev["pos_keys"][q0:].data_ptr(), ev["pos_count"][q0:].data_ptr()
    N.check(L.ctl_eval_matrix_collect(d.data_ptr(), rows, ng, ld, *idp, pk, pc, ev["ovf"].data_ptr(), s))
    N.check(L.ctl_sort_key_rows(pk, pc, rows, mp, s))
    N.check(L.ctl_eval_matrix_count(d.data_ptr(), rows, ng, ld, *idp, pk, pc, ev["buckets"][q0:].data_ptr(), s))


@dataclass
class RerankPlan:
    """ctl_rerank_plan: rank columns kept (kr = max(k1 + 1, k2)), h = round-half-even(k1 / 2), and the row capacities
    of V (v_cap = (k1 + 1)(h + 2)) and of the query-expanded V (q_cap = k2 v_cap, or v_cap when k2 = 1)."""

    kr: int
    h: int
    v_cap: int
    q_cap: int


def rerank_plan(nq: int, ng: int, k1: int, k2: int) -> RerankPlan:
    import ctypes as C

    v = [C.c_int32() for _ in range(4)]
    N.check(N.lib().ctl_rerank_plan(int(nq), int(ng), int(k1), int(k2), *[C.byref(x) for x in v]))
    return RerankPlan(*[x.value for x in v])


def _rerank_inputs(q: torch.Tensor, g: torch.Tensor, normalize: bool):
    N.require_cuda(q, g)
    if q.dim() != 2 or g.dim() != 2 or q.shape[1] != g.shape[1]:
        raise ValueError(f"expected [Q, d] and [G, d] features, got {tuple(q.shape)} and {tuple(g.shape)}")
    return build_planes(torch.cat([q.detach().float(), g.detach().float().to(q.device)]), "euclidean", normalize)


def _rerank_enqueue(planes: Planes, nq: int, ng: int, k1: int, k2: int, lambda_value: float, out: torch.Tensor,
                    status: torch.Tensor, ws: torch.Tensor):
    """ctl_rerank (enqueue only, capturable in a CUDA graph)."""
    N.check(N.lib().ctl_rerank(planes.ptr, nq, ng, planes.d, planes.flags, int(k1), int(k2), float(lambda_value),
                               out.data_ptr(), out.stride(0), status.data_ptr(), ws.data_ptr(), ws.numel(),
                               N.stream_ptr()))


def rerank(q: torch.Tensor, g: torch.Tensor, k1: int = 20, k2: int = 6, lambda_value: float = 0.3,
           normalize: bool = False) -> torch.Tensor:
    """k-reciprocal re-ranking (Zhong et al., CVPR 2017) of queries q [Q, d] against gallery g [G, d]: the [Q, G] float32
    re-ranked distance matrix on the device (re_ranking(probFea, galFea, k1, k2, lambda_value) of the reid-strong-baseline
    lineage; semantics in include/ctl_b200.h).  `normalize`: L2-normalise the features first (TEST.FEAT_NORM).
    Differences from that function: V, the query expansion and the Jaccard sums are float32 instead of float16, and the
    neighbour lists order equal distances by column index (np.argsort's default quicksort leaves their order
    unspecified).  Needs N = Q + G rows of N^2 * 4 bytes of workspace (1.5 GB at Market-1501 size).  Raises ValueError
    when a row of the distance matrix has no positive maximum (N = 1, or all features identical)."""
    planes = _rerank_inputs(q, g, normalize)
    nq, ng = q.shape[0], g.shape[0]
    L = N.lib()
    ws_bytes = L.ctl_rerank_workspace_bytes(nq, ng, int(k1), int(k2))
    if ws_bytes == 0:
        rerank_plan(nq, ng, k1, k2)  # raises with the reason
    dev = q.device
    out = torch.empty(nq, ng, dtype=torch.float32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _rerank_enqueue(planes, nq, ng, k1, k2, lambda_value, out, status, ws)
        _check_status(status)
    return out


def _check_status(status: torch.Tensor):
    if int(status.item()):
        raise ValueError("re-ranking: a row of the distance matrix has no positive maximum (N = 1 or identical features)")


def rerank_stages(q: torch.Tensor, g: torch.Tensor, k1: int = 20, k2: int = 6, lambda_value: float = 0.3,
                  normalize: bool = False) -> dict:
    """rerank() one stage entry point at a time, every stage reading the previous stage's device output, with every
    intermediate kept: {nd [N, N], rank [N, kr], v_idx / v_val [N, v_cap], v_cnt, q_idx / q_val / q_cnt (the expanded
    V; the same tensors as v_* when k2 = 1), col_ptr, inv_row, inv_val, out [Q, G], status, plan}.  For tests and
    inspection: it holds every buffer at once."""
    planes = _rerank_inputs(q, g, normalize)
    nq, ng = q.shape[0], g.shape[0]
    n = nq + ng
    pl = rerank_plan(nq, ng, k1, k2)
    L = N.lib()
    dev = q.device
    i32, f32 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.float32, device=dev)
    r = {"plan": pl, "nd": torch.empty(n, n, **f32), "rank": torch.empty(n, pl.kr, **i32),
         "status": torch.zeros(1, **i32), "v_idx": torch.full((n, pl.v_cap), -1, **i32),
         "v_val": torch.zeros(n, pl.v_cap, **f32), "v_cnt": torch.zeros(n, **i32)}
    if k2 > 1:
        r.update(q_idx=torch.full((n, pl.q_cap), -1, **i32), q_val=torch.zeros(n, pl.q_cap, **f32),
                 q_cnt=torch.zeros(n, **i32))
    else:
        r.update(q_idx=r["v_idx"], q_val=r["v_val"], q_cnt=r["v_cnt"])
    cap = r["q_idx"].shape[1]
    r.update(col_ptr=torch.empty(n + 1, **i32), inv_row=torch.full((ng * cap,), -1, **i32),
             inv_val=torch.zeros(ng * cap, **f32), out=torch.empty(nq, ng, **f32))
    cursor = torch.empty(n, **i32)
    with torch.cuda.device(dev):
        s = N.stream_ptr()
        N.check(L.ctl_dist_matrix(planes.ptr, n, planes.ptr, n, planes.d, planes.flags, r["nd"].data_ptr(), n, s))
        N.check(L.ctl_rerank_rank(r["nd"].data_ptr(), n, n, pl.kr, r["rank"].data_ptr(), r["status"].data_ptr(), s))
        N.check(L.ctl_rerank_expand(r["nd"].data_ptr(), n, n, r["rank"].data_ptr(), k1, k2, r["v_idx"].data_ptr(),
                                    r["v_val"].data_ptr(), r["v_cnt"].data_ptr(), s))
        if k2 > 1:
            N.check(L.ctl_rerank_qe(r["rank"].data_ptr(), n, k1, k2, r["v_idx"].data_ptr(), r["v_val"].data_ptr(),
                                    r["v_cnt"].data_ptr(), r["q_idx"].data_ptr(), r["q_val"].data_ptr(),
                                    r["q_cnt"].data_ptr(), s))
        N.check(L.ctl_rerank_invert(nq, ng, r["q_idx"].data_ptr(), r["q_val"].data_ptr(), r["q_cnt"].data_ptr(), cap,
                                    r["col_ptr"].data_ptr(), cursor.data_ptr(), r["inv_row"].data_ptr(),
                                    r["inv_val"].data_ptr(), s))
        N.check(L.ctl_rerank_jaccard(nq, ng, r["q_idx"].data_ptr(), r["q_val"].data_ptr(), r["q_cnt"].data_ptr(), cap,
                                     r["col_ptr"].data_ptr(), r["inv_row"].data_ptr(), r["inv_val"].data_ptr(),
                                     r["nd"].data_ptr(), n, float(lambda_value), r["out"].data_ptr(), ng, s))
    return r


# ----------------------------------------------------------------------------------------
# row-blocked re-ranking: galleries beyond the N^2 bound
# ----------------------------------------------------------------------------------------

RERANK_BLOCK_BYTES = 2 << 30  # default size of the [block_rows, N] fp32 slice of the distance matrix


def rerank_block_rows(nq: int, ng: int, budget: int = RERANK_BLOCK_BYTES) -> int:
    """The default block of rerank_topk: the largest multiple of 128 rows whose [R, N] fp32 block fits in `budget`
    bytes (fewer rows, at least 1, when not even 128 fit), and never more than N = nq + ng."""
    n = int(nq) + int(ng)
    rows = int(budget) // (4 * n)
    r = rows // 128 * 128 if rows >= 128 else max(1, rows)
    return int(min(r, n))


def rerank_fits_dense(nq: int, ng: int, k1: int, k2: int, free_bytes: int) -> bool:
    """Which re-ranking eval_reranked runs: the dense ctl_rerank (plus its [Q, G] result) when its workspace and output
    fit in `free_bytes` of device memory, otherwise the row-blocked ctl_rerank_topk (bit-identical results, workspace
    linear in N).  Host-only."""
    ws = N.lib().ctl_rerank_workspace_bytes(int(nq), int(ng), int(k1), int(k2))
    return ws > 0 and ws + 4 * int(nq) * int(ng) <= int(free_bytes)


def rerank_topk_workspace_bytes(nq: int, ng: int, d: int, k1: int, k2: int, k: int, block_rows: int) -> int:
    """ctl_rerank_topk_workspace_bytes (host-only; 0 for unsupported arguments)."""
    return int(N.lib().ctl_rerank_topk_workspace_bytes(int(nq), int(ng), int(d), int(k1), int(k2), int(k),
                                                        int(block_rows)))


def _rerank_topk_args(nq, ng, d, k1, k2, k, block_rows):
    """validated (k, block_rows, workspace bytes); raises with the library's reason."""
    block_rows = rerank_block_rows(nq, ng) if block_rows is None else int(block_rows)
    ws_bytes = rerank_topk_workspace_bytes(nq, ng, d, k1, k2, k, block_rows)
    if ws_bytes == 0:
        rerank_plan(nq, ng, k1, k2)  # raises for what the dense plan rejects
        raise ValueError(f"blocked re-ranking needs 1 <= k <= min(128, ng) and block_rows >= 1 (k={k}, ng={ng}, "
                         f"block_rows={block_rows}) and d a positive multiple of 8 (d={d})")
    return int(k), block_rows, ws_bytes


def _rerank_topk_enqueue(planes: Planes, nq: int, ng: int, k1: int, k2: int, lambda_value: float, k: int,
                         block_rows: int, idx: torch.Tensor, dst: torch.Tensor, ev: Optional[dict], status: torch.Tensor,
                         ws: torch.Tensor):
    """ctl_rerank_topk (enqueue only, capturable in a CUDA graph).  `ev`: {ids, pos_keys, pos_count, buckets, ovf} or
    None."""
    if ev is None:
        e = [0, 0, 0, 0, 1, 0, 0, 0, 0]
    else:
        ids = ev["ids"]
        e = [ids.q_pid.data_ptr(), ids.q_cam.data_ptr(), ids.g_pid.data_ptr(), ids.g_mask.data_ptr(), ids.max_pos,
             ev["pos_keys"].data_ptr(), ev["pos_count"].data_ptr(), ev["buckets"].data_ptr(), ev["ovf"].data_ptr()]
    N.check(N.lib().ctl_rerank_topk(planes.ptr, nq, ng, planes.d, planes.flags, int(k1), int(k2), float(lambda_value),
                                    int(k), int(block_rows), idx.data_ptr(), dst.data_ptr(), *e, status.data_ptr(),
                                    ws.data_ptr(), ws.numel(), N.stream_ptr()))


def _rerank_topk_run(q, g, k, k1, k2, lambda_value, normalize, block_rows, ids_args=None, max_rank=50):
    """ctl_rerank_topk from features; ids_args = (q_pids, g_pids, q_camids, g_camids, respect_camids) adds the
    evaluation."""
    planes = _rerank_inputs(q, g, normalize)
    nq, ng = q.shape[0], g.shape[0]
    k, block_rows, ws_bytes = _rerank_topk_args(nq, ng, planes.d, k1, k2, k, block_rows)
    dev = q.device
    idx = torch.empty(nq, k, dtype=torch.int64, device=dev)
    dst = torch.empty(nq, k, dtype=torch.float32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    ev = None
    if ids_args is not None:
        ev = _eval_buffers(encode_ids(*ids_args, dev), nq, dev)
    with torch.cuda.device(dev):
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        _rerank_topk_enqueue(planes, nq, ng, k1, k2, lambda_value, k, block_rows, idx, dst, ev, status, ws)
        del ws
        if ev is not None:
            ranks, pack = _finalize(ev["buckets"], ev["pos_count"], nq, ev["ids"].max_pos, ev["ovf"])
        _check_status(status)
        if ev is None:
            return idx, dst, None
        return (idx, dst) + _eval_result(ranks, pack, ids_args[0], ng, max_rank)


def rerank_topk(q: torch.Tensor, g: torch.Tensor, k: int, k1: int = 20, k2: int = 6, lambda_value: float = 0.3,
                normalize: bool = False, block_rows: Optional[int] = None):
    """Each query's k <= 128 nearest gallery rows under k-reciprocal re-ranking, without the N x N or the [Q, G] matrix:
    (idx [Q, k] int64, dist [Q, k] float32) on the device, ascending (distance, gallery index) -- the first k columns of
    the stable sort of rerank()'s output, bit for bit, for any block_rows.  Three sweeps over [block_rows, N] blocks of
    the distance matrix (ctl_rerank_topk); memory grows linearly in N = Q + G.  block_rows defaults to
    rerank_block_rows (a 2 GiB block)."""
    idx, dst, _ = _rerank_topk_run(q, g, k, k1, k2, lambda_value, normalize, block_rows)
    return idx, dst


def rerank_topk_and_eval(q: torch.Tensor, g: torch.Tensor, k: int, q_pids, g_pids, q_camids, g_camids, k1: int = 20,
                         k2: int = 6, lambda_value: float = 0.3, normalize: bool = False, max_rank: int = 50,
                         respect_camids: bool = False, block_rows: Optional[int] = None):
    """rerank_topk plus eval_func's CMC / mAP of the re-ranked distances, computed block by block from the final
    distances of sweep C: (idx, dist, EvalResult) as topk_and_eval.  The EvalResult equals
    evaluate_matrix(rerank(...)) bit for bit."""
    ids_args = (q_pids, g_pids, q_camids, g_camids, respect_camids)
    return _rerank_topk_run(q, g, k, k1, k2, lambda_value, normalize, block_rows, ids_args, max_rank)


def rerank_blocked_stages(q: torch.Tensor, g: torch.Tensor, k: int, k1: int = 20, k2: int = 6,
                          lambda_value: float = 0.3, normalize: bool = False, block_rows: Optional[int] = None,
                          q_pids=None, g_pids=None, q_camids=None, g_camids=None, max_rank: int = 50,
                          respect_camids: bool = False, events: Optional[list] = None) -> dict:
    """rerank_topk one row-block stage entry point at a time (ctl_rerank_dist_rows / _rank_rows / _expand_rows, qe,
    invert, _jaccard_rows / _topk_rows), keeping every intermediate that is linear in N: {rank [N, kr], rowmax [N],
    v_idx / v_val / v_cnt, q_idx / q_val / q_cnt, col_ptr, inv_row, inv_val, idx / dist [Q, k], status, plan, planes,
    block_rows}, plus `eval` (the EvalResult) when identities are given.  For tests and inspection: `events`, a list,
    receives (name, CUDA event) pairs recorded before the sweeps ("start") and after each ("A", "B", "qe_invert", "C").
    The one-rank case of the sharded protocol (_rerank_sharded); like rerank(), raises ValueError when a row of the
    distance matrix has no positive maximum."""
    ids_args = None if q_pids is None else (q_pids, g_pids, q_camids, g_camids, respect_camids)

    def mark(name):
        if events is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            events.append((name, e))

    return _rerank_sharded(ShardExchange(None), q, g, k, k1, k2, lambda_value, normalize, block_rows, ids_args, max_rank,
                           mark)


def _rerank_tables(planes: Planes, nq: int, ng: int, k: int, k1: int, k2: int, lambda_value: float, R: int) -> dict:
    """The global tables of the row-blocked stages, every one linear in N = nq + ng (see rerank_blocked_stages)."""
    n = nq + ng
    pl = rerank_plan(nq, ng, k1, k2)
    dev = planes.buf.device
    i32, f32 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.float32, device=dev)
    r = {"plan": pl, "planes": planes, "block_rows": R, "lambda": float(lambda_value), "rank": torch.empty(n, pl.kr, **i32),
         "rowmax": torch.empty(n, **f32), "status": torch.zeros(1, **i32), "v_idx": torch.full((n, pl.v_cap), -1, **i32),
         "v_val": torch.zeros(n, pl.v_cap, **f32), "v_cnt": torch.zeros(n, **i32),
         "idx": torch.empty(nq, k, dtype=torch.int64, device=dev), "dist": torch.empty(nq, k, **f32)}
    if k2 > 1:
        r.update(q_idx=torch.full((n, pl.q_cap), -1, **i32), q_val=torch.zeros(n, pl.q_cap, **f32),
                 q_cnt=torch.zeros(n, **i32))
    else:
        r.update(q_idx=r["v_idx"], q_val=r["v_val"], q_cnt=r["v_cnt"])
    cap = r["q_idx"].shape[1]
    r.update(col_ptr=torch.empty(n + 1, **i32), inv_row=torch.full((ng * cap,), -1, **i32),
             inv_val=torch.zeros(ng * cap, **f32))
    return r


def _rerank_sweep_a(r: dict, lo: int, hi: int, blk: torch.Tensor):
    """Sweep A over rows [lo, hi) in blocks of r["block_rows"]: rank and rowmax of those rows (status OR-ed).  `blk` holds
    min(block_rows, hi - lo) rows of N floats."""
    L = N.lib()
    planes, R = r["planes"], r["block_rows"]
    n, s = planes.n, N.stream_ptr()
    for r0 in range(lo, hi, R):
        rows = min(R, hi - r0)
        N.check(L.ctl_rerank_dist_rows(planes.ptr, n, planes.d, planes.flags, r0, rows, 0, n, None, blk.data_ptr(), n, s))
        N.check(L.ctl_rerank_rank_rows(blk.data_ptr(), r0, rows, n, n, r["plan"].kr, r["rank"].data_ptr(),
                                       r["rowmax"].data_ptr(), r["status"].data_ptr(), s))


def _rerank_sweep_b(r: dict, lo: int, hi: int, blk: torch.Tensor, k1: int, k2: int):
    """Sweep B over rows [lo, hi): the expansion V of those rows.  Reads rowmax of those rows and the rank table of
    every row (the reciprocity test), so both must be complete."""
    L = N.lib()
    planes, R = r["planes"], r["block_rows"]
    n, s = planes.n, N.stream_ptr()
    for r0 in range(lo, hi, R):
        rows = min(R, hi - r0)
        N.check(L.ctl_rerank_dist_rows(planes.ptr, n, planes.d, planes.flags, r0, rows, 0, n, r["rowmax"].data_ptr(),
                                       blk.data_ptr(), n, s))
        N.check(L.ctl_rerank_expand_rows(blk.data_ptr(), r0, rows, n, n, r["rank"].data_ptr(), k1, k2,
                                         r["v_idx"].data_ptr(), r["v_val"].data_ptr(), r["v_cnt"].data_ptr(), s))


def _rerank_qe_invert(r: dict, k1: int, k2: int):
    """Query expansion (k2 > 1) and the inverted index of the gallery rows, over the whole V."""
    L = N.lib()
    n = r["planes"].n
    nq = r["idx"].shape[0]
    cap = r["q_idx"].shape[1]
    s = N.stream_ptr()
    if k2 > 1:
        N.check(L.ctl_rerank_qe(r["rank"].data_ptr(), n, k1, k2, r["v_idx"].data_ptr(), r["v_val"].data_ptr(),
                                r["v_cnt"].data_ptr(), r["q_idx"].data_ptr(), r["q_val"].data_ptr(),
                                r["q_cnt"].data_ptr(), s))
    cursor = torch.empty(n, dtype=torch.int32, device=r["rank"].device)
    N.check(L.ctl_rerank_invert(nq, n - nq, r["q_idx"].data_ptr(), r["q_val"].data_ptr(), r["q_cnt"].data_ptr(), cap,
                                r["col_ptr"].data_ptr(), cursor.data_ptr(), r["inv_row"].data_ptr(),
                                r["inv_val"].data_ptr(), s))


def _rerank_sweep_c(r: dict, lo: int, hi: int, ev: Optional[dict]):
    """Sweep C over queries [lo, hi) against the whole gallery: their top-k rows of r["idx"] / r["dist"] and, with
    `ev` (_eval_buffers over all queries), the collect / sort / count passes of those rows."""
    if hi <= lo:
        return
    L = N.lib()
    nq = r["idx"].shape[0]
    ng = r["planes"].n - nq
    k = r["idx"].shape[1]
    s = N.stream_ptr()
    Rq = min(r["block_rows"], hi - lo)
    fin = torch.empty(Rq, ng, dtype=torch.float32, device=r["rank"].device)
    for q0 in range(lo, hi, Rq):
        rows = min(Rq, hi - q0)
        out = rerank_final_rows(r, q0, rows, out=fin)
        N.check(L.ctl_rerank_topk_rows(out.data_ptr(), q0, rows, ng, ng, k, r["idx"].data_ptr(), r["dist"].data_ptr(), s))
        if ev is not None:
            _eval_matrix_rows(out, q0, rows, ng, ng, ev)


def rerank_final_rows(r: dict, q0: int, rows: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The re-ranked distances of queries [q0, q0 + rows) against the whole gallery, [rows, G] float32, from the tables of
    rerank_blocked_stages (sweep C of one query block: ctl_rerank_dist_rows normalised by the stored row maxima, then
    ctl_rerank_jaccard_rows) -- the same rows of rerank()'s output, bit for bit."""
    L = N.lib()
    planes = r["planes"]
    nq, ng = r["idx"].shape[0], r["inv_row"].numel() // r["q_idx"].shape[1]
    n = nq + ng
    dev = r["rank"].device
    nd = torch.empty(rows, ng, dtype=torch.float32, device=dev)
    if out is None:
        out = torch.empty(rows, ng, dtype=torch.float32, device=dev)
    out = out[:rows]
    with torch.cuda.device(dev):
        s = N.stream_ptr()
        N.check(L.ctl_rerank_dist_rows(planes.ptr, n, planes.d, planes.flags, q0, rows, nq, ng, r["rowmax"].data_ptr(),
                                       nd.data_ptr(), ng, s))
        N.check(L.ctl_rerank_jaccard_rows(nq, ng, q0, rows, r["q_idx"].data_ptr(), r["q_val"].data_ptr(),
                                          r["q_cnt"].data_ptr(), r["q_idx"].shape[1], r["col_ptr"].data_ptr(),
                                          r["inv_row"].data_ptr(), r["inv_val"].data_ptr(), nd.data_ptr(), ng,
                                          r["lambda"], out.data_ptr(), ng, s))
    return out


# ----------------------------------------------------------------------------------------
# row-blocked re-ranking sharded over ranks
# ----------------------------------------------------------------------------------------


def row_shares(n: int, world: int) -> list:
    """The contiguous share [lo, hi) of n rows that each of `world` ranks computes: sizes differ by at most one, and a
    rank gets no rows when world > n."""
    return [(j * int(n) // world, (j + 1) * int(n) // world) for j in range(world)]


def _local_error(q_local, g_local, ids_args):
    """What is wrong with this rank's own arguments, as (exception class, message), or None."""
    try:
        N.require_cuda(q_local, g_local)
        if q_local.dim() != 2 or g_local.dim() != 2 or q_local.shape[1] != g_local.shape[1]:
            raise ValueError(f"expected [Q_r, d] and [G_r, d] features, got {tuple(q_local.shape)} and "
                             f"{tuple(g_local.shape)}")
        if q_local.device != g_local.device:
            raise ValueError("query and gallery shards are on different devices")
        if ids_args is not None and len(ids_args[1]) != g_local.shape[0]:
            raise ValueError(f"{len(ids_args[1])} gallery pids for {g_local.shape[0]} gallery rows")
    except (RuntimeError, ValueError) as e:
        return type(e), str(e)
    return None


def _rerank_sharded(ex, q_local: torch.Tensor, g_local: torch.Tensor, k: int, k1: int, k2: int, lambda_value: float,
                    normalize: bool, block_rows: Optional[int], ids_args=None, max_rank: int = 50, mark=None) -> dict:
    """The sharded protocol of rerank_topk_sharded / rerank_topk_and_eval_sharded over the exchange `ex` (ShardExchange,
    or a stand-in with its methods); with ShardExchange(None), rerank_blocked_stages.  ids_args = (q_pids of all queries,
    this rank's g_pids, q_camids of all queries, this rank's g_camids, respect_camids) adds the evaluation.  `mark(name)`,
    if given, is called on the device's stream before the sweeps ("start") and after each ("A", "B", "qe_invert", "C").
    Returns the gathered tables of rerank_blocked_stages (rank, rowmax, v_*, q_*, col_ptr, inv_*, idx, dist, status,
    plan, planes, block_rows; `eval` with identities), the same on every rank."""
    # 1. shard sizes, identities and local errors in ONE exchange; then every rank checks the same global arguments and
    #    raises the same error before any data is exchanged
    err = _local_error(q_local, g_local, ids_args)
    ok = err is None
    mine = {"nq": q_local.shape[0] if ok else 0, "ng": g_local.shape[0] if ok else 0, "d": q_local.shape[1] if ok else 0,
            "err": err}
    if ids_args is not None:
        mine.update(nq_ids=len(ids_args[0]), g_pids=np.asarray(ids_args[1]),
                    g_camids=list(ids_args[3])[: mine["ng"]])
    meta = ex.objects(mine)
    for j, m in enumerate(meta):
        if m["err"] is not None:
            raise m["err"][0](f"rank {j}: {m['err'][1]}")
    nq_r, ng_r = [m["nq"] for m in meta], [m["ng"] for m in meta]
    nq, ng = sum(nq_r), sum(ng_r)
    if len({m["d"] for m in meta}) != 1:
        raise ValueError(f"feature widths differ across ranks: {[m['d'] for m in meta]}")
    d = meta[0]["d"]
    k, R, _ = _rerank_topk_args(nq, ng, d, k1, k2, k, block_rows)
    if ids_args is not None and any(m["nq_ids"] != nq for m in meta):
        raise ValueError(f"q_pids must cover all {nq} queries; ranks give {[m['nq_ids'] for m in meta]}")

    # 2. features of all N rows on every rank, in the order [queries by rank; gallery by rank]
    dev = q_local.device
    q = ex.rows(q_local.detach().float().contiguous(), nq_r)
    g = ex.rows(g_local.detach().float().to(dev).contiguous(), ng_r)
    planes = _rerank_inputs(q, g, normalize)
    del q, g
    r = _rerank_tables(planes, nq, ng, k, k1, k2, lambda_value, R)
    ev = None
    if ids_args is not None:
        q_pids, _, q_camids, _, respect_camids = ids_args
        g_pids = np.concatenate([m["g_pids"] for m in meta])
        g_camids = [c for m in meta for c in m["g_camids"]]
        ev = _eval_buffers(encode_ids(q_pids, g_pids, q_camids, g_camids, respect_camids, dev), nq, dev)
    n = nq + ng
    shares, q_shares = row_shares(n, ex.world), row_shares(nq, ex.world)
    lo, hi = shares[ex.rank]
    qlo, qhi = q_shares[ex.rank]
    counts, q_counts = [b - a for a, b in shares], [b - a for a, b in q_shares]
    mark = mark or (lambda name: None)
    with torch.cuda.device(dev):
        # 3. sweep A on this rank's rows -> the whole rank table and row maxima
        blk = torch.empty(min(R, hi - lo) * n, dtype=torch.float32, device=dev)
        mark("start")
        _rerank_sweep_a(r, lo, hi, blk)
        mark("A")
        r["rank"] = ex.rows(r["rank"][lo:hi], counts)
        r["rowmax"] = ex.rows(r["rowmax"][lo:hi], counts)
        ex.max_(r["status"])
        # 4. sweep B on the same rows -> the whole V
        _rerank_sweep_b(r, lo, hi, blk, k1, k2)
        mark("B")
        del blk
        for key in ("v_idx", "v_val", "v_cnt"):
            r[key] = ex.rows(r[key][lo:hi], counts)
        if k2 == 1:
            r.update(q_idx=r["v_idx"], q_val=r["v_val"], q_cnt=r["v_cnt"])
        # 5. query expansion and the inverted index, whole, on every rank
        _rerank_qe_invert(r, k1, k2)
        mark("qe_invert")
        # 6. sweep C on this rank's queries against the whole gallery, then the per-query results of every rank
        _rerank_sweep_c(r, qlo, qhi, ev)
        mark("C")
        r["idx"] = ex.rows(r["idx"][qlo:qhi], q_counts)
        r["dist"] = ex.rows(r["dist"][qlo:qhi], q_counts)
        if ev is not None:
            mp = ev["ids"].max_pos
            ex.max_(ev["ovf"])
            if qhi > qlo:
                ranks, pack = _finalize(ev["buckets"][qlo:qhi], ev["pos_count"][qlo:qhi], qhi - qlo, mp, ev["ovf"])
            else:
                ranks = torch.empty(0, mp, dtype=torch.int32, device=dev)
                pack = torch.empty(1, 3, dtype=torch.float64, device=dev)
            ranks = ex.rows(ranks, q_counts)
            pack = torch.cat([ex.rows(pack[: qhi - qlo], q_counts), ev["ovf"].double().expand(1, 3)])
        _check_status(r["status"])
        if ev is not None:
            r["eval"] = _eval_result(ranks, pack, q_pids, ng, max_rank)[0]
    return r


def rerank_topk_sharded(q_local: torch.Tensor, g_local: torch.Tensor, k: int, k1: int = 20, k2: int = 6,
                        lambda_value: float = 0.3, normalize: bool = False, block_rows: Optional[int] = None, group=None):
    """rerank_topk with the queries and the gallery sharded over the ranks of `group` (torch.distributed; None: one
    rank).  Rank j holds q_local [Q_j, d] and g_local [G_j, d]; the problem is queries [all q_local in rank order] against
    gallery [all g_local in rank order], and returned gallery indices are positions in that concatenation.  Every rank
    returns the full (idx [Q, k] int64, dist [Q, k] float32), bit-identical to rerank_topk on the concatenated features.
    The N = Q + G rows of sweeps A and B and the Q queries of sweep C are split in contiguous shares (row_shares); the
    rank table, the row maxima, V and the results are all-gathered between the sweeps (DESIGN.md §5)."""
    r = _rerank_sharded(ShardExchange(group), q_local, g_local, k, k1, k2, lambda_value, normalize, block_rows)
    return r["idx"], r["dist"]


def rerank_topk_and_eval_sharded(q_local: torch.Tensor, g_local: torch.Tensor, k: int, q_pids, g_pids_local, q_camids,
                                 g_camids_local, k1: int = 20, k2: int = 6, lambda_value: float = 0.3,
                                 normalize: bool = False, max_rank: int = 50, respect_camids: bool = False,
                                 block_rows: Optional[int] = None, group=None):
    """rerank_topk_and_eval with the queries and the gallery sharded over the ranks of `group`, as rerank_topk_sharded.
    q_pids / q_camids cover ALL queries (as in topk_and_eval_sharded); g_pids_local / g_camids_local this rank's gallery
    rows.  Every rank returns (idx, dist, EvalResult), bit-identical to rerank_topk_and_eval on the concatenation."""
    ids_args = (q_pids, g_pids_local, q_camids, g_camids_local, respect_camids)
    r = _rerank_sharded(ShardExchange(group), q_local, g_local, k, k1, k2, lambda_value, normalize, block_rows, ids_args,
                        max_rank)
    return r["idx"], r["dist"], r["eval"]
