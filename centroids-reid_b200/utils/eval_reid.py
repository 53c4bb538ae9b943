"""Drop-in for utils/eval_reid.py of the reference.

`eval_func` keeps the reference signature (it consumes a full [Q, G] ranking that the caller
already holds on the host) and is vectorised host code; the product path does NOT build that
ranking at all: `eval_streamed` computes the same (cmc, mAP, all_topk, single_performance)
straight from the features on the H100 (retrieval.evaluate_streamed), which is what
`R1_mAP.compute` in utils/reid_metric.py calls.
"""
from __future__ import annotations

import numpy as np

from .. import retrieval as _R

k_list = [1, 5, 10, 20, 50]  # utils/eval_reid.py:15


def top_k_retrieval(row_matches: np.ndarray, k: list):
    """utils/eval_reid.py:18-22."""
    return [int(np.any(row_matches[:kk])) for kk in k]


def eval_func(indices, q_pids, g_pids, q_camids, g_camids, max_rank=50, respect_camids=False):
    """utils/eval_reid.py:25-92, same arguments and return values, without the per-query
    Python loop (chunks of queries, cumulative sums over the kept ranking).

    Evaluation with the market1501 metric: for each query, gallery samples with the same pid
    AND the same camera (or, with respect_camids, whose camera set contains the query camera)
    are discarded before CMC / AP are computed over the whole remaining ranking.
    """
    indices = np.asarray(indices)
    q_pids, g_pids = np.asarray(q_pids), np.asarray(g_pids)
    num_q, num_g = indices.shape
    if num_g < max_rank:
        max_rank = num_g
        print("Note: number of gallery samples is quite small, got {}".format(num_g))
    qp, qc, gp, gm, _ = _R.encode_identities(q_pids, g_pids, q_camids, g_camids, respect_camids)
    all_cmc = np.zeros(max_rank, dtype=np.float32)
    aps, topk_rows, single = [], [], []
    chunk = max(1, (1 << 24) // max(1, num_g))
    for s in range(0, num_q, chunk):
        idx = indices[s : s + chunk]
        same = gp[idx] == qp[s : s + chunk, None]
        in_cam = ((gm[idx] >> qc[s : s + chunk, None].astype(np.uint64)) & np.uint64(1)).astype(bool)
        keep = ~(same & in_cam)
        hits = same & keep
        kept_rank = np.cumsum(keep, axis=1)          # 1-based rank among kept rows
        hit_cum = np.cumsum(hits, axis=1)
        n_rel = hit_cum[:, -1]
        for r in np.nonzero(n_rel > 0)[0]:
            pos = np.nonzero(hits[r])[0]
            ranks = kept_rank[r, pos]
            first = int(ranks[0])
            if first <= max_rank:
                all_cmc[first - 1 :] += 1.0
            prec = hit_cum[r, pos] / (ranks.astype(np.float64))
            ap = float(prec.sum() / n_rel[r])
            aps.append(ap)
            single.append([s + r, q_pids[s + r], ap])
            topk_rows.append([int(first <= kk) for kk in k_list])
    if not aps:
        raise RuntimeError("no valid query: no query identity appears in the gallery")
    num_valid_q = float(len(aps))
    all_cmc = all_cmc / num_valid_q
    return all_cmc, np.mean(aps), np.mean(np.vstack(topk_rows), 0), np.array(single)


def eval_streamed(q_feats, g_feats, q_pids, g_pids, q_camids, g_camids, max_rank=50, respect_camids=False,
                  dist_func="euclidean", feat_norm=False):
    """eval_func's results computed on the H100 directly from query / gallery features
    (no distance matrix, no argsort).  Host tensors are staged to the current CUDA device."""
    import torch

    q = torch.as_tensor(q_feats)
    g = torch.as_tensor(g_feats)
    if not q.is_cuda:
        q = q.cuda(non_blocking=True)
    if not g.is_cuda:
        g = g.cuda(non_blocking=True)
    go = _R.pid_order(g_pids) if len(g_pids) == g.shape[0] else None  # identity order: cheap collect pass
    qp = _R.build_planes(q, dist_func, feat_norm, order=_R.pid_order(q_pids))
    gp = _R.build_planes(g, dist_func, feat_norm, order=go)
    res = _R.evaluate_streamed(qp, gp, q_pids, g_pids, q_camids, g_camids, max_rank, respect_camids)
    return res.cmc, res.mAP, res.all_topk, res.single_performance


def eval_reranked(q_feats, g_feats, q_pids, g_pids, q_camids, g_camids, max_rank=50, respect_camids=False, k1=20, k2=6,
                  lambda_value=0.3, feat_norm=False):
    """eval_func's results on k-reciprocal re-ranked distances, on the H100.  Same 4-tuple as eval_streamed.  Host
    tensors are staged to the current CUDA device.  When the dense re-ranking and its [Q, G] matrix fit in the device's
    free memory (retrieval.rerank_fits_dense): retrieval.rerank, then retrieval.evaluate_matrix; otherwise (galleries
    beyond the N^2 bound) the row-blocked retrieval.rerank_topk_and_eval, whose results are bit-identical."""
    import torch

    q = torch.as_tensor(q_feats)
    g = torch.as_tensor(g_feats)
    if not q.is_cuda:
        q = q.cuda(non_blocking=True)
    if not g.is_cuda:
        g = g.to(q.device, non_blocking=True)
    free, _ = torch.cuda.mem_get_info(q.device)
    if _R.rerank_fits_dense(q.shape[0], g.shape[0], k1, k2, free):
        dist = _R.rerank(q, g, k1, k2, lambda_value, feat_norm)
        res = _R.evaluate_matrix(dist, q_pids, g_pids, q_camids, g_camids, max_rank, respect_camids)
    else:
        _, _, res = _R.rerank_topk_and_eval(q, g, 1, q_pids, g_pids, q_camids, g_camids, k1, k2, lambda_value, feat_norm,
                                            max_rank, respect_camids)
    return res.cmc, res.mAP, res.all_topk, res.single_performance
