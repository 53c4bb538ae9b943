"""Float64 restatement of k-reciprocal re-ranking (Zhong, Zheng, Cao, Li, "Re-ranking Person Re-identification with
k-reciprocal Encoding", CVPR 2017) as the engine implements it (include/ctl_b200.h, DESIGN.md section 4), in two
independent forms:

- `rerank_loop`: a literal per-row loop that follows the paper -- forward neighbours, the backward check that makes them
  k-reciprocal, the 2/3 rule written as the paper's fraction, a dense V, a dense query expansion, and the Jaccard distance
  accumulated query by query through an inverted index;
- the sparse vectorised stages `rank_table`, `expansion`, `query_expansion`, `jaccard_blend` (composed by
  `rerank_sparse`): array operations over all rows and scipy.sparse matrices, so a Market-1501-sized problem fits.

Both take either features (`nd_from_features`) or a given normalised distance matrix `nd` (teacher forcing: the engine's
own matrix).  They were written from the paper and from the engine's contract.  No third-party implementation is
vendored or pinned: the reference re-ID project has no re-ranking, so there is nothing of it to compare against.

Where the engine's contract differs from the widely used numpy implementation of the paper, the oracle follows the
engine: V, the query expansion and the Jaccard sums are exact float64 here (float32 in the engine, float16 in that
implementation), and equal distances are ordered by column index (np.argsort's default sort is not stable).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp


def half_k(k1: int) -> int:
    """h = round-half-even(k1 / 2), numpy's around: k1 = 5 -> 2, k1 = 7 -> 4."""
    return int(np.around(k1 / 2.0))


def nd_from_features(feats, normalize: bool = False) -> np.ndarray:
    """Step 1 + 2 as the engine rounds them: squared euclidean distances of the rows among themselves (float64, then
    float32 like the engine's matrix), divided row by row by the row maximum in float32 (one IEEE division).  A float64
    division could keep apart two values that the float32 one merges into a tie.  Returns float32 [N, N]."""
    x = np.asarray(feats, dtype=np.float64)
    if normalize:
        x = x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-12)
    sq = (x * x).sum(1)
    d32 = (sq[:, None] + sq[None, :] - 2.0 * (x @ x.T)).astype(np.float32)
    mx = d32.max(axis=1)
    if not (mx > 0).all():
        raise ValueError("a row of the distance matrix has no positive maximum")
    return d32 / mx[:, None]


# ------------------------------------------------------------------------------------------
# form 1: the literal per-row loop
# ------------------------------------------------------------------------------------------


def rerank_loop(nd, nq: int, k1: int, k2: int, lambda_value: float) -> dict:
    """The paper's algorithm, one row at a time.  Returns {rank (full stable argsort), R, E (sorted arrays), V, V_qe
    (dense float64 [N, N]), out [Q, G]}."""
    nd = np.asarray(nd)
    n = nd.shape[0]
    h = half_k(k1)
    rank = np.argsort(nd, axis=1, kind="stable")  # ascending (distance, index)
    V = np.zeros((n, n), dtype=np.float64)
    R_all, E_all = [], []
    for i in range(n):
        forward = rank[i, : k1 + 1]
        R = [int(j) for j in forward if i in rank[j, : k1 + 1]]  # backward check: i among j's own k1 + 1 nearest
        E = set(R)
        for c in R:
            cand_forward = rank[c, : h + 1]
            Rc = [int(m) for m in cand_forward if c in rank[m, : h + 1]]
            if len(set(Rc) & set(R)) > 2.0 / 3.0 * len(Rc):
                E |= set(Rc)
        E = np.array(sorted(E), dtype=np.int64)
        w = np.exp(-nd[i, E].astype(np.float64))
        V[i, E] = w / w.sum()
        R_all.append(np.array(R, dtype=np.int64))
        E_all.append(E)
    if k2 > 1:
        V_qe = np.zeros_like(V)
        for i in range(n):
            V_qe[i] = V[rank[i, :k2]].mean(axis=0)
    else:
        V_qe = V
    ng = n - nq
    inv = [np.nonzero(V_qe[nq:, c])[0] for c in range(n)]  # inverted index: gallery rows with a non-zero in column c
    out = np.empty((nq, ng), dtype=np.float64)
    for i in range(nq):
        acc = np.zeros(ng, dtype=np.float64)
        for c in np.nonzero(V_qe[i])[0]:
            rows = inv[c]
            acc[rows] += np.minimum(V_qe[i, c], V_qe[nq + rows, c])
        jac = 1.0 - acc / (2.0 - acc)
        out[i] = jac * (1.0 - lambda_value) + nd[i, nq:].astype(np.float64) * lambda_value
    return {"rank": rank, "R": R_all, "E": E_all, "V": V, "V_qe": V_qe, "out": out}


# ------------------------------------------------------------------------------------------
# form 2: sparse, vectorised stages
# ------------------------------------------------------------------------------------------


def rank_table(nd, kr: int) -> np.ndarray:
    """Step 3: the first min(kr, N) columns of every row by (value, column), via a partition instead of a full sort:
    every value below the kr-th smallest, then the ties at it in column order.  int64 [N, kr], -1 beyond N columns."""
    nd = np.asarray(nd)
    n = nd.shape[0]
    k = min(kr, n)
    thr = np.partition(nd, k - 1, axis=1)[:, k - 1]
    lt = nd < thr[:, None]
    eq = nd == thr[:, None]
    need = k - lt.sum(axis=1)
    sel = lt | (eq & (np.cumsum(eq, axis=1, dtype=np.int32) <= need[:, None]))
    rows, cols = np.nonzero(sel)  # k per row, ascending columns
    cols = cols.reshape(n, k)
    vals = nd[rows.reshape(n, k), cols]
    order = np.argsort(vals, axis=1, kind="stable")  # (value, column): columns are ascending already
    out = np.full((n, kr), -1, dtype=np.int64)
    out[:, :k] = np.take_along_axis(cols, order, axis=1)
    return out


def _reciprocal(rank: np.ndarray, k: int) -> np.ndarray:
    """[N, k] bool: rank[i, t] has i among its own first k columns."""
    n = rank.shape[0]
    f = rank[:, :k]
    return (rank[f][:, :, :k] == np.arange(n)[:, None, None]).any(axis=2)


def expansion(rank, k1: int, nd) -> sp.csr_matrix:
    """Step 4 for every row at once: V as a float64 CSR matrix (sorted, unique column indices per row).  `nd` is the
    [N, N] matrix or a callable gather(rows, cols) -> values (the weights only need nd at the expansion sets)."""
    rank = np.asarray(rank, dtype=np.int64)
    n = rank.shape[0]
    h = half_k(k1)
    nf, nh = min(k1 + 1, n), min(h + 1, n)
    F, Fh = rank[:, :nf], rank[:, :nh]
    rec = _reciprocal(rank, nf)            # [N, nf]: F[i, t] in R(i)
    rec_h = _reciprocal(rank, nh)          # [N, nh]: Fh[c, u] in R_h(c)
    mem = Fh[F]                            # [N, nf, nh]: forward h-neighbours of candidate F[i, t]
    mem_ok = rec_h[F]                      # ... that are h-reciprocal to it
    in_R = ((mem[..., None] == F[:, None, None, :]) & rec[:, None, None, :]).any(axis=3)
    length = mem_ok.sum(axis=2)
    inter = (mem_ok & in_R).sum(axis=2)
    accept = rec & (3 * inter > 2 * length)
    r1, t1 = np.nonzero(rec)
    ra, ta, ua = np.nonzero(accept[:, :, None] & mem_ok)
    rows = np.concatenate([r1, ra])
    cols = np.concatenate([F[r1, t1], mem[ra, ta, ua]])
    key = np.unique(rows * n + cols)
    rows, cols = key // n, key % n
    vals = nd(rows, cols) if callable(nd) else np.asarray(nd)[rows, cols]
    w = np.exp(-np.asarray(vals, dtype=np.float64))
    w = w / np.bincount(rows, weights=w, minlength=n)[rows]
    return sp.csr_matrix((w, (rows, cols)), shape=(n, n))


def query_expansion(rank, V: sp.csr_matrix, k2: int) -> sp.csr_matrix:
    """Step 5: V_qe[i] = mean of V over rows rank[i, :k2] (V itself when k2 = 1)."""
    if k2 <= 1:
        return V
    rank = np.asarray(rank)
    n = rank.shape[0]
    m = min(k2, n)
    P = sp.csr_matrix((np.full(n * m, 1.0 / m), (np.repeat(np.arange(n), m), rank[:, :m].reshape(-1))), shape=(n, n))
    out = (P @ V).tocsr()
    out.sort_indices()
    return out


def jaccard_sums(V_qe: sp.csr_matrix, nq: int, queries=None) -> np.ndarray:
    """s[i, j] = sum_c min(V_qe[i, c], V_qe[nq + j, c]) for the given query rows (default: all), float64 [len, G]."""
    V_qe = V_qe.tocsr()
    n = V_qe.shape[0]
    ng = n - nq
    G = V_qe[nq:].tocsc()
    queries = range(nq) if queries is None else queries
    out = np.zeros((len(queries), ng), dtype=np.float64)
    for a, i in enumerate(queries):
        lo, hi = V_qe.indptr[i], V_qe.indptr[i + 1]
        cols, vals = V_qe.indices[lo:hi], V_qe.data[lo:hi]
        sub = G[:, cols]
        data = np.minimum(sub.data, np.repeat(vals, np.diff(sub.indptr)))
        out[a] = np.bincount(sub.indices, weights=data, minlength=ng)
    return out


def jaccard_blend(s: np.ndarray, nd_qg, lambda_value: float) -> np.ndarray:
    """Step 6's blend: (1 - lambda) (1 - s / (2 - s)) + lambda nd[i, Q + j]."""
    jac = 1.0 - s / (2.0 - s)
    return jac * (1.0 - lambda_value) + np.asarray(nd_qg, dtype=np.float64) * lambda_value


def rerank_sparse(nd, nq: int, k1: int, k2: int, lambda_value: float) -> dict:
    """Steps 3-6 through the sparse stages: {rank, V, V_qe, out}."""
    nd = np.asarray(nd)
    rank = rank_table(nd, max(k1 + 1, k2))
    V = expansion(rank, k1, nd)
    V_qe = query_expansion(rank, V, k2)
    out = jaccard_blend(jaccard_sums(V_qe, nq), nd[:nq, nq:], lambda_value)
    return {"rank": rank, "V": V, "V_qe": V_qe, "out": out}


def csr_rows(M: sp.csr_matrix, i: int):
    """(columns, values) of row i of a CSR matrix, columns ascending."""
    lo, hi = M.indptr[i], M.indptr[i + 1]
    o = np.argsort(M.indices[lo:hi], kind="stable")
    return M.indices[lo:hi][o], M.data[lo:hi][o]
