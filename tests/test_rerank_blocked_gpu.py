"""GPU: row-blocked k-reciprocal re-ranking (ctl_rerank_topk and its row-block stages) against the dense path.

The contract is bit identity: for every block_rows, the rank table, V, the expanded V and the inverted index equal
rerank_stages' buffers, the top-k equals the stable sort of rerank()'s output, and the EvalResult equals
evaluate_matrix(rerank(...)).  It rests on a distance depending only on its two rows (asserted here through rowmax and
the tables), on the exact row maximum, on the same IEEE division, and on the later kernels being the dense path's.
Beyond the dense bound (N^2 * 4 bytes larger than the card) the rows of a fixed sample are checked against the engine's
own 1 x N distance rows and the float64 oracle (oracle/rerank_oracle.py), as in tests/test_rerank_gpu.py.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from ctl_b200 import retrieval as R
from oracle import ctl_oracle as O
from oracle import rerank_oracle as RO

pytestmark = pytest.mark.gpu

K1, K2, LAM = 20, 6, 0.3


def _csr(idx, val, cnt, n):
    m = max(1, int(cnt.max()))
    idx, val, cnt = idx[:, :m].cpu().numpy(), val[:, :m].cpu().numpy().astype(np.float64), cnt.cpu().numpy()
    rows = np.repeat(np.arange(n), cnt)
    mask = np.arange(m)[None, :] < cnt[:, None]
    return sp.csr_matrix((val[mask], (rows, idx[mask])), shape=(n, n))


def _inverted_sorted(r):
    """The inverted index with every column's (row, value) entries sorted by row: the set per column."""
    col_ptr = r["col_ptr"].cpu().numpy()
    nnz = int(col_ptr[-1])
    inv_row, inv_val = r["inv_row"][:nnz].cpu().numpy(), r["inv_val"][:nnz].cpu().numpy()
    seg = np.repeat(np.arange(len(col_ptr) - 1), np.diff(col_ptr))
    o = np.lexsort((inv_row, seg))
    return col_ptr, inv_row[o], inv_val[o]


def _stable_topk(out, k):
    o = torch.sort(out, dim=1, stable=True).indices[:, :k]
    return o, out.gather(1, o)


def _assert_eval_equal(a, b):
    assert np.array_equal(a.cmc, b.cmc)
    assert a.mAP == b.mAP
    assert np.array_equal(a.all_topk, b.all_topk)
    assert np.array_equal(a.ranks, b.ranks)
    assert np.array_equal(a.single_performance, b.single_performance)


def _ids(nq, pids, cams, respect_camids):
    q_pids = pids[:nq].copy()
    q_pids[::11] = 5000 + np.arange(len(q_pids[::11]))  # queries without a positive in the gallery
    g_cams = [[int(c), int(c + 2) % 6] for c in cams[nq:]] if respect_camids else cams[nq:]
    return q_pids, pids[nq:], cams[:nq], g_cams


_DENSE = {}


def _dense(d):
    """rerank_stages at N = 2000 (Q = 400), one per feature width."""
    if d not in _DENSE:
        nq, ng = 400, 1600
        feats, pids, cams = O.synth_retrieval(nq, ng, 60, d, 3.0, 100 + d)
        q, g = feats[:nq].cuda(), feats[nq:].cuda()
        _DENSE[d] = (q, g, pids, cams, R.rerank_stages(q, g, K1, K2, LAM))
    return _DENSE[d]


@pytest.mark.parametrize("block_rows", [1, 7, 128, 333, 2000])
@pytest.mark.parametrize("d", [72, 512])
def test_blocked_equals_dense(d, block_rows):
    q, g, pids, cams, dense = _dense(d)
    nq = q.shape[0]
    k = 50
    ids = _ids(nq, pids, cams, respect_camids=block_rows % 2 == 1)
    r = R.rerank_blocked_stages(q, g, k, K1, K2, LAM, block_rows=block_rows, q_pids=ids[0], g_pids=ids[1],
                                q_camids=ids[2], g_camids=ids[3], respect_camids=block_rows % 2 == 1)
    assert int(r["status"].item()) == 0
    # rowmax: the exact row maxima of ctl_dist_matrix of [q; g]
    F = torch.cat([q, g])
    assert torch.equal(r["rowmax"], R.dist_matrix(F, F).max(dim=1).values)
    for key in ("rank", "v_idx", "v_val", "v_cnt", "q_idx", "q_val", "q_cnt", "col_ptr"):
        assert torch.equal(r[key], dense[key]), key
    a, b = _inverted_sorted(r), _inverted_sorted(dense)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    idx, dst = _stable_topk(dense["out"], k)
    assert torch.equal(r["idx"], idx) and torch.equal(r["dist"], dst)
    _assert_eval_equal(r["eval"], R.evaluate_matrix(dense["out"], *ids, 50, block_rows % 2 == 1))
    # the final rows of one query block, and the one-call entry point
    q0 = min(nq - 1, 3 * block_rows)
    assert torch.equal(R.rerank_final_rows(r, q0, min(nq - q0, 9)), dense["out"][q0: q0 + 9])
    idx1, dst1, ev1 = R.rerank_topk_and_eval(q, g, k, *ids, K1, K2, LAM, respect_camids=block_rows % 2 == 1,
                                             block_rows=block_rows)
    assert torch.equal(idx1, r["idx"]) and torch.equal(dst1, r["dist"])
    _assert_eval_equal(ev1, r["eval"])


@pytest.mark.parametrize("lam,k2,normalize,k", [(0.0, 6, False, 10), (1.0, 6, False, 10), (0.3, 1, False, 10),
                                                (0.3, 6, True, 10), (0.3, 6, False, 1), (0.3, 6, False, 128)])
def test_edge_parameters(lam, k2, normalize, k):
    feats, pids, cams = O.synth_retrieval(100, 500, 30, 72, 3.0, 31)
    q, g = feats[:100].cuda(), feats[100:].cuda()
    dense = R.rerank(q, g, K1, k2, lam, normalize)
    idx, dst = R.rerank_topk(q, g, k, K1, k2, lam, normalize, block_rows=37)
    ri, rd = _stable_topk(dense, k)
    assert torch.equal(idx, ri) and torch.equal(dst, rd)
    _, _, ev = R.rerank_topk_and_eval(q, g, k, pids[:100], pids[100:], cams[:100], cams[100:], K1, k2, lam, normalize,
                                      block_rows=64)
    _assert_eval_equal(ev, R.evaluate_matrix(dense, pids[:100], pids[100:], cams[:100], cams[100:]))


def test_duplicated_gallery_rows_tie_in_column_order():
    """lambda = 1: the final distance is nd, so duplicated gallery rows tie exactly; the ties come out in column order."""
    feats, _, _ = O.synth_retrieval(60, 200, 20, 72, 3.0, 41)
    g = torch.cat([feats[60:], feats[60:160]]).cuda()  # gallery rows j and 200 + j are equal for j < 100
    q = feats[:60].cuda()
    dense = R.rerank(q, g, K1, K2, 1.0)
    idx, dst = R.rerank_topk(q, g, 40, K1, K2, 1.0, block_rows=17)
    ri, rd = _stable_topk(dense, 40)
    assert torch.equal(idx, ri) and torch.equal(dst, rd)
    ties = (dst[:, 1:] == dst[:, :-1])
    assert int(ties.sum()) > 100
    assert bool((idx[:, 1:][ties] > idx[:, :-1][ties]).all())


def test_market_shape_bit_identical_to_dense():
    nq, ng = 3368, 15913
    feats, pids, cams = O.synth_retrieval(nq, ng, 751, 2048, 3.0, 17)
    q, g = feats[:nq].cuda(), feats[nq:].cuda()
    del feats
    dense = R.rerank(q, g)
    ref = R.evaluate_matrix(dense, pids[:nq], pids[nq:], cams[:nq], cams[nq:])
    ri, rd = _stable_topk(dense, 100)
    del dense
    for block_rows in (None, 4096):  # default (the whole matrix fits in one 2 GiB block), and five row blocks
        idx, dst, ev = R.rerank_topk_and_eval(q, g, 100, pids[:nq], pids[nq:], cams[:nq], cams[nq:],
                                              block_rows=block_rows)
        assert torch.equal(idx, ri) and torch.equal(dst, rd), block_rows
        _assert_eval_equal(ev, ref)


def _device_features(n, ids, d, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    pids = torch.randint(0, ids, (n,), generator=gen, device="cuda")
    cams = torch.randint(0, 6, (n,), generator=gen, device="cuda")
    x = torch.randn(ids, d, generator=gen, device="cuda")[pids]
    x.add_(torch.randn(n, d, generator=gen, device="cuda"), alpha=3.0)
    x = torch.nn.functional.normalize(x, dim=1)
    return x, pids.cpu().numpy(), cams.cpu().numpy()


def test_beyond_the_dense_bound():
    """Q = 10 000, G = 140 000, d = 2048: the N x N matrix alone would be 90 GB."""
    nq, ng, d, k = 10000, 140000, 2048, 100
    n = nq + ng
    x, pids, cams = _device_features(n, 7000, d, 5)
    assert n * n * 4 > torch.cuda.get_device_properties(0).total_memory
    q, g = x[:nq], x[nq:]
    args = (pids[:nq], pids[nq:], cams[:nq], cams[nq:])
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    idx, dst, ev = R.rerank_topk_and_eval(q, g, k, *args, block_rows=4096)
    peak = torch.cuda.max_memory_allocated() - base
    ws = R.rerank_topk_workspace_bytes(nq, ng, d, K1, K2, k, 4096)
    # the workspace, [q; g] and its planes (2 N d 4 bytes), identities and results: no hidden N^2 buffer
    assert peak <= ws + 2 * n * d * 4 + (256 << 20), (peak, ws)
    assert ev.mAP > 0
    r = R.rerank_blocked_stages(q, g, k, K1, K2, LAM, block_rows=3000)
    assert int(r["status"].item()) == 0
    assert torch.equal(r["idx"], idx) and torch.equal(r["dist"], dst)  # another block size, bit for bit

    rng = np.random.default_rng(0)
    sample = np.sort(np.concatenate([rng.choice(nq, 8, replace=False), nq + rng.choice(ng, 8, replace=False)]))
    planes = r["planes"]
    rows_nd = {}
    for i in sample:  # the engine's own nd rows: a 1 x N ctl_dist_matrix, divided by its maximum
        row = torch.empty(1, n, device="cuda")
        R.N.check(R.N.lib().ctl_rerank_dist_rows(planes.ptr, n, d, planes.flags, int(i), 1, 0, n, None,
                                                 row.data_ptr(), n, R.N.stream_ptr()))
        assert float(row.max()) == float(r["rowmax"][i])
        rows_nd[int(i)] = (row[0] / r["rowmax"][i] + 0.0).cpu().numpy()
    rank = r["rank"].cpu().numpy().astype(np.int64)
    kr = r["plan"].kr
    for i in sample:
        assert np.array_equal(rank[i], np.argsort(rows_nd[int(i)], kind="stable")[:kr]), i

    def gather(rows, cols):  # nd at the expansion sets; only the sampled rows are checked
        out = np.zeros(len(rows))
        for i, v in rows_nd.items():
            m = rows == i
            out[m] = v[cols[m]]
        return out

    V = RO.expansion(rank, K1, gather)
    v_idx, v_val, v_cnt = r["v_idx"].cpu().numpy(), r["v_val"].cpu().numpy(), r["v_cnt"].cpu().numpy()
    for i in sample:
        cols, vals = RO.csr_rows(V, i)
        assert v_cnt[i] == len(cols) and np.array_equal(v_idx[i, : v_cnt[i]], cols), i
        np.testing.assert_allclose(v_val[i, : v_cnt[i]], vals, rtol=0, atol=1e-6, err_msg=str(i))
    # final rows of a query block, teacher-forced on the engine's expanded V
    q0 = int(sample[0])
    fin = R.rerank_final_rows(r, q0, 4)
    Q_gpu = _csr(r["q_idx"], r["q_val"], r["q_cnt"], n)
    s = RO.jaccard_sums(Q_gpu, nq, queries=list(range(q0, q0 + 4)))
    nd_rows = []
    for i in range(q0, q0 + 4):
        row = torch.empty(1, ng, device="cuda")
        R.N.check(R.N.lib().ctl_rerank_dist_rows(planes.ptr, n, d, planes.flags, i, 1, nq, ng, r["rowmax"].data_ptr(),
                                                 row.data_ptr(), ng, R.N.stream_ptr()))
        nd_rows.append(row[0].cpu().numpy())
    np.testing.assert_allclose(fin.cpu().numpy(), RO.jaccard_blend(s, np.stack(nd_rows), LAM), rtol=0, atol=1e-5)
    fi, fd = _stable_topk(fin, k)
    assert torch.equal(fi, idx[q0: q0 + 4]) and torch.equal(fd, dst[q0: q0 + 4])


def test_repeats_and_graph_replay_are_bit_identical():
    nq, ng, k, rows = 200, 1100, 30, 300
    feats, pids, cams = O.synth_retrieval(nq, ng, 40, 512, 3.0, 5)
    q, g = feats[:nq].cuda(), feats[nq:].cuda()
    args = (pids[:nq], pids[nq:], cams[:nq], cams[nq:])
    a = R.rerank_topk_and_eval(q, g, k, *args, block_rows=rows)
    b = R.rerank_topk_and_eval(q, g, k, *args, block_rows=rows)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    _assert_eval_equal(a[2], b[2])
    planes = R._rerank_inputs(q, g, False)
    dev = q.device
    idx = torch.empty(nq, k, dtype=torch.int64, device=dev)
    dst = torch.empty(nq, k, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    ev = R._eval_buffers(R.encode_ids(*args, False, dev), nq, dev)
    ws = torch.empty(R.rerank_topk_workspace_bytes(nq, ng, 512, K1, K2, k, rows), dtype=torch.uint8, device=dev)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        R._rerank_topk_enqueue(planes, nq, ng, K1, K2, LAM, k, rows, idx, dst, ev, status, ws)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        R._rerank_topk_enqueue(planes, nq, ng, K1, K2, LAM, k, rows, idx, dst, ev, status, ws)
    idx.zero_()
    dst.zero_()
    ev["buckets"].fill_(7)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(idx, a[0]) and torch.equal(dst, a[1]) and int(status.item()) == 0
    ranks, pack = R._finalize(ev["buckets"], ev["pos_count"], nq, ev["ids"].max_pos, ev["ovf"])
    assert np.array_equal(ranks.cpu().numpy(), a[2].ranks)


def test_eval_reranked_takes_the_blocked_path_when_the_dense_one_does_not_fit(monkeypatch):
    from ctl_b200.utils.eval_reid import eval_reranked

    feats, pids, cams = O.synth_retrieval(60, 300, 20, 256, 3.0, 9)
    q, g = feats[:60], feats[60:]
    args = (pids[:60], pids[60:], cams[:60], cams[60:])
    dense = eval_reranked(q, g, *args, feat_norm=True)
    monkeypatch.setattr(R, "rerank_fits_dense", lambda *a: False)
    blocked = eval_reranked(q, g, *args, feat_norm=True)
    assert np.array_equal(dense[0], blocked[0]) and dense[1] == blocked[1]
    assert np.array_equal(dense[2], blocked[2]) and np.array_equal(dense[3], blocked[3])
