"""GPU: k-reciprocal re-ranking (csrc/rerank.cu) stage by stage against the float64 oracle (oracle/rerank_oracle.py),
end to end from features, determinism, and CMC / mAP from a materialised matrix (ctl_eval_matrix_collect / _count).

Tolerance of the final distances: 1e-5 absolute against float64, teacher-forced on the engine's own nd (u = 2^-24).
- Values: every V value lies in [0, 1] and every row of V sums to 1 (a softmax; the query expansion averages such rows).
  So a Jaccard sum s has at most k2 (k1 + 1)(h + 2) fp32 terms (1512 at k1 = 20, k2 = 6), all >= 0, with total <= 1.
- A weight w = e / S: e is an fp32 exp (<= 2 ulp).  S sums <= 252 terms, lane-strided (<= 8 per lane), then a 5-level
  shuffle tree, so <= 13 u relative.  The division adds one rounding.  So w is within ~1e-6 relative.
- The mean of k2 rows adds <= k2 u.  So every expanded V value is within ~1.5e-6 relative, and so is every min.
- s adds its <= 1512 terms one after the other in shared memory (fixed column order).  Worst case 1512 u = 9e-5
  relative.  Rounding errors of a fixed-order sum of non-negative terms add like a random walk: sqrt(1512) u = 2.3e-6.
  So |s - s64| is a few 1e-6 for s <= 1.
- 1 - s / (2 - s) has slope in [-2, -1/2] on s in [0, 1], and the blend multiplies by 1 - lambda <= 1.
So 1e-5 holds with margin, and it still catches any wrong set, weight or missing term: each of those moves a
distance by at least about 1 / (k2 (k1 + 1)(h + 2)) = 7e-4.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from ctl_b200 import retrieval as R
from oracle import ctl_oracle as O
from oracle import rerank_oracle as RO

pytestmark = pytest.mark.gpu


def _dyadic(nq, ng, d, seed, ids=30):
    feats, pids, cams = O.synth_retrieval(nq, ng, ids, d, 3.0, seed, dyadic=True)
    return feats, pids, cams


def _gap_fixture(n_clusters, d, seed):
    """Clusters of 6 points made of two tight sub-clusters of 3: for k1 = 5 (h + 1 = 3 neighbours, k1 + 1 = 6) every
    set boundary falls between sub-clusters or clusters, far from any rounding."""
    rng = np.random.default_rng(seed)
    centres = 10.0 * rng.standard_normal((n_clusters, d))
    subs = np.repeat(centres, 2, axis=0) + rng.standard_normal((2 * n_clusters, d))
    pts = np.repeat(subs, 3, axis=0) + 0.1 * rng.standard_normal((6 * n_clusters, d))
    return torch.from_numpy(pts[rng.permutation(len(pts))].astype(np.float32))


def _csr(idx, val, cnt, n):
    idx, val, cnt = idx.cpu().numpy(), val.cpu().numpy().astype(np.float64), cnt.cpu().numpy()
    rows = np.repeat(np.arange(n), cnt)
    mask = np.arange(idx.shape[1])[None, :] < cnt[:, None]
    return sp.csr_matrix((val[mask], (rows, idx[mask])), shape=(n, n))


def _check_rows(idx, val, cnt, ref: sp.csr_matrix, atol, rows=None):
    idx, val, cnt = idx.cpu().numpy(), val.cpu().numpy(), cnt.cpu().numpy()
    for i in range(ref.shape[0]) if rows is None else rows:
        cols, vals = RO.csr_rows(ref, i)
        assert cnt[i] == len(cols), (i, cnt[i], len(cols))
        assert np.array_equal(idx[i, : cnt[i]], cols), i
        assert np.all(np.diff(idx[i, : cnt[i]]) > 0)
        np.testing.assert_allclose(val[i, : cnt[i]], vals, rtol=0, atol=1e-6, err_msg=str(i))


def _check_stages(r, nq, k1, k2, lam):
    """Every stage against the oracle applied to the previous GPU stage's output."""
    n = r["nd"].shape[0]
    nd = r["nd"].cpu().numpy()
    kr = r["plan"].kr
    assert int(r["status"].item()) == 0
    rank = r["rank"].cpu().numpy().astype(np.int64)
    assert np.array_equal(rank, RO.rank_table(nd, kr))
    assert np.array_equal(rank, np.argsort(nd, axis=1, kind="stable")[:, :kr])
    V = RO.expansion(rank, k1, nd)
    _check_rows(r["v_idx"], r["v_val"], r["v_cnt"], V, 1e-6)
    V_gpu = _csr(r["v_idx"], r["v_val"], r["v_cnt"], n)
    V_qe = RO.query_expansion(rank, V_gpu, k2)
    if k2 > 1:
        _check_rows(r["q_idx"], r["q_val"], r["q_cnt"], V_qe, 1e-6)
    else:
        assert r["q_idx"] is r["v_idx"]
    Q_gpu = _csr(r["q_idx"], r["q_val"], r["q_cnt"], n)
    # inverted index: the gallery rows (local) holding each column, with their values
    col_ptr = r["col_ptr"].cpu().numpy()
    inv_row, inv_val = r["inv_row"].cpu().numpy(), r["inv_val"].cpu().numpy()
    Gc = Q_gpu[nq:].tocsc()
    assert col_ptr[0] == 0 and col_ptr[-1] == Gc.nnz
    for c in range(n):
        lo, hi = col_ptr[c], col_ptr[c + 1]
        o = np.argsort(inv_row[lo:hi])
        assert np.array_equal(inv_row[lo:hi][o], Gc.indices[Gc.indptr[c]: Gc.indptr[c + 1]]), c
        assert np.array_equal(inv_val[lo:hi][o].astype(np.float64), Gc.data[Gc.indptr[c]: Gc.indptr[c + 1]]), c
    out_tf = RO.jaccard_blend(RO.jaccard_sums(Q_gpu, nq), nd[:nq, nq:], lam)
    out = r["out"].cpu().numpy()
    np.testing.assert_allclose(out, out_tf, rtol=0, atol=1e-5)
    # the whole float64 chain from the engine's nd
    np.testing.assert_allclose(out, RO.rerank_sparse(nd, nq, k1, k2, lam)["out"], rtol=0, atol=1e-5)
    return nd, rank


@pytest.mark.parametrize("d", [72, 512, 2048])
@pytest.mark.parametrize("n", [300, 2000])
def test_stages_teacher_forced(n, d):
    nq = n // 5
    feats, _, _ = _dyadic(nq, n - nq, d, seed=n + d)
    q, g = feats[:nq].cuda(), feats[nq:].cuda()
    r = R.rerank_stages(q, g, 20, 6, 0.3)
    _check_stages(r, nq, 20, 6, 0.3)
    assert torch.equal(r["out"], R.rerank(q, g, 20, 6, 0.3))


@pytest.mark.parametrize("k1,k2", [(1, 1), (2, 2), (7, 3), (5, 9), (20, 1)])
def test_stages_small_k(k1, k2):
    feats, _, _ = _dyadic(60, 240, 72, seed=k1 * 10 + k2)
    r = R.rerank_stages(feats[:60].cuda(), feats[60:].cuda(), k1, k2, 0.3)
    _check_stages(r, 60, k1, k2, 0.3)


def test_end_to_end_dyadic_from_features():
    """Dyadic features: the GEMM is exact, so the oracle run from the features has the engine's nd bit for bit, and
    ranks and sets are exact."""
    nq, n = 80, 400
    feats, _, _ = _dyadic(nq, n - nq, 72, seed=7)
    r = R.rerank_stages(feats[:nq].cuda(), feats[nq:].cuda(), 20, 6, 0.3)
    nd_host = RO.nd_from_features(feats.numpy())
    assert np.array_equal(r["nd"].cpu().numpy(), nd_host)
    ref = RO.rerank_loop(nd_host, nq, 20, 6, 0.3)
    assert np.array_equal(r["rank"].cpu().numpy(), ref["rank"][:, :21])
    V = sp.csr_matrix(ref["V"])
    _check_rows(r["v_idx"], r["v_val"], r["v_cnt"], V, 1e-6)
    _check_rows(r["q_idx"], r["q_val"], r["q_cnt"], sp.csr_matrix(ref["V_qe"]), 1e-6)
    np.testing.assert_allclose(r["out"].cpu().numpy(), ref["out"], rtol=0, atol=1e-5)


@pytest.mark.parametrize("normalize", [False, True])
def test_end_to_end_gap_separated_from_features(normalize):
    k1, k2, lam, nq = 5, 3, 0.3, 60
    x = _gap_fixture(60, 64, seed=3)
    nd_host = RO.nd_from_features(x.numpy().astype(np.float64), normalize)
    s = np.sort(nd_host, axis=1)
    for b in (RO.half_k(k1) + 1, k1 + 1, k2):  # the set boundaries
        assert (s[:, b] - s[:, b - 1]).min() > 1e-3, b
    r = R.rerank_stages(x[:nq].cuda(), x[nq:].cuda(), k1, k2, lam, normalize=normalize)
    rank = r["rank"].cpu().numpy()
    ref = RO.rerank_sparse(nd_host, nq, k1, k2, lam)
    for b in (RO.half_k(k1) + 1, k1 + 1, k2):
        assert np.array_equal(np.sort(rank[:, :b], 1), np.sort(ref["rank"][:, :b], 1)), b
    v_idx, v_cnt = r["v_idx"].cpu().numpy(), r["v_cnt"].cpu().numpy()
    for i in range(x.shape[0]):
        assert np.array_equal(v_idx[i, : v_cnt[i]], RO.csr_rows(ref["V"], i)[0]), i
    np.testing.assert_allclose(r["out"].cpu().numpy(), ref["out"], rtol=0, atol=1e-4)


def test_lambda_one_and_k2_one():
    feats, _, _ = _dyadic(50, 250, 72, seed=11)
    q, g = feats[:50].cuda(), feats[50:].cuda()
    r = R.rerank_stages(q, g, 20, 6, 1.0)
    assert torch.equal(r["out"], r["nd"][:50, 50:])
    r1 = R.rerank_stages(q, g, 20, 1, 0.3)
    assert r1["q_idx"] is r1["v_idx"]
    _check_stages(r1, 50, 20, 1, 0.3)
    assert torch.equal(R.rerank(q, g, 20, 1, 0.3), r1["out"])


def test_repeats_and_graph_replay_are_bit_identical():
    feats, _, _ = O.synth_retrieval(200, 1100, 40, 512, 3.0, 5)
    q, g = feats[:200].cuda(), feats[200:].cuda()
    a, b = R.rerank(q, g), R.rerank(q, g)
    assert torch.equal(a, b)
    planes = R._rerank_inputs(q, g, False)
    out = torch.empty(200, 1100, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = torch.empty(R.N.lib().ctl_rerank_workspace_bytes(200, 1100, 20, 6), dtype=torch.uint8, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        R._rerank_enqueue(planes, 200, 1100, 20, 6, 0.3, out, status, ws)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        R._rerank_enqueue(planes, 200, 1100, 20, 6, 0.3, out, status, ws)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a) and int(status.item()) == 0


def test_identical_features_are_rejected():
    x = torch.ones(10, 64, device="cuda")
    with pytest.raises(ValueError):
        R.rerank(x[:4], x[4:])


def test_drop_ins():
    from ctl_b200.utils.eval_reid import eval_reranked
    from ctl_b200.utils.re_ranking import re_ranking

    feats, pids, cams = O.synth_retrieval(60, 300, 20, 256, 3.0, 9)
    q, g = feats[:60], feats[60:]
    out = re_ranking(q, g, 20, 6, 0.3)
    assert out.dtype == np.float32 and out.shape == (60, 300)
    assert np.array_equal(out, R.rerank(q.cuda(), g.cuda()).cpu().numpy())
    with pytest.raises(NotImplementedError):
        re_ranking(q, g, 20, 6, 0.3, local_distmat=np.zeros((360, 360)))
    cmc, mAP, topk, single = eval_reranked(q, g, pids[:60], pids[60:], cams[:60], cams[60:], feat_norm=True)
    ref = O.eval_func(O.rank_indices(R.rerank(q.cuda(), g.cuda(), normalize=True).cpu().numpy()), pids[:60],
                      pids[60:], cams[:60], cams[60:], 50)
    assert np.array_equal(cmc, ref[0]) and abs(mAP - ref[1]) < 1e-12
    np.testing.assert_allclose(single[:, 2], ref[3][:, 2], rtol=1e-12)


@pytest.mark.parametrize("respect_camids", [False, True])
def test_evaluate_matrix_against_eval_func(respect_camids):
    """Integer distances (exact ties, positives among them) and queries whose identity is not in the gallery."""
    nq, ng = 70, 900
    feats, pids, cams = _dyadic(nq, ng, 72, seed=21, ids=25)
    q_pids, g_pids = pids[:nq].copy(), pids[nq:]
    q_pids[::9] = 1000 + np.arange(len(q_pids[::9]))  # no positive in the gallery
    M = torch.round(R.dist_matrix(feats[:nq].cuda(), feats[nq:].cuda()) * 2.0)
    Mh = M.cpu().numpy()
    assert (np.diff(np.sort(Mh, 1), axis=1) == 0).mean() > 0.5
    q_cams = cams[:nq]
    g_cams = [[int(c), int(c + 1) % 6] for c in cams[nq:]] if respect_camids else cams[nq:]
    res = R.evaluate_matrix(M, q_pids, g_pids, q_cams, g_cams, 50, respect_camids)
    cmc, mAP, topk, single = O.eval_func(O.rank_indices(Mh), q_pids, g_pids, q_cams, g_cams, 50, respect_camids)
    assert np.array_equal(res.cmc, cmc)
    assert abs(res.mAP - mAP) < 1e-12
    np.testing.assert_allclose(res.all_topk, topk, rtol=1e-12)
    assert len(res.single_performance) == len(single) < nq
    np.testing.assert_allclose(res.single_performance.astype(np.float64), single.astype(np.float64), rtol=1e-14)
    # a strided view: the leading dimension is the row stride
    wide = torch.zeros(nq, ng + 17, device="cuda")
    wide[:, :ng] = M
    res2 = R.evaluate_matrix(wide[:, :ng], q_pids, g_pids, q_cams, g_cams, 50, respect_camids)
    assert np.array_equal(res2.ranks, res.ranks) and res2.mAP == res.mAP


def test_evaluate_matrix_equals_evaluate_streamed():
    nq, ng = 150, 2500
    feats, pids, cams = O.synth_retrieval(nq, ng, 60, 2048, 3.0, 13)
    q, g = feats[:nq].cuda(), feats[nq:].cuda()
    a = R.evaluate_matrix(R.dist_matrix(q, g), pids[:nq], pids[nq:], cams[:nq], cams[nq:])
    b = R.evaluate_streamed(R.build_planes(q), R.build_planes(g), pids[:nq], pids[nq:], cams[:nq], cams[nq:])
    assert np.array_equal(a.ranks, b.ranks)
    assert np.array_equal(a.cmc, b.cmc) and a.mAP == b.mAP
    assert np.array_equal(a.single_performance, b.single_performance)


def test_market_shape_sampled_rows():
    """Q = 3368, G = 15913, d = 2048 (Market-1501's evaluation shape), 751 identities: the stages teacher-forced on a
    fixed sample of 64 query rows, with V built on the host for every row from the engine's rank table and gathered nd
    values."""
    nq, ng, k1, k2, lam = 3368, 15913, 20, 6, 0.3
    feats, _, _ = O.synth_retrieval(nq, ng, 751, 2048, 3.0, 17)
    q, g = feats[:nq].cuda(), feats[nq:].cuda()
    del feats
    r = R.rerank_stages(q, g, k1, k2, lam)
    n = nq + ng
    sample = np.sort(np.random.default_rng(0).choice(nq, 64, replace=False))
    nd_dev = r["nd"]
    rank = r["rank"].cpu().numpy().astype(np.int64)
    rows_nd = nd_dev[torch.from_numpy(sample).cuda()].cpu().numpy()
    assert np.array_equal(rank[sample], np.argsort(rows_nd, axis=1, kind="stable")[:, : r["plan"].kr])

    def gather(rows, cols):
        return nd_dev[torch.from_numpy(rows).cuda(), torch.from_numpy(cols).cuda()].cpu().numpy()

    V = RO.expansion(rank, k1, gather)
    _check_rows(r["v_idx"], r["v_val"], r["v_cnt"], V, 1e-6)
    V_gpu = _csr(r["v_idx"], r["v_val"], r["v_cnt"], n)
    V_qe = RO.query_expansion(rank, V_gpu, k2)
    _check_rows(r["q_idx"], r["q_val"], r["q_cnt"], V_qe, 1e-6, rows=sample)
    Q_gpu = _csr(r["q_idx"], r["q_val"], r["q_cnt"], n)
    s = RO.jaccard_sums(Q_gpu, nq, queries=list(sample))
    ref = RO.jaccard_blend(s, rows_nd[:, nq:], lam)
    np.testing.assert_allclose(r["out"][torch.from_numpy(sample).cuda()].cpu().numpy(), ref, rtol=0, atol=1e-5)
