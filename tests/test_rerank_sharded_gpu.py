"""GPU: the row-blocked k-reciprocal re-ranking sharded over ranks (retrieval.rerank_topk_sharded /
rerank_topk_and_eval_sharded) against the one-GPU path on the same device, with torch.equal throughout.

W ranks are emulated on one device: each runs the protocol in a thread of its own, one at a time, and the exchange
stand-in hands the parts over (shard_exchange.Shards).  The query and gallery features are split unevenly over the
ranks, some ranks holding none; the row shares of the sweeps put boundaries inside the queries and, at W = 2 with
Q = G, exactly at the query / gallery boundary.
"""
import socket

import numpy as np
import pytest
import torch
from shard_exchange import Shards

from ctl_b200 import retrieval as R
from oracle import ctl_oracle as O

pytestmark = pytest.mark.gpu

K1, K2, LAM = 20, 6, 0.3


def _cuts(n, world, seed):
    """Uneven contiguous shards of n rows: rank j holds [c[j], c[j + 1]); some ranks may hold none."""
    rng = np.random.default_rng(seed)
    return np.concatenate([[0], np.sort(rng.integers(0, n + 1, world - 1)), [n]])


def _sharded(world, q, g, k, ids=None, respect=False, k1=K1, k2=K2, lam=LAM, normalize=False, block_rows=None,
             seed=0, qc=None, gc=None):
    qc = _cuts(q.shape[0], world, seed) if qc is None else qc
    gc = _cuts(g.shape[0], world, seed + 1) if gc is None else gc

    def fn(ex):
        j = ex.rank
        ids_args = None
        if ids is not None:
            ids_args = (ids[0], ids[1][gc[j]: gc[j + 1]], ids[2], ids[3][gc[j]: gc[j + 1]], respect)
        return R._rerank_sharded(ex, q[qc[j]: qc[j + 1]], g[gc[j]: gc[j + 1]], k, k1, k2, lam, normalize, block_rows,
                                 ids_args)

    return Shards(world).run(fn)


def _assert_eval_equal(a, b):
    assert np.array_equal(a.cmc, b.cmc)
    assert a.mAP == b.mAP
    assert np.array_equal(a.all_topk, b.all_topk)
    assert np.array_equal(a.ranks, b.ranks)
    assert np.array_equal(a.single_performance, b.single_performance)


def _inverted_sorted(r):
    col_ptr = r["col_ptr"].cpu().numpy()
    nnz = int(col_ptr[-1])
    inv_row, inv_val = r["inv_row"][:nnz].cpu().numpy(), r["inv_val"][:nnz].cpu().numpy()
    seg = np.repeat(np.arange(len(col_ptr) - 1), np.diff(col_ptr))
    o = np.lexsort((inv_row, seg))
    return col_ptr, inv_row[o], inv_val[o]


def _ids(nq, pids, cams, respect_camids):
    q_pids = pids[:nq].copy()
    q_pids[::11] = 5000 + np.arange(len(q_pids[::11]))  # queries without a positive in the gallery
    g_cams = [[int(c), int(c + 2) % 6] for c in cams[nq:]] if respect_camids else cams[nq:]
    return q_pids, pids[nq:], cams[:nq], g_cams


_DATA = {}


def _data(d):
    """N = 2000 with Q = G = 1000: the W = 2 row shares split exactly at the query / gallery boundary."""
    if d not in _DATA:
        feats, pids, cams = O.synth_retrieval(1000, 1000, 60, d, 3.0, 200 + d)
        _DATA[d] = (feats[:1000].cuda(), feats[1000:].cuda(), pids, cams)
    return _DATA[d]


@pytest.mark.parametrize("world", [1, 2, 3, 7])
@pytest.mark.parametrize("block_rows", [1, 7, 128])
@pytest.mark.parametrize("d", [72, 512])
def test_sharded_equals_one_gpu(d, block_rows, world):
    q, g, pids, cams = _data(d)
    nq, k = q.shape[0], 50
    respect = block_rows % 2 == 1
    ids = _ids(nq, pids, cams, respect)
    ref = R.rerank_blocked_stages(q, g, k, K1, K2, LAM, block_rows=block_rows, q_pids=ids[0], g_pids=ids[1],
                                  q_camids=ids[2], g_camids=ids[3], respect_camids=respect)
    assert int(ref["status"].item()) == 0
    ri, rd = R.rerank_topk(q, g, k, K1, K2, LAM, block_rows=block_rows)
    _, _, rev = R.rerank_topk_and_eval(q, g, k, *ids, K1, K2, LAM, respect_camids=respect, block_rows=block_rows)
    outs = _sharded(world, q, g, k, ids, respect, block_rows=block_rows, seed=world * 10 + block_rows)
    ref_inv = _inverted_sorted(ref)
    for r in outs:
        for key in ("rank", "rowmax", "v_idx", "v_val", "v_cnt", "q_idx", "q_val", "q_cnt", "col_ptr"):
            assert torch.equal(r[key], ref[key]), key
        assert all(np.array_equal(a, b) for a, b in zip(_inverted_sorted(r), ref_inv))
        assert torch.equal(r["idx"], ri) and torch.equal(r["dist"], rd)
        _assert_eval_equal(r["eval"], rev)


@pytest.mark.parametrize("lam,k2,normalize,k", [(0.0, 6, False, 10), (1.0, 6, False, 10), (0.3, 1, False, 10),
                                                (0.3, 6, True, 10), (0.3, 6, False, 1), (0.3, 6, False, 128)])
def test_edge_parameters(lam, k2, normalize, k):
    feats, pids, cams = O.synth_retrieval(100, 500, 30, 72, 3.0, 31)
    q, g = feats[:100].cuda(), feats[100:].cuda()
    ids = (pids[:100], pids[100:], cams[:100], cams[100:])
    ri, rd = R.rerank_topk(q, g, k, K1, k2, lam, normalize, block_rows=37)
    _, _, rev = R.rerank_topk_and_eval(q, g, k, *ids, K1, k2, lam, normalize, block_rows=37)
    for r in _sharded(3, q, g, k, ids, k2=k2, lam=lam, normalize=normalize, block_rows=37, seed=k):
        assert torch.equal(r["idx"], ri) and torch.equal(r["dist"], rd)
        _assert_eval_equal(r["eval"], rev)


def test_more_ranks_than_queries():
    """W = 7 and Q = 5: two ranks compute no query of sweep C, and one holds no query features."""
    feats, pids, cams = O.synth_retrieval(5, 400, 20, 72, 3.0, 3)
    q, g = feats[:5].cuda(), feats[5:].cuda()
    ids = (pids[:5], pids[5:], cams[:5], cams[5:])
    ri, rd, rev = R.rerank_topk_and_eval(q, g, 20, *ids, block_rows=64)
    qc = np.array([0, 0, 1, 2, 3, 4, 4, 5])
    for r in _sharded(7, q, g, 20, ids, block_rows=64, qc=qc):
        assert torch.equal(r["idx"], ri) and torch.equal(r["dist"], rd)
        _assert_eval_equal(r["eval"], rev)


def test_duplicated_gallery_rows_tie_across_a_shard_boundary():
    """lambda = 1: the final distance is nd, so gallery rows j and 200 + j tie exactly; they sit on different ranks (data)
    and in different row shares (sweeps), and still come out in column order."""
    feats, _, _ = O.synth_retrieval(60, 200, 20, 72, 3.0, 41)
    g = torch.cat([feats[60:], feats[60:160]]).cuda()
    q = feats[:60].cuda()
    ri, rd = R.rerank_topk(q, g, 40, K1, K2, 1.0, block_rows=17)
    for r in _sharded(2, q, g, 40, lam=1.0, block_rows=17, qc=np.array([0, 30, 60]), gc=np.array([0, 200, 300])):
        assert torch.equal(r["idx"], ri) and torch.equal(r["dist"], rd)
    ties = rd[:, 1:] == rd[:, :-1]
    assert int(ties.sum()) > 100


def test_market_shape_world4_equals_dense():
    nq, ng = 3368, 15913
    feats, pids, cams = O.synth_retrieval(nq, ng, 751, 2048, 3.0, 17)
    q, g = feats[:nq].cuda(), feats[nq:].cuda()
    del feats
    ids = (pids[:nq], pids[nq:], cams[:nq], cams[nq:])
    dense = R.rerank(q, g)
    ref = R.evaluate_matrix(dense, *ids)
    o = torch.sort(dense, dim=1, stable=True).indices[:, :100]
    ri, rd = o, dense.gather(1, o)
    del dense
    for r in _sharded(4, q, g, 100, ids, seed=4):
        assert torch.equal(r["idx"], ri) and torch.equal(r["dist"], rd)
        _assert_eval_equal(r["eval"], ref)


def test_one_rank_nccl_group_equals_one_gpu():
    import torch.distributed as dist

    feats, pids, cams = O.synth_retrieval(150, 700, 30, 256, 3.0, 8)
    q, g = feats[:150].cuda(), feats[150:].cuda()
    ids = (pids[:150], pids[150:], cams[:150], cams[150:])
    ri, rd, rev = R.rerank_topk_and_eval(q, g, 30, *ids, block_rows=100)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        idx, dst, ev = R.rerank_topk_and_eval_sharded(q, g, 30, *ids, block_rows=100, group=dist.group.WORLD)
        idx2, dst2 = R.rerank_topk_sharded(q, g, 30, block_rows=100, group=dist.group.WORLD)
    finally:
        dist.destroy_process_group()
    assert torch.equal(idx, ri) and torch.equal(dst, rd) and torch.equal(idx2, ri) and torch.equal(dst2, rd)
    _assert_eval_equal(ev, rev)
    # group=None: one rank, nothing exchanged
    idx3, dst3, ev3 = R.rerank_topk_and_eval_sharded(q, g, 30, *ids, block_rows=100)
    assert torch.equal(idx3, ri) and torch.equal(dst3, rd)
    _assert_eval_equal(ev3, rev)


def test_status_error_raises_on_every_rank():
    """Identical features: every row maximum is 0."""
    q = torch.ones(20, 64, device="cuda")
    g = torch.ones(50, 64, device="cuda")
    shards = Shards(3)
    with pytest.raises(ValueError, match="no positive maximum"):
        shards.run(lambda ex: R._rerank_sharded(ex, q[ex.rank * 5: ex.rank * 5 + 5 + 5 * (ex.rank == 2)],
                                                 g[ex.rank * 10: ex.rank * 10 + 10 + 20 * (ex.rank == 2)],
                                                 5, K1, K2, LAM, False, 16))
    assert all(isinstance(e, ValueError) for e in shards.errors)
    with pytest.raises(ValueError, match="no positive maximum"):
        R.rerank_topk_sharded(q, g, 5)


def test_two_calls_in_a_row_are_bit_identical():
    feats, pids, cams = O.synth_retrieval(200, 1100, 40, 512, 3.0, 5)
    q, g = feats[:200].cuda(), feats[200:].cuda()
    ids = (pids[:200], pids[200:], cams[:200], cams[200:])
    a = _sharded(3, q, g, 30, ids, block_rows=300)
    b = _sharded(3, q, g, 30, ids, block_rows=300)
    for x, y in zip(a, b):
        assert torch.equal(x["idx"], y["idx"]) and torch.equal(x["dist"], y["dist"])
        _assert_eval_equal(x["eval"], y["eval"])


class _Recorder:
    """Passes every exchange through and keeps its result on the host."""

    def __init__(self, ex):
        self.ex, self.rank, self.world, self.log = ex, ex.rank, ex.world, []

    def objects(self, obj):
        out = self.ex.objects(obj)
        self.log.append(out)
        return out

    def rows(self, t, counts):
        out = self.ex.rows(t, counts)
        self.log.append(out.cpu())
        return out

    def max_(self, t):
        self.ex.max_(t)
        self.log.append(t.cpu())
        return t

    def sum_(self, t):
        self.ex.sum_(t)
        self.log.append(t.cpu())
        return t


class _Replay:
    """One rank alone: every exchange returns what the recorded run got."""

    def __init__(self, rank, world, log):
        self.rank, self.world, self.log, self.i = rank, world, log, 0

    def _next(self):
        self.i += 1
        return self.log[self.i - 1]

    def objects(self, obj):
        return self._next()

    def rows(self, t, counts):
        return self._next().to(t.device)

    def max_(self, t):
        return t.copy_(self._next())

    def sum_(self, t):
        return t.copy_(self._next())


def _device_features(n, ids, d, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    pids = torch.randint(0, ids, (n,), generator=gen, device="cuda")
    cams = torch.randint(0, 6, (n,), generator=gen, device="cuda")
    x = torch.randn(ids, d, generator=gen, device="cuda")[pids]
    x.add_(torch.randn(n, d, generator=gen, device="cuda"), alpha=3.0)
    x = torch.nn.functional.normalize(x, dim=1)
    return x, pids.cpu().numpy(), cams.cpu().numpy()


def test_peak_allocation_per_rank():
    """W = 4 emulated, N = 20 000: rank 0 alone, its exchanges replayed from a recorded run, allocates at most the
    one-GPU workspace plus the gathered features (and their planes) and the outputs."""
    nq, ng, d, k, world = 4000, 16000, 256, 100, 4
    n = nq + ng
    x, pids, cams = _device_features(n, 1000, d, 7)
    q, g = x[:nq], x[nq:]
    ids = (pids[:nq], pids[nq:], cams[:nq], cams[nq:])
    qc, gc = _cuts(nq, world, 1), _cuts(ng, world, 2)
    rec = {}

    def shard_args(j):
        return (q[qc[j]: qc[j + 1]], g[gc[j]: gc[j + 1]], k, K1, K2, LAM, False, None,
                (ids[0], ids[1][gc[j]: gc[j + 1]], ids[2], ids[3][gc[j]: gc[j + 1]], False))

    def fn(ex):
        if ex.rank == 0:
            ex = rec["ex"] = _Recorder(ex)
        return R._rerank_sharded(ex, *shard_args(ex.rank))["idx"]

    full = Shards(world).run(fn)[0]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    r = R._rerank_sharded(_Replay(0, world, rec["ex"].log), *shard_args(0))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert torch.equal(r["idx"], full)
    ws = R.rerank_topk_workspace_bytes(nq, ng, d, K1, K2, k, R.rerank_block_rows(nq, ng))
    gathered = 3 * n * d * 4  # the gathered q and g, their concatenation, the planes (2 fp16 planes per row)
    assert peak <= ws + gathered + (64 << 20), (peak, ws)
