"""CPU: the host side of the sharded row-blocked re-ranking -- the row shares of the sweeps, the padded all-gather of
uneven shards (gloo, world 2, host tensors) and argument rejection, which must raise the same error on every rank
before any data is exchanged."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from ctl_b200 import retrieval as R


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.parametrize("world", range(1, 10))
def test_row_shares_cover_every_row_once(world):
    for n in (0, 1, 2, 3, 7, 8, 9, 400, 2000, 250000):
        shares = R.row_shares(n, world)
        assert len(shares) == world
        covered = np.concatenate([np.arange(lo, hi) for lo, hi in shares])
        assert np.array_equal(covered, np.arange(n)), (n, world)
        sizes = [hi - lo for lo, hi in shares]
        assert max(sizes) - min(sizes) <= 1
        if world > n:
            assert sizes.count(0) == world - n  # ranks without query rows


def _run(world, target):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=180) for _ in procs], key=lambda x: x[0])
    for p in procs:
        p.join(60)
    return [x[1] for x in res]


def _exchange_worker(rank, world, port, out_q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ex = R.ShardExchange(dist.group.WORLD)
    out = {"rank": ex.rank, "world": ex.world}
    counts = [3, 0] if world == 2 else None
    a = torch.arange(counts[rank] * 5, dtype=torch.int32).reshape(-1, 5) + 100 * rank
    out["int_uneven"] = ex.rows(a, counts).numpy()
    b = torch.full((rank + 2, 2, 3), float(rank) + 0.5)          # [2, 2, 3] and [3, 2, 3]
    out["float_uneven"] = ex.rows(b, [2, 3]).numpy()
    c = torch.arange(4, dtype=torch.int64) * (rank + 1)            # even shards take the unpadded path
    out["even"] = ex.rows(c, [4, 4]).numpy()
    out["objects"] = ex.objects({"r": rank})
    m = torch.tensor([rank, 1 - rank], dtype=torch.int32)
    out["max"] = ex.max_(m).numpy()
    t = torch.tensor([[rank + 1, 10 * rank], [-3, 7]], dtype=torch.int32)
    out["sum"] = ex.sum_(t).numpy()
    out_q.put((rank, out))
    dist.destroy_process_group()


def test_padded_all_gather_of_uneven_shards_world2_gloo():
    res = _run(2, _exchange_worker)
    for rank, out in enumerate(res):
        assert out["rank"] == rank and out["world"] == 2
        assert np.array_equal(out["int_uneven"], np.arange(15, dtype=np.int32).reshape(3, 5))
        assert np.array_equal(out["float_uneven"], np.concatenate([np.full((2, 2, 3), 0.5), np.full((3, 2, 3), 1.5)]))
        assert np.array_equal(out["even"], np.concatenate([np.arange(4), 2 * np.arange(4)]))
        assert out["objects"] == [{"r": 0}, {"r": 1}]
        assert np.array_equal(out["max"], [1, 1])
        assert np.array_equal(out["sum"], [[3, 10], [-6, 14]])


class _Spy(R.ShardExchange):
    """Counts the data exchanges (everything but the first object gather)."""

    data_calls = 0

    def rows(self, t, counts):
        self.data_calls += 1
        return super().rows(t, counts)

    def max_(self, t):
        self.data_calls += 1
        return super().max_(t)

    def sum_(self, t):
        self.data_calls += 1
        return super().sum_(t)


def _reject_worker(rank, world, port, out_q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    R.N.require_cuda = lambda *a: None  # host tensors: the checks below all come before any device work
    g = torch.Generator().manual_seed(rank)

    def feats(n, d):
        return torch.randn(n, d, generator=g)

    pids = np.arange(8)
    cases = {
        "d differs": dict(q=feats(3, 64 if rank == 0 else 72), g=feats(4, 64 if rank == 0 else 72)),
        "k > G": dict(q=feats(3, 64), g=feats(2 + rank, 64), k=6),
        "d % 8": dict(q=feats(3, 60), g=feats(4, 60)),
        "k > 128": dict(q=feats(100, 64), g=feats(100, 64), k=129),
        "k1 < 1": dict(q=feats(3, 64), g=feats(4, 64), k1=0),
        "3-D shard": dict(q=feats(3, 64) if rank == 0 else torch.zeros(3, 64, 1), g=feats(4, 64)),
        "g_pids length": dict(q=feats(3, 64), g=feats(4, 64), ids=(np.arange(6), pids[: 4 - rank], np.zeros(6),
                                                                   np.zeros(4))),
        "q_pids length": dict(q=feats(3, 64), g=feats(4, 64), ids=(np.arange(5 + rank), pids[:4], np.zeros(6),
                                                                   np.zeros(4))),
    }
    out = {}
    for name, c in cases.items():
        ex = _Spy(dist.group.WORLD)
        ids = c.get("ids")
        if ids is not None:
            ids = ids + (False,)
        try:
            R._rerank_sharded(ex, c["q"], c["g"], c.get("k", 5), c.get("k1", 20), 6, 0.3, False, None, ids)
            out[name] = ("no error", "", ex.data_calls)
        except Exception as e:  # noqa: BLE001 -- the type and message are compared across ranks
            out[name] = (type(e).__name__, str(e), ex.data_calls)
    out_q.put((rank, out))
    dist.destroy_process_group()


def test_argument_rejection_is_the_same_on_every_rank_world2_gloo():
    r0, r1 = _run(2, _reject_worker)
    assert r0.keys() == r1.keys()
    for name in r0:
        assert r0[name] == r1[name], name
        kind, msg, calls = r0[name]
        assert kind in ("ValueError",), (name, kind, msg)
        assert calls == 0, name  # raised before any data exchange
    assert "rank 1" in r0["3-D shard"][1]
    assert "widths differ" in r0["d differs"][1]
