"""CPU, world_size 2, gloo: the host-side logic of the sharded (N > 1) retrieval path --
the top-k merge of the streamed passes (every rank's k best packed keys all-gathered over ShardExchange, one sort of
the unsigned keys per row gives the canonical (distance, index) order), exchange 1 of the streamed
passes (retrieval._gather_keys over ShardExchange: every rank's positives' keys, unused slots
masked), the all-reduce of the integer bucket counts (ShardExchange.sum_) -- with the device
kernels (and the row sort) emulated in numpy from the oracle's distance matrix."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import ctl_oracle as O


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _key(d, idx):
    b = d.astype(np.float32).view(np.uint32).astype(np.uint64)
    ordb = np.where(b & np.uint64(0x80000000), ~b & np.uint64(0xFFFFFFFF), b | np.uint64(0x80000000))
    return (ordb << np.uint64(32)) | idx.astype(np.uint64)


def _worker(rank, world, port, out_q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import ctl_b200  # noqa: F401
    from ctl_b200 import retrieval as R

    nq, ng, k = 40, 600, 25
    feats, pids, cams = O.synth_retrieval(nq, ng, 30, 128, 2.0, 21, num_cams=3)
    D = O.get_euclidean(feats[:nq], feats[nq:]).numpy()
    shard = np.array_split(np.arange(ng), world)[rank]
    off = int(shard[0])
    Dl = D[:, shard]
    ex = R.ShardExchange(dist.group.WORLD)
    # --- top-k: local ascending lists with GLOBAL indices, their keys all-gathered and sorted ---------------
    order = np.argsort(Dl, axis=1, kind="stable")[:, :k]
    keys_l = R.pack_keys(torch.from_numpy(np.take_along_axis(Dl, order, 1)), torch.from_numpy(order + off))
    best = ex.rows(keys_l, [nq] * world).view(world, nq, k).permute(1, 0, 2).reshape(nq, world * k)
    merged = np.sort(best.numpy().view(np.uint64), axis=1)[:, :k]  # ctl_sort_key_rows + ctl_topk_emit on the device
    midx = (merged & np.uint64(0xFFFFFFFF)).astype(np.int64)
    o = (merged >> np.uint64(32)).astype(np.uint32)
    mdst = np.where(o & 0x80000000, o ^ 0x80000000, ~o).astype(np.uint32).view(np.float32)
    ref = np.argsort(D, axis=1, kind="stable")[:, :k]
    ok_topk = np.array_equal(midx, ref) and np.array_equal(mdst, np.take_along_axis(D, ref, 1))
    # --- eval: collect (emulated) -> all-gather keys -> sort -> count (emulated) -> all-reduce ----
    gp, gc = pids[nq:][shard], cams[nq:][shard]
    same = gp[None, :] == pids[:nq, None]
    junk = same & (gc[None, :] == cams[:nq, None])
    pos = same & ~junk
    max_pos = int(np.bincount(pids[nq:]).max())
    keys = np.full((nq, max_pos), 12345, dtype=np.uint64)  # unused slots: whatever the collect left there
    cnt = pos.sum(1).astype(np.int32)
    allk = _key(Dl, np.broadcast_to(shard[None, :], Dl.shape))
    for q in range(nq):
        keys[q, : cnt[q]] = allk[q][pos[q]]
    gk, gcnt = R._gather_keys(ex, torch.from_numpy(keys.view(np.int64)), torch.from_numpy(cnt))
    ok_shape = tuple(gk.shape) == (nq, world * max_pos)
    gk = np.sort(gk.numpy().view(np.uint64), axis=1)  # ctl_sort_key_rows over the whole row: unused slots sort last
    gcnt = gcnt.numpy()
    buckets = np.zeros((nq, max_pos + 1), dtype=np.int32)
    for q in range(nq):
        thr = np.sort(gk[q, : gcnt[q]])
        gk[q, : gcnt[q]] = thr
        kept = allk[q][~junk[q]]
        j = np.searchsorted(thr, kept, side="right")
        np.add.at(buckets[q], j[j < gcnt[q]], 1)
    buckets = ex.sum_(torch.from_numpy(buckets)).numpy()
    ranks = np.full((nq, max_pos), -1, dtype=np.int32)
    ap = np.full(nq, np.nan)
    for q in range(nq):
        n = gcnt[q]
        if n:
            r = np.cumsum(buckets[q, :n]) + 1
            ranks[q, :n] = r
            ap[q] = np.sum((np.arange(n) + 1.0) / r) / n
    res = R._aggregate(ranks, ap, gcnt, pids[:nq], ng, 50)
    cmc, mAP, topk, single = O.eval_func(O.rank_indices(D), pids[:nq], pids[nq:], cams[:nq], cams[nq:], 50)
    ok_eval = np.array_equal(res.cmc, cmc) and abs(res.mAP - mAP) < 1e-12 and np.allclose(res.all_topk, topk)
    ok_eval = ok_eval and ok_shape
    if rank == 0:
        out_q.put((ok_topk, ok_eval))
    dist.destroy_process_group()


def test_sharded_key_merge_and_key_exchange_world2_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    ok_topk, ok_eval = q.get(timeout=180)
    for p in procs:
        p.join(60)
    assert ok_topk, "merged per-shard top-k differs from the global stable ranking"
    assert ok_eval, "sharded CMC/mAP differs from eval_func on the full ranking"


def _grad_worker(rank, world, port, out_q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import ctl_b200  # noqa: F401
    from ctl_b200 import parallel

    g = torch.Generator().manual_seed(100 + rank)
    shapes = [(64, 3, 7, 7), (64,), (256, 64, 1, 1), (751, 2048), (5,)]
    params = [torch.nn.Parameter(torch.zeros(s)) for s in shapes]
    for p_ in params:
        p_.grad = torch.randn(p_.shape, generator=g)
    local = [p_.grad.clone() for p_ in params]
    calls = parallel.allreduce_gradients(params, bucket_bytes=1 << 20)  # small buckets: several collectives
    gathered = [[torch.empty_like(t) for _ in range(world)] for t in local]
    for lst, t in zip(gathered, local):
        dist.all_gather(lst, t)
    ok = all(torch.allclose(p_.grad, torch.stack(lst).mean(0), rtol=0, atol=1e-7) for p_, lst in zip(params, gathered))
    # GradientReducer: one flat buffer, no copy-back; the second step starts from the re-pointed views of the first
    red = parallel.GradientReducer(params)
    for step in range(2):
        for p_ in params:
            p_.grad = torch.randn(p_.shape, generator=g)
        local2 = [p_.grad.clone() for p_ in params]
        red.allreduce_mean()
        for p_, t in zip(params, local2):
            lst = [torch.empty_like(t) for _ in range(world)]
            dist.all_gather(lst, t)
            ok = ok and torch.allclose(p_.grad, torch.stack(lst).mean(0), rtol=0, atol=1e-7)
        ok = ok and all(p_.grad.data_ptr() == v.data_ptr() for p_, v in zip(params, red.views))
    pids = np.arange(37)
    mine = parallel.shard_pids(pids, world, rank)
    sizes = [torch.tensor([len(mine)]) for _ in range(world)]
    dist.all_gather(sizes, torch.tensor([len(mine)]))
    ok_shard = sum(int(t) for t in sizes) == 37 and np.array_equal(mine, np.array_split(pids, world)[rank])
    out_q.put((rank, bool(ok), calls, bool(ok_shard)))
    dist.destroy_process_group()


def test_gradient_allreduce_and_pid_sharding_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_grad_worker, args=(r, 2, port, q)) for r in range(2)]
    for p_ in procs:
        p_.start()
    res = [q.get(timeout=120) for _ in procs]
    for p_ in procs:
        p_.join(60)
    assert all(ok and ok_shard for _, ok, _, ok_shard in res), res
    assert all(calls >= 2 for _, _, calls, _ in res), res
