"""Row-blocked k-reciprocal re-ranking sharded over ranks (retrieval.rerank_topk_and_eval_sharded) at BASELINE config 5:
Q = 50 000, G = 200 000, d = 2048, 20 000 identities, sigma = 3, generated on the device from a seed (the recipe of
tools/bench_rerank_blocked.py); k = 100, k1 = 20, k2 = 6, lambda = 0.3, the default block.

  torchrun --nproc-per-node W tools/bench_rerank_sharded.py
      queries and gallery split evenly over the W ranks: medians of --reps sharded calls with their range, each timed
      by the host clock between two barriers after a device synchronise (all ranks in step).  Then a bit-identity check
      (torch.equal on idx, dist, ranks, AP and CMC) of a --check-q x --check-g sub-problem, sharded, against rank 0
      running rerank_topk_and_eval alone.
  python tools/bench_rerank_sharded.py --emulate-world W
      one GPU: rank 0's share of a W-rank run -- its row share of sweeps A and B, the whole query expansion + inverted
      index, its query share of sweep C and its finalize -- on the tables of an untimed one-GPU run (which stands in for
      the other ranks' rows), in --reps windows alternated with the one-GPU rerank_topk_and_eval (CUDA events), and the
      bytes each all-gather leaves on every rank.  That is per-rank compute at W on one H100; the collectives' time is
      not measured.
Prints one JSON line per measurement with the card's name and power limit.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import ctl_b200  # noqa: E402,F401
from ctl_b200 import retrieval as R  # noqa: E402
from tools.bench_basic import card  # noqa: E402

K1, K2 = 20, 6


def features(nq, ng, d, nid, seed=0):
    n = nq + ng
    gen = torch.Generator(device="cuda").manual_seed(seed)
    pid = torch.randint(0, nid, (n,), generator=gen, device="cuda")
    cam = torch.randint(0, 6, (n,), generator=gen, device="cuda")
    x = torch.randn(nid, d, generator=gen, device="cuda")[pid]
    x.add_(torch.randn(n, d, generator=gen, device="cuda"), alpha=3.0)
    x = torch.nn.functional.normalize(x, dim=1)
    return x, pid.cpu().numpy(), cam.cpu().numpy()


def med(ts):
    ts = sorted(ts)
    return round(ts[len(ts) // 2], 3), [round(ts[0], 3), round(ts[-1], 3)]


def exchange_bytes(nq, ng, d, k, max_pos):
    """Bytes each all-gather leaves on every rank (a rank receives (W - 1) / W of them)."""
    n = nq + ng
    pl = R.rerank_plan(nq, ng, K1, K2)
    return {"features": n * d * 4, "rank_table": n * pl.kr * 4 + n * 4, "V": n * pl.v_cap * 8 + n * 4,
            "results": nq * k * 12 + nq * max_pos * 4 + nq * 3 * 8}


def emulate(a, name, power):
    nq, ng, d, k, world = a.nq, a.ng, a.d, a.k, a.emulate_world
    n = nq + ng
    x, pids, cams = features(nq, ng, d, a.ids)
    q, g = x[:nq], x[nq:]
    ids = (pids[:nq], pids[nq:], cams[:nq], cams[nq:])
    dev = q.device
    r = R.rerank_blocked_stages(q, g, k, K1, K2, q_pids=ids[0], g_pids=ids[1], q_camids=ids[2], g_camids=ids[3])
    ref_idx, ref_dist = r["idx"].clone(), r["dist"].clone()
    enc = R.encode_ids(*ids, False, dev)
    (lo, hi), (qlo, qhi) = R.row_shares(n, world)[0], R.row_shares(nq, world)[0]
    names = ("A", "B", "qe_invert", "C")

    def share():
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        ev[0].record()
        blk = torch.empty(min(r["block_rows"], hi - lo) * n, dtype=torch.float32, device=dev)
        R._rerank_sweep_a(r, lo, hi, blk)
        ev[1].record()
        R._rerank_sweep_b(r, lo, hi, blk, K1, K2)
        ev[2].record()
        del blk
        R._rerank_qe_invert(r, K1, K2)
        ev[3].record()
        e = R._eval_buffers(enc, nq, dev)
        R._rerank_sweep_c(r, qlo, qhi, e)
        R._finalize(e["buckets"][qlo:qhi], e["pos_count"][qlo:qhi], qhi - qlo, enc.max_pos, e["ovf"])
        ev[4].record()
        torch.cuda.synchronize()
        return [ev[i].elapsed_time(ev[i + 1]) / 1e3 for i in range(4)]

    def one_gpu():
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        R.rerank_topk_and_eval(q, g, k, *ids)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3

    share()
    one_gpu()
    ts_share, ts_one, stages = [], [], {s: [] for s in names}
    for _ in range(a.reps):
        st = share()
        ts_share.append(sum(st))
        for s, t in zip(names, st):
            stages[s].append(t)
        ts_one.append(one_gpu())
    assert torch.equal(r["idx"], ref_idx) and torch.equal(r["dist"], ref_dist)  # rank 0's rows recomputed, same bits
    m_s, rng_s = med(ts_share)
    m_o, rng_o = med(ts_one)
    res = {"mode": f"per-rank compute at W = {world} on one H100; collective time not measured", "gpu": name,
           "power_limit": power, "nq": nq, "ng": ng, "d": d, "k": k, "world": world, "block_rows": r["block_rows"],
           "rank0_rows": [lo, hi], "rank0_queries": [qlo, qhi], "rank0_share_s": m_s, "rank0_share_min_max": rng_s,
           "rank0_stages_s": {s: med(stages[s])[0] for s in names}, "one_gpu_s": m_o, "one_gpu_min_max": rng_o,
           "windows": a.reps, "gathered_bytes_per_rank": exchange_bytes(nq, ng, d, k, enc.max_pos)}
    print(json.dumps(res), flush=True)


def distributed(a, name, power):
    import torch.distributed as dist

    dist.init_process_group("nccl")
    rank, world = dist.get_rank(), dist.get_world_size()
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))

    def shard(nq, ng, d, seed):
        x, pids, cams = features(nq, ng, d, a.ids, seed)
        (q0, q1), (g0, g1) = R.row_shares(nq, world)[rank], R.row_shares(ng, world)[rank]
        local = (x[q0:q1].clone(), x[nq + g0: nq + g1].clone(), pids[:nq], pids[nq:][g0:g1], cams[:nq], cams[nq:][g0:g1])
        return x, pids, cams, local

    def call(local, k):
        ql, gl, qp, gp, qc, gc = local
        return R.rerank_topk_and_eval_sharded(ql, gl, k, qp, gp, qc, gc, group=dist.group.WORLD)

    x, _, _, local = shard(a.nq, a.ng, a.d, 0)
    del x
    call(local, a.k)
    ts = []
    for _ in range(a.reps):
        torch.cuda.synchronize()
        dist.barrier()
        t0 = time.perf_counter()
        call(local, a.k)
        torch.cuda.synchronize()
        dist.barrier()
        ts.append(time.perf_counter() - t0)
    t = torch.tensor(ts, dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    del local
    x, pids, cams, local = shard(a.check_q, a.check_g, a.d, 1)
    idx, dst, ev = call(local, a.k)
    equal = None
    if rank == 0:
        nq = a.check_q
        ri, rd, rev = R.rerank_topk_and_eval(x[:nq], x[nq:], a.k, pids[:nq], pids[nq:], cams[:nq], cams[nq:])
        equal = bool(torch.equal(idx, ri) and torch.equal(dst, rd) and np.array_equal(ev.ranks, rev.ranks)
                     and np.array_equal(ev.single_performance, rev.single_performance)
                     and np.array_equal(ev.cmc, rev.cmc) and ev.mAP == rev.mAP)
        m, rng = med(t.cpu().tolist())
        print(json.dumps({"mode": f"sharded over {world} GPUs", "gpu": name, "power_limit": power, "nq": a.nq,
                          "ng": a.ng, "d": a.d, "k": a.k, "world": world, "sharded_s": m, "min_max": rng,
                          "windows": a.reps, "check_shape": [a.check_q, a.check_g], "bit_identical": equal}),
              flush=True)
    dist.destroy_process_group()
    if equal is False:
        raise SystemExit("sharded result differs from the one-GPU result")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--emulate-world", type=int, default=0)
    ap.add_argument("--nq", type=int, default=50000)
    ap.add_argument("--ng", type=int, default=200000)
    ap.add_argument("--d", type=int, default=2048)
    ap.add_argument("--ids", type=int, default=20000)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check-q", type=int, default=5000)
    ap.add_argument("--check-g", type=int, default=20000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    name, power = card()
    if a.emulate_world:
        emulate(a, name, power)
    else:
        distributed(a, name, power)


if __name__ == "__main__":
    main()
