"""Row-blocked k-reciprocal re-ranking (retrieval.rerank_topk_and_eval, ctl_rerank_topk) at two shapes.

  market : Q = 3368, G = 15 913, d = 2048 (Market-1501's evaluation shape; 751 clustered identities, sigma = 3, host
           generator of oracle/ctl_oracle.synth_retrieval).  The dense retrieval.rerank + evaluate_matrix and the blocked
           rerank_topk_and_eval (k = 100) in alternating windows in one process, medians of --reps windows with their
           range (CUDA events around one synchronised call each); the two results are asserted equal.  The blocked path
           runs at its default block (the whole N x N matrix fits in 2 GiB here) and at --market-block rows.
  config5: Q = 50 000, G = 200 000, d = 2048 (BASELINE config 5), 20 000 identities, sigma = 3, generated on the device
           from a seed.  rerank_topk_and_eval with k = 100 at the default block (2048 rows): median of --reps5 runs,
           the peak of torch.cuda.max_memory_allocated, and the time split into sweeps A and B, query expansion + the
           inverted index, and sweep C (CUDA events of one rerank_blocked_stages run); mAP / CMC with and without
           re-ranking (the latter: evaluate_streamed).
Algorithmic GEMM work from the shapes: 2 N^2 d for each of sweeps A and B, 2 Q G d for sweep C (the dense path: 2 N^2 d).
Prints one JSON line per shape with the card's name and power limit.

    python tools/bench_rerank_blocked.py [--shapes market,config5] [--reps 5] [--reps5 2]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import ctl_b200  # noqa: E402,F401
from ctl_b200 import retrieval as R  # noqa: E402
from oracle import ctl_oracle as O  # noqa: E402
from tools.bench_basic import card  # noqa: E402


def timed(fn):
    """(result, ms) of one call, CUDA events around it (the call synchronises on its own read-back)."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1)


def med(ts):
    ts = sorted(ts)
    return round(ts[len(ts) // 2], 2), [round(ts[0], 2), round(ts[-1], 2)]


def tflop(nq, ng, d):
    n = nq + ng
    return {"gemm_tflop_blocked": round((4.0 * n * n * d + 2.0 * nq * ng * d) / 1e12, 2),
            "gemm_tflop_dense": round(2.0 * n * n * d / 1e12, 2)}


def same(a, b):
    return (np.array_equal(a.cmc, b.cmc) and a.mAP == b.mAP and np.array_equal(a.ranks, b.ranks)
            and np.array_equal(a.single_performance, b.single_performance))


def market(a, name, power):
    nq, ng, d, k = 3368, 15913, 2048, 100
    feats, pids, cams = O.synth_retrieval(nq, ng, 751, d, 3.0, 0)
    q, g = feats[:nq].cuda(), feats[nq:].cuda()
    ids = (pids[:nq], pids[nq:], cams[:nq], cams[nq:])

    def dense():
        out = R.rerank(q, g)
        return out, R.evaluate_matrix(out, *ids)

    def blocked(rows):
        return lambda: R.rerank_topk_and_eval(q, g, k, *ids, block_rows=rows)

    variants = {"dense": dense, "blocked": blocked(None), f"blocked_{a.market_block}": blocked(a.market_block)}
    for fn in variants.values():  # warm-up
        fn()
    ts = {v: [] for v in variants}
    for _ in range(a.reps):
        for v, fn in variants.items():
            ts[v].append(timed(fn)[1])
    out_d, ev_d = dense()
    ref = torch.sort(out_d, dim=1, stable=True).indices[:, :k]
    for v in variants:
        if v == "dense":
            continue
        idx, dst, ev = variants[v]()
        assert torch.equal(idx, ref) and torch.equal(dst, out_d.gather(1, ref)) and same(ev, ev_d), v
    res = {"shape": "market", "gpu": name, "power_limit": power, "nq": nq, "ng": ng, "d": d, "k": k,
           "default_block_rows": R.rerank_block_rows(nq, ng), "equal": True, **tflop(nq, ng, d)}
    for v in variants:
        m, rng = med(ts[v])
        res[f"{v}_ms"], res[f"{v}_min_max"] = m, rng
    res["mAP_rerank"] = round(ev_d.mAP, 6)
    print(json.dumps(res), flush=True)


def config5(a, name, power):
    nq, ng, d, k, nid = 50000, 200000, 2048, 100, 20000
    n = nq + ng
    gen = torch.Generator(device="cuda").manual_seed(0)
    pid = torch.randint(0, nid, (n,), generator=gen, device="cuda")
    cam = torch.randint(0, 6, (n,), generator=gen, device="cuda")
    x = torch.randn(nid, d, generator=gen, device="cuda")[pid]
    x.add_(torch.randn(n, d, generator=gen, device="cuda"), alpha=3.0)
    x = torch.nn.functional.normalize(x, dim=1)
    pids, cams = pid.cpu().numpy(), cam.cpu().numpy()
    del pid, cam
    q, g = x[:nq], x[nq:]
    ids = (pids[:nq], pids[nq:], cams[:nq], cams[nq:])
    rows = R.rerank_block_rows(nq, ng)
    ts, ev, idx0 = [], None, None
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(a.reps5):
        (idx, dst, ev), t = timed(lambda: R.rerank_topk_and_eval(q, g, k, *ids))
        ts.append(t / 1e3)
        assert idx0 is None or torch.equal(idx, idx0)
        idx0 = idx
        del dst
    peak = torch.cuda.max_memory_allocated() - base
    ws = R.rerank_topk_workspace_bytes(nq, ng, d, 20, 6, k, rows)
    marks = []
    r = R.rerank_blocked_stages(q, g, k, events=marks)
    torch.cuda.synchronize()
    assert torch.equal(r["idx"], idx0)
    split = {f"{b}_s": round(ea.elapsed_time(eb) / 1e3, 2) for (_, ea), (b, eb) in zip(marks, marks[1:])}
    del r
    plain = R.evaluate_streamed(R.build_planes(q), R.build_planes(g), *ids)
    m, rng = sorted(ts)[len(ts) // 2], [min(ts), max(ts)]
    res = {"shape": "config5", "gpu": name, "power_limit": power, "nq": nq, "ng": ng, "d": d, "k": k, "ids": nid,
           "block_rows": rows, **tflop(nq, ng, d), "rerank_topk_and_eval_s": round(m, 2),
           "min_max": [round(t, 2) for t in rng], "runs": a.reps5, "sweeps_staged": split,
           "peak_alloc_gb": round(peak / 1e9, 2), "workspace_gb": round(ws / 1e9, 2),
           "dense_matrix_gb": round(4.0 * n * n / 1e9, 1),
           "mAP_rerank": round(ev.mAP, 6), "cmc_rerank": [round(float(ev.cmc[i - 1]), 6) for i in (1, 5, 10)],
           "mAP_plain": round(plain.mAP, 6), "cmc_plain": [round(float(plain.cmc[i - 1]), 6) for i in (1, 5, 10)]}
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="market,config5")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--reps5", type=int, default=2)
    ap.add_argument("--market-block", type=int, default=4096)
    a = ap.parse_args()
    name, power = card()
    shapes = a.shapes.split(",")
    if "market" in shapes:
        market(a, name, power)
        torch.cuda.empty_cache()
    if "config5" in shapes:
        config5(a, name, power)


if __name__ == "__main__":
    main()
