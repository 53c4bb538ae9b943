"""k-reciprocal re-ranking + CMC / mAP from the re-ranked matrix at Market-1501's evaluation shape.

Synthetic clustered features (SURVEY section 8d): 751 identities, sigma = 3, Q = 3368, G = 15 913, d = 2048.  Times, each
the median of --reps windows (CUDA events, after a warm-up) with the windows' min and max:
  - rerank_eval: retrieval.rerank (k1 = 20, k2 = 6, lambda = 0.3) + retrieval.evaluate_matrix on its output, as
    eval_reranked runs them (both read a status / the packed results back, so each window is one synchronised call);
  - rerank: retrieval.rerank alone;  dist: the N x N distance GEMM alone (ctl_dist_matrix into a preallocated matrix);
  - plain_eval: evaluate_streamed on the same features without re-ranking.
Also printed: mAP / CMC with and without re-ranking, the GEMM's algorithmic work 2 N^2 d, the card's name and power limit.
With --cpu, the float64 oracle's per-row loop form (oracle/rerank_oracle.rerank_loop) is timed once at the same size on
the host cores, and the core count is printed.

    python tools/bench_rerank.py [--reps 5] [--cpu]
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
from ctl_b200 import _native as N  # noqa: E402
from ctl_b200 import retrieval as R  # noqa: E402
from oracle import ctl_oracle as O  # noqa: E402
from oracle import rerank_oracle as RO  # noqa: E402
from tools.bench_basic import card, spread, time_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nq", type=int, default=3368)
    ap.add_argument("--ng", type=int, default=15913)
    ap.add_argument("--ids", type=int, default=751)
    ap.add_argument("--dim", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu", action="store_true")
    a = ap.parse_args()
    nq, ng, d = a.nq, a.ng, a.dim
    n = nq + ng
    feats, pids, cams = O.synth_retrieval(nq, ng, a.ids, d, 3.0, 0)
    qp, gp, qc, gc = pids[:nq], pids[nq:], cams[:nq], cams[nq:]
    name, power = card()
    out = {"gpu": name, "power_limit": power, "nq": nq, "ng": ng, "d": d, "k1": 20, "k2": 6, "lambda": 0.3,
           "gemm_tflop": round(2.0 * n * n * d / 1e12, 3)}
    if not a.cpu:
        q, g = feats[:nq].cuda(), feats[nq:].cuda()

        def rerank_eval():
            return R.evaluate_matrix(R.rerank(q, g), qp, gp, qc, gc)

        t = time_ms(rerank_eval, 1, a.reps)
        out.update(rerank_eval_ms=round(t[0], 2), rerank_eval_min_max=spread(t))
        t = time_ms(lambda: R.rerank(q, g), 1, a.reps)
        out.update(rerank_ms=round(t[0], 2), rerank_min_max=spread(t))
        planes = R.build_planes(torch.cat([q, g]))
        dm = torch.empty(n, n, device="cuda")

        def dist():
            N.check(N.lib().ctl_dist_matrix(planes.ptr, n, planes.ptr, n, d, planes.flags, dm.data_ptr(), n,
                                            N.stream_ptr()))

        t = time_ms(dist, 1, a.reps)
        out.update(dist_ms=round(t[0], 2), dist_min_max=spread(t), dist_tflops=round(2.0 * n * n * d / t[0] / 1e9, 1))
        del dm, planes
        t = time_ms(lambda: R.evaluate_streamed(R.build_planes(q), R.build_planes(g), qp, gp, qc, gc), 1, a.reps)
        out.update(plain_eval_ms=round(t[0], 2), plain_eval_min_max=spread(t))
        rr = rerank_eval()
        pl = R.evaluate_streamed(R.build_planes(q), R.build_planes(g), qp, gp, qc, gc)
        out.update(mAP_rerank=round(rr.mAP, 6), cmc_rerank=[round(float(rr.cmc[k - 1]), 6) for k in (1, 5, 10)],
                   mAP_plain=round(pl.mAP, 6), cmc_plain=[round(float(pl.cmc[k - 1]), 6) for k in (1, 5, 10)])
    else:
        out.update(cpu_cores=os.cpu_count(), torch_threads=torch.get_num_threads())
        t0 = time.perf_counter()
        nd = RO.nd_from_features(feats.numpy())
        res = RO.rerank_loop(nd, nq, 20, 6, 0.3)
        out.update(cpu_loop_s=round(time.perf_counter() - t0, 1))
        res_eval = O.eval_func(O.rank_indices(res["out"]), qp, gp, qc, gc, 50)
        out.update(mAP_rerank=round(float(res_eval[1]), 6))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
