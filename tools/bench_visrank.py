"""TEST.VISUALIZE at the Market shape (Q = 3368, G = 15 913, topk 10, 256x128 cells): utils/visrank.py's ranked-result
grids.  Sources are seeded smooth colour fields saved by Pillow at quality 90, 4:2:0, 128x64 (bench_jpeg.py's); 512
distinct files are written under a temporary directory once per gallery and query path.  Features are seeded
normals (d = 2048) with Market-like identities (751 ids, 6 cameras).

  rank    : device time of the ranked list from identity-ordered planes (streamed top-k with k = topk + the largest
            junk count, then ctl_visrank_select), per grid
  decode / resize / compose : device time per grid of one chunk of --chunk grids (its distinct images decoded once)
  png     : host time to encode one grid as a PNG on one core (zlib level 1)
  wall    : visualize_ranked_planes end to end, from the planes to every PNG on disk, per grid and in total
Times are medians of --windows windows with their range; every line is JSON with the card's name and power limit.
With --reference N (no GPU needed), the reference's own visualize_ranked_results is timed instead on the host for its
first N queries at the same shape (oracle/ref_import.py; needs OpenCV and the reference tree).

    python tools/bench_visrank.py [--windows 5] [--chunk 256]
    python tools/bench_visrank.py --reference 50
"""
import argparse
import json
import os
import sys
import tempfile
import time
from types import SimpleNamespace as NS

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_jpeg import jpeg, smooth  # noqa: E402

NQ, NG, TOPK, SIZE = 3368, 15913, 10, (256, 128)


def dataset(root):
    rng = np.random.default_rng(0)
    pids, cams = rng.integers(0, 751, NQ + NG), rng.integers(1, 7, NQ + NG)
    blobs = [jpeg(smooth(128, 64, i)) for i in range(512)]
    samples = []
    for i in range(NQ + NG):
        path = os.path.join(root, f"{'q' if i < NQ else 'g'}{i:05d}_c{cams[i]}.jpg")
        with open(path, "wb") as f:
            f.write(blobs[i % len(blobs)])
        samples.append((path, int(pids[i]), int(cams[i]), i))
    return samples


def cfg(max_number):
    return NS(MODEL=NS(USE_CENTROIDS=False, KEEP_CAMID_CENTROIDS=True), INPUT=NS(SIZE_TEST=list(SIZE)),
              TEST=NS(VISUALIZE="yes", VISUALIZE_TOPK=TOPK, VISUALIZE_MAX_NUMBER=max_number))


def emit(**kw):
    print(json.dumps(kw), flush=True)


def reference(n, samples, root):
    from oracle import ref_import

    ref = ref_import.load_reference()
    sys.path.insert(0, ref_import.REFERENCE_ROOT)
    from utils.visrank import visualize_ranked_results

    c = ref_import.default_cfg(ref, TEST__VISUALIZE_MAX_NUMBER=n - 1, INPUT__SIZE_TEST=list(SIZE))
    f = torch.randn(NQ + NG, 2048, generator=torch.Generator().manual_seed(0))
    f = torch.nn.functional.normalize(f, dim=1)
    distmat = torch.cdist(f[:NQ], f[NQ:]).pow(2).numpy()
    t0 = time.perf_counter()
    visualize_ranked_results(distmat, samples, "image", c, width=SIZE[1], height=SIZE[0],
                             save_dir=os.path.join(root, "ref"), topk=TOPK)
    wall = time.perf_counter() - t0
    emit(case="reference_host", grids=n, wall_s=round(wall, 3), ms_per_grid=round(1e3 * wall / n, 3),
         host_cores=os.cpu_count(), note="the reference on the host cores (argsort of the full distmat included)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--chunk", type=int, default=256)
    ap.add_argument("--reference", type=int, default=0)
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as root:
        samples = dataset(root)
        if a.reference:
            return reference(a.reference, samples, root)
        import ctl_b200  # noqa: F401
        from ctl_b200 import retrieval as R
        from ctl_b200.datasets import transforms as T
        from ctl_b200.utils import visrank as VR
        from tools.bench_basic import card
        from tools.bench_resize import med, window_ms

        assert torch.cuda.is_available(), "bench_visrank.py measures on the GPU"
        name, power = card()
        f = torch.randn(NQ + NG, 2048, generator=torch.Generator().manual_seed(0)).cuda()
        pids = [s[1] for s in samples]
        qp = R.build_planes(f[:NQ], normalize=True, order=R.pid_order(pids[:NQ]))
        gp = R.build_planes(f[NQ:], normalize=True, order=R.pid_order(pids[NQ:]))
        query, gallery, _ = VR._galleries(samples, NQ, False, True)
        ids, k = VR._ids(query, gallery, False, TOPK, "cuda")

        def rank():
            return VR.ranked_lists(VR._rank_planes(qp, gp, k), ids, NG, TOPK)

        ranks = [window_ms(rank, 3) / NQ for _ in range(a.windows)]
        idx, matched, _ = rank()
        idx, matched = idx.cpu().numpy(), matched.cpu().numpy()
        # one chunk of grids: its distinct images, cells and device buffers
        paths, rows, cells = [], {}, []
        for g in range(a.chunk):
            for col, j in enumerate([-2] + [int(x) for x in idx[g]]):
                if j == -1:
                    continue
                p = query[g][0] if j == -2 else gallery[j][0]
                rows.setdefault(p, len(paths))
                if rows[p] == len(paths):
                    paths.append(p)
                cells.append((rows[p], g, col, 0xFF0000))
        batch = T.pack_jpegs(paths).to("cuda")
        out = torch.empty(max(batch.out_bytes, 1), dtype=torch.uint8, device="cuda")
        st = torch.zeros(len(batch), dtype=torch.int32, device="cuda")
        ws = torch.empty(batch.workspace_bytes, dtype=torch.uint8, device="cuda")
        T._decode_enqueue(batch, out, st, ws)
        ragged = T.RaggedImages(out, batch.out_table, batch.rows)
        resized, _ = VR._resize_linear_cv_enqueue(ragged, SIZE)
        grids, _ = VR.compose(resized, cells, a.chunk, TOPK)
        dev_cells = torch.tensor(cells, dtype=torch.int32, device="cuda")
        parts = {"decode": lambda: T._decode_enqueue(batch, out, st, ws),
                 "resize": lambda: VR._resize_linear_cv_enqueue(ragged, SIZE),
                 "compose": lambda: VR.compose(resized, dev_cells, a.chunk, TOPK)}
        res = {n: [] for n in parts}
        for _ in range(a.windows):
            for n, fn in parts.items():
                res[n].append(window_ms(fn, 10) / a.chunk)
        host = grids.cpu().numpy()
        png = []
        for _ in range(a.windows):
            t0 = time.perf_counter()
            for i in range(16):
                VR.png_bytes(host[i])
            png.append((time.perf_counter() - t0) * 1e3 / 16)
        walls = []
        for w in range(max(1, a.windows // 2)):
            d = os.path.join(root, f"out{w}")
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            VR.visualize_ranked_planes(qp, gp, samples, cfg(1000000), width=SIZE[1], height=SIZE[0], save_dir=d,
                                       topk=TOPK)
            walls.append(time.perf_counter() - t0)
            assert len(os.listdir(d)) == NQ
        common = dict(gpu=name, power_limit=power, nq=NQ, ng=NG, topk=TOPK, size=list(SIZE), host_cores=os.cpu_count())
        emit(case="device_ms_per_grid", rank=med(ranks), **{n: med(v) for n, v in res.items()},
             distinct_images_per_chunk=len(paths), chunk=a.chunk, **common)
        emit(case="host_png_ms_per_grid_one_core", png=med(png), **common)
        emit(case="wall_to_disk", seconds=med(walls), ms_per_grid=med([1e3 * w / NQ for w in walls]), **common)


if __name__ == "__main__":
    main()
