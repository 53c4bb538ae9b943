"""Writes tests/golden/visrank_*.npz: the ranked-result grids the reference's own visualize_ranked_results
(utils/visrank.py, imported unmodified through oracle/ref_import.py; needs OpenCV) writes for small synthetic
datasets, for tests/test_visrank_cpu.py and tests/test_visrank_gpu.py.

Every case has the same image files: ragged Pillow-saved JPEGs at 4:2:0 and 4:4:4, grayscale JPEGs and PNGs, two
queries with the same basename in different directories.  Features are drawn until every row of the squared-L2
distance matrix of the L2-normalised features (R1_mAP.compute's distmat) has gaps of at least 1e-3 between sorted
distances, so the reference's unstable np.argsort and any exact (distance, index) ranking agree.  Arrays per case:
  file_data uint8, file_offsets int64 [n + 1], file_names str [n]  the image files (relative paths)
  samples str (JSON)     the dataset: [path, pid, camid, index] per query then gallery sample
  feats float32 [Q + G, D], pids / camids str (JSON)              R1_mAP.compute's inputs (G: gallery or centroids)
  distmat float32 [Q, G]   the distances visualize_ranked_results ranks
  cfg str (JSON)           USE_CENTROIDS, KEEP_CAMID_CENTROIDS, VISUALIZE_TOPK, VISUALIZE_MAX_NUMBER, SIZE_TEST
  names str [m], grids uint8 [m, h, Wg, 3]   the PNGs written (decoded, RGB), or
  error str                the exception type the reference raised

    python tools/make_visrank_golden.py
"""
import io
import json
import os
import sys
import tempfile

import cv2
import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402

SIZE_TEST = [64, 32]
# (relative path, pid, camid, (h, w), format) -- queries first
QUERIES = [("q/0001_c1s1.jpg", 1, 1, (40, 20), "420"), ("q/0002_c2s1.jpg", 2, 2, (57, 23), "444"),
           ("q/0003_c1s1.png", 3, 1, (30, 31), "png"), ("a/0004_same.jpg", 4, 3, (9, 5), "gray"),
           ("b/0004_same.jpg", 1, 2, (128, 64), "420"), ("q/0005_c3s1.jpg", 5, 3, (1, 7), "444")]
GALLERY_PIDS = [1, 1, 1, 2, 2, 2, 3, 3, 4, 4, 5, 6, 6, 7, 1, 2, 3, 4, 5, 6, 7, 8]
GALLERY_CAMS = [1, 2, 3, 2, 2, 1, 1, 3, 3, 1, 2, 1, 2, 3, 1, 3, 2, 3, 3, 1, 2, 1]
CASES = {
    "plain": dict(USE_CENTROIDS=False, KEEP_CAMID_CENTROIDS=True, VISUALIZE_TOPK=10, VISUALIZE_MAX_NUMBER=1000000),
    "topk3_max2": dict(USE_CENTROIDS=False, KEEP_CAMID_CENTROIDS=False, VISUALIZE_TOPK=3, VISUALIZE_MAX_NUMBER=2),
    "centroid_keep": dict(USE_CENTROIDS=True, KEEP_CAMID_CENTROIDS=True, VISUALIZE_TOPK=10, VISUALIZE_MAX_NUMBER=1000000),
    "centroid_nokeep": dict(USE_CENTROIDS=True, KEEP_CAMID_CENTROIDS=False, VISUALIZE_TOPK=10,
                            VISUALIZE_MAX_NUMBER=1000000),
}


def _content(h, w, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([x * 255 // max(w - 1, 1), y * 255 // max(h - 1, 1), ((x + 2 * y) * 9 + seed * 37) % 256], -1)
    return np.clip(base + rng.integers(-20, 21, (h, w, 3)), 0, 255).astype(np.uint8)


def _encode(img, fmt):
    buf = io.BytesIO()
    if fmt == "png":
        Image.fromarray(img).save(buf, format="PNG")
    elif fmt == "gray":
        Image.fromarray(img).convert("L").save(buf, format="JPEG", quality=90)
    else:
        Image.fromarray(img).save(buf, format="JPEG", quality=85, subsampling={"444": 0, "420": 2}[fmt])
    return buf.getvalue()


def files():
    out, samples = {}, []
    fmts = ["420", "444", "gray", "png"]
    entries = list(QUERIES) + [(f"g/{p:04d}_c{c}_{i:02d}.{'png' if i % 4 == 3 else 'jpg'}", p, c,
                                (20 + (i * 7) % 50, 10 + (i * 5) % 30), fmts[i % 4])
                               for i, (p, c) in enumerate(zip(GALLERY_PIDS, GALLERY_CAMS))]
    for i, (path, pid, cam, (h, w), fmt) in enumerate(entries):
        out[path] = _encode(_content(h, w, i), fmt)
        samples.append([path, pid, cam, i])
    return out, samples


def separated_feats(n_q, n_g, seed):
    """float32 features whose distmat rows (squared L2 of the normalised rows) have sorted gaps >= 1e-3."""
    rng = np.random.default_rng(seed)
    while True:
        f = rng.standard_normal((n_q + n_g, 16)).astype(np.float32)
        fn = f / np.linalg.norm(f.astype(np.float64), axis=1, keepdims=True)
        d = ((fn[:n_q, None, :] - fn[None, n_q:, :]) ** 2).sum(-1)
        if np.diff(np.sort(d, axis=1), axis=1).min() >= 1e-3:
            return f, d.astype(np.float32)


def run_case(ref, name, opts, blobs, samples, tmp):
    from visrank_oracle import galleries

    sys.path.insert(0, ref_import.REFERENCE_ROOT)
    try:
        from utils.visrank import visualize_ranked_results
    finally:
        sys.path.remove(ref_import.REFERENCE_ROOT)
    n_q = len(QUERIES)
    abs_samples = [(os.path.join(tmp, s[0]), s[1], s[2], s[3]) for s in samples]
    _, gallery, respect = galleries(abs_samples, n_q, opts["USE_CENTROIDS"], opts["KEEP_CAMID_CENTROIDS"])
    n_g = len(gallery) if opts["USE_CENTROIDS"] else len(samples) - n_q
    # without KEEP_CAMID_CENTROIDS the reference builds no centroid (visrank.py:90) and asserts; the distmat keeps
    # the gallery's width
    feats, dist = separated_feats(n_q, n_g or len(samples) - n_q, seed=len(name))
    rows = gallery if opts["USE_CENTROIDS"] and gallery else samples[n_q:]
    pids = [s[1] for s in samples[:n_q]] + [int(g[1]) for g in rows]
    camids = [s[2] for s in samples[:n_q]] + [list(map(int, g[2])) if respect else int(g[2]) for g in rows]
    cfg = ref_import.default_cfg(ref, **{"MODEL__USE_CENTROIDS": opts["USE_CENTROIDS"],
                                         "MODEL__KEEP_CAMID_CENTROIDS": opts["KEEP_CAMID_CENTROIDS"],
                                         "TEST__VISUALIZE_TOPK": opts["VISUALIZE_TOPK"],
                                         "TEST__VISUALIZE_MAX_NUMBER": opts["VISUALIZE_MAX_NUMBER"],
                                         "INPUT__SIZE_TEST": SIZE_TEST})
    out_dir = os.path.join(tmp, "out_" + name)
    arrays = dict(cfg=json.dumps(dict(opts, SIZE_TEST=SIZE_TEST)), samples=json.dumps(samples),
                  feats=feats, pids=json.dumps(pids), camids=json.dumps(camids), distmat=dist)
    try:
        visualize_ranked_results(dist, abs_samples, "image", cfg, width=SIZE_TEST[1], height=SIZE_TEST[0],
                                 save_dir=out_dir, topk=opts["VISUALIZE_TOPK"])
    except AssertionError as exc:
        arrays["error"] = type(exc).__name__
    else:
        names = sorted(os.listdir(out_dir))
        arrays["names"] = np.array(names)
        arrays["grids"] = np.stack([cv2.imread(os.path.join(out_dir, n))[:, :, ::-1] for n in names])
    names = sorted(blobs)
    arrays["file_names"] = np.array(names)
    arrays["file_offsets"] = np.cumsum([0] + [len(blobs[n]) for n in names]).astype(np.int64)
    arrays["file_data"] = np.frombuffer(b"".join(blobs[n] for n in names), dtype=np.uint8)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", f"visrank_{name}.npz"), **arrays)
    print(name, arrays.get("error") or f"{len(arrays['names'])} grids")


def main():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    ref = ref_import.load_reference()
    blobs, samples = files()
    with tempfile.TemporaryDirectory() as tmp:
        for path, data in blobs.items():
            os.makedirs(os.path.dirname(os.path.join(tmp, path)), exist_ok=True)
            with open(os.path.join(tmp, path), "wb") as f:
                f.write(data)
        for name, opts in CASES.items():
            run_case(ref, name, opts, blobs, samples, tmp)


if __name__ == "__main__":
    main()
