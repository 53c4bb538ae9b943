"""CPU: the visrank oracle (tests/visrank_oracle.py) against OpenCV where it imports, and against the grids the
reference's own visualize_ranked_results wrote (tests/golden/visrank_*.npz); the drop-in's host pieces."""
import glob
import os
import random

import numpy as np
import pytest

import visrank_oracle as V
from conftest import GOLDEN, load_golden
from ctl_b200.utils import visrank as VR

CASES = sorted(os.path.basename(p)[len("visrank_"):-len(".npz")] for p in glob.glob(os.path.join(GOLDEN, "visrank_*.npz")))


def _shapes():
    rng = np.random.default_rng(0)
    out = [(int(rng.integers(1, 400)), int(rng.integers(1, 300)), int(rng.integers(1, 400)), int(rng.integers(1, 300)))
           for _ in range(300)]
    for a in (1, 2, 3):  # 1-row / 1-column sources and targets, larger than 320
        for b in (1, 2, 7, 400):
            for t in ((256, 128), (1, 1), (1, 300), (700, 1), (641, 333), (2, 3)):
                out += [(a, b) + t, (b, a) + t]
    out += [(256, 128, 128, 64), (512, 256, 256, 128), (134, 262, 128, 256), (128, 64, 256, 128), (1, 1, 64, 32)]
    return out


def test_cv_resize_matches_opencv():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(1)
    for H, W, h, w in _shapes():
        src = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        assert np.array_equal(V.cv_resize(src, h, w), cv2.resize(src, (w, h))), (H, W, h, w)


def test_border_cell_and_grid_match_opencv():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(2)
    h, w, topk = 64, 32, 3
    imgs = [rng.integers(0, 256, (int(rng.integers(1, 90)), int(rng.integers(1, 60)), 3), dtype=np.uint8)
            for _ in range(4)]
    for img in imgs:
        for colour in (V.BLACK, V.GREEN, V.RED):
            # channels are independent, so an RGB image with an RGB colour is what cv2 does in BGR
            ref = cv2.resize(cv2.copyMakeBorder(cv2.resize(img, (w, h)), 3, 3, 3, 3, cv2.BORDER_CONSTANT,
                                                value=colour), (w, h))
            assert np.array_equal(V.cell(img, h, w, colour), ref)
    g = V.grid(imgs[0], [(imgs[1], True), (imgs[2], False)], h, w, topk)
    assert g.shape == (h, (topk + 1) * w + topk * 2 + 8, 3)
    assert (g[:, w: w + 8] == 255).all() and (g[:, V.cell_x(3, w):] == 255).all()  # spacing and the empty rank


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_reference_golden(name, tmp_path):
    case = V.load_case(load_golden(f"visrank_{name}.npz"), str(tmp_path))
    cfg = case["cfg"]
    args = (case["distmat"], case["samples"], V.load_rgb, cfg["USE_CENTROIDS"], cfg["KEEP_CAMID_CENTROIDS"],
            cfg["VISUALIZE_MAX_NUMBER"], cfg["VISUALIZE_TOPK"], *cfg["SIZE_TEST"])
    if case["error"]:
        with pytest.raises(AssertionError):
            V.visualize(*args)
        return
    got = V.visualize(*args)
    assert sorted(got) == sorted(case["expected"])
    for n, grid in case["expected"].items():
        assert np.array_equal(got[n], grid), n


def test_goldens_cover_the_issue_cases(tmp_path):
    """ranked lists shorter than topk, junk entries, repeated basenames and MAX_NUMBER < Q are all exercised."""
    seen = set()
    for name in CASES:
        case = V.load_case(load_golden(f"visrank_{name}.npz"), str(tmp_path / name))
        cfg, d = case["cfg"], case["distmat"]
        if case["error"]:
            seen.add("error")
            continue
        nq = len(case["samples"]) - (len(case["samples"]) - d.shape[0])
        q, g, respect = V.galleries(case["samples"], d.shape[0], cfg["USE_CENTROIDS"], cfg["KEEP_CAMID_CENTROIDS"])
        for i in range(min(nq, cfg["VISUALIZE_MAX_NUMBER"] + 1)):
            n_junk = sum(V.is_junk(q[i], x, respect) for x in g)
            seen |= {"junk"} if n_junk else set()
            seen |= {"short"} if len(V.ranked(d[i], q[i], g, respect, cfg["VISUALIZE_TOPK"])) < cfg["VISUALIZE_TOPK"] else set()
        seen |= {"max"} if cfg["VISUALIZE_MAX_NUMBER"] + 1 < nq else set()
        seen |= {"dup"} if len(case["expected"]) < min(nq, cfg["VISUALIZE_MAX_NUMBER"] + 1) else set()
        seen |= {"respect"} if respect else set()
    assert seen == {"error", "junk", "short", "max", "dup", "respect"}


@pytest.mark.parametrize("name", CASES)
def test_drop_in_gallery_picks_and_topk_width(name, tmp_path):
    """utils/visrank.py's centroid picks equal the oracle's and leave the caller's random state alone; its top-k
    width holds every query's topk non-junk rows."""
    case = V.load_case(load_golden(f"visrank_{name}.npz"), str(tmp_path))
    cfg, d = case["cfg"], case["distmat"]
    random.seed(123)
    state = random.getstate()
    q, g, respect = VR._galleries(case["samples"], d.shape[0], cfg["USE_CENTROIDS"], cfg["KEEP_CAMID_CENTROIDS"])
    assert random.getstate() == state
    oq, og, orespect = V.galleries(case["samples"], d.shape[0], cfg["USE_CENTROIDS"], cfg["KEEP_CAMID_CENTROIDS"])
    assert (q, g, respect) == (oq, og, orespect)
    if not g:
        return
    ids, k = VR._ids(q, g, respect, cfg["VISUALIZE_TOPK"], "cpu")
    junk = [sum(V.is_junk(x, y, respect) for y in g) for x in q]
    assert k == min(len(g), cfg["VISUALIZE_TOPK"] + max(junk))


def test_png_writer_round_trips(tmp_path):
    rng = np.random.default_rng(3)
    for h, w in ((1, 1), (64, 380), (7, 3)):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        p = tmp_path / f"{h}x{w}.png"
        p.write_bytes(VR.png_bytes(img))
        assert np.array_equal(V.load_rgb(str(p)), img)
