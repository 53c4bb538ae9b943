"""GPU: ranked-result grids (utils/visrank.py) on the device -- ctl_resize_linear_cv_u8, ctl_visrank_compose and
ctl_visrank_select bit for bit against tests/visrank_oracle.py, and R1_mAP.compute with TEST.VISUALIZE = "yes"
against the PNGs the reference wrote (tests/golden/visrank_*.npz)."""
import glob
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

import visrank_oracle as V
from conftest import GOLDEN, load_golden
from ctl_b200 import retrieval as R
from ctl_b200.datasets import transforms as T
from ctl_b200.utils import visrank as VR
from ctl_b200.utils.reid_metric import R1_mAP

pytestmark = pytest.mark.gpu
CASES = sorted(os.path.basename(p)[len("visrank_"):-len(".npz")] for p in glob.glob(os.path.join(GOLDEN, "visrank_*.npz")))


def _images(rng, n, max_side=300):
    out = []
    for i in range(n):
        if i % 7 == 3:
            out.append(None)  # mock row
            continue
        h, w = (1, int(rng.integers(1, 50))) if i % 5 == 1 else (int(rng.integers(1, max_side)), int(rng.integers(1, max_side)))
        if i % 5 == 2:
            h, w = w, 1
        out.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
    return out


@pytest.mark.parametrize("size", [(256, 128), (64, 32), (137, 263), (320, 320), (1, 1)])
def test_resize_linear_cv_matches_oracle(size):
    rng = np.random.default_rng(size[0])
    imgs = _images(rng, 40)
    out = VR.resize_linear_cv(T.pack_images(imgs).to("cuda"), size).cpu().numpy()
    for i, im in enumerate(imgs):
        ref = np.zeros((*size, 3), np.uint8) if im is None else V.cv_resize(im, *size)
        assert np.array_equal(out[i], ref), (i, None if im is None else im.shape)


def test_resize_linear_cv_bad_entries_set_their_status():
    rng = np.random.default_rng(5)
    imgs = _images(rng, 6)
    ragged = T.pack_images(imgs, pin=False)
    table = ragged.table.clone()
    table[1] = torch.tensor([ragged.data.numel() - 3, 2, 2])   # runs past the buffer
    table[4] = torch.tensor([0, -1, 5])                         # negative side
    bad = T.RaggedImages(ragged.data, table, ragged.rows).to("cuda")
    out, status = VR._resize_linear_cv_enqueue(bad, (16, 8))
    assert status.cpu().tolist() == [0, 1, 0, 0, 1, 0]
    out = out.cpu().numpy()
    assert not out[1].any() and not out[4].any()
    assert np.array_equal(out[0], V.cv_resize(imgs[0], 16, 8))
    with pytest.raises(ValueError, match=r"\[1, 4\]"):
        VR.resize_linear_cv(bad, (16, 8))


@pytest.mark.parametrize("h,w,topk", [(256, 128, 10), (64, 32, 3), (5, 3, 1)])
def test_compose_matches_oracle(h, w, topk):
    rng = np.random.default_rng(h)
    n_rows, n_grids = 9, 4
    resized = rng.integers(0, 256, (n_rows, h, w, 3), dtype=np.uint8)
    cells, ref = [], np.full((n_grids, h, V.grid_width(w, topk), 3), 255, np.uint8)
    colours = {0x000000: V.BLACK, 0x00FF00: V.GREEN, 0xFF0000: V.RED}
    for g in range(n_grids):
        for col in range(0, topk + 1 - g % 2):  # odd grids leave their last rank empty (white)
            row, colour = int(rng.integers(0, n_rows)), int(rng.choice(list(colours)))
            cells.append((row, g, col, colour))
            x = V.cell_x(col, w)
            ref[g, :, x: x + w] = V.cv_resize(V.border(resized[row], colours[colour]), h, w)
    out, status = VR.compose(torch.from_numpy(resized).cuda(), cells, n_grids, topk)
    assert status.item() == 0
    assert np.array_equal(out.cpu().numpy(), ref)
    out, status = VR.compose(torch.from_numpy(resized).cuda(), cells + [(n_rows, 0, 1, 0), (0, 0, topk + 1, 0)],
                             n_grids, topk)
    assert status.item() == 1 and np.array_equal(out.cpu().numpy(), ref)  # out-of-range cells are skipped


def _ranked_case(nq, ng, n_ids, n_cams, respect, seed, ties):
    g = torch.Generator().manual_seed(seed)
    feats = torch.randn(nq + ng, 64, generator=g)
    if ties:  # exact duplicates in the gallery: equal distances, ranked by index
        feats[nq + 1::3] = feats[nq]
    rng = np.random.default_rng(seed)
    pids, cams = rng.integers(0, n_ids, nq + ng), rng.integers(0, n_cams, nq + ng)
    q = [(f"q{i}", int(pids[i]), int(cams[i])) for i in range(nq)]
    if respect:
        gal = [(f"g{j}", int(pids[nq + j]), tuple(sorted({int(cams[nq + j]), int(cams[nq + j] + 1) % n_cams})))
               for j in range(ng)]
    else:
        gal = [(f"g{j}", int(pids[nq + j]), int(cams[nq + j])) for j in range(ng)]
    return feats, q, gal


@pytest.mark.parametrize("respect", [False, True])
@pytest.mark.parametrize("ties", [False, True])
def test_ranked_lists_match_oracle(respect, ties):
    nq, ng, topk = 37, 300, 10
    feats, q, gal = _ranked_case(nq, ng, 12, 4, respect, 7 + ties, ties)
    qd, gd = feats[:nq].cuda(), feats[nq:].cuda()
    d = R.dist_matrix(qd, gd)
    dh = d.cpu().numpy()
    ids, k = VR._ids(q, gal, respect, topk, "cuda")
    for idx_dev in (VR._rank_dense(d, k, 1 << 30), VR._rank_planes(R.build_planes(qd), R.build_planes(gd), k)):
        idx, matched, status = VR.ranked_lists(idx_dev, ids, ng, topk)
        assert status.item() == 0
        idx, matched = idx.cpu().numpy(), matched.cpu().numpy()
        for i in range(nq):
            ref = V.ranked(dh[i], q[i], gal, respect, topk)
            n = len(ref)
            assert idx[i, :n].tolist() == [g for g, _ in ref] and (idx[i, n:] == -1).all(), i
            assert matched[i, :n].tolist() == [int(m) for _, m in ref], i


def test_ranked_lists_market_shape():
    """Q = 3368, G = 15 913, topk 10: the streamed top-k from identity-ordered planes, and the column-blocked sort of
    the distance matrix, against the stable argsort of that matrix."""
    nq, ng, topk = 3368, 15913, 10
    feats, q, gal = _ranked_case(nq, ng, 751, 6, False, 11, False)
    qd, gd = feats[:nq].cuda(), feats[nq:].cuda()
    ids, k = VR._ids(q, gal, False, topk, "cuda")
    q_pids, g_pids = [s[1] for s in q], [s[1] for s in gal]
    qp = R.build_planes(qd, order=R.pid_order(q_pids))
    gp = R.build_planes(gd, order=R.pid_order(g_pids))
    d = R.dist_matrix(qd, gd)
    order = np.argsort(d.cpu().numpy(), axis=1, kind="stable")[:, :k]
    assert np.array_equal(VR._rank_planes(qp, gp, k).cpu().numpy(), order)
    assert np.array_equal(VR._rank_dense(d, k, 64 << 20).cpu().numpy(), order)
    idx, matched, _ = VR.ranked_lists(torch.from_numpy(order).cuda(), ids, ng, topk)
    idx = idx.cpu().numpy()
    for i in range(0, nq, 97):
        ref = V.ranked(d[i].cpu().numpy(), q[i], gal, False, topk)
        assert idx[i].tolist() == [g for g, _ in ref]


def _cfg(case, out_dir, visualize="yes"):
    c = case["cfg"]
    return NS(MODEL=NS(USE_CENTROIDS=c["USE_CENTROIDS"], KEEP_CAMID_CENTROIDS=c["KEEP_CAMID_CENTROIDS"]),
              SOLVER=NS(DISTANCE_FUNC="euclidean"), INPUT=NS(SIZE_TEST=c["SIZE_TEST"]), OUTPUT_DIR=str(out_dir),
              TEST=NS(VISUALIZE=visualize, VISUALIZE_TOPK=c["VISUALIZE_TOPK"],
                      VISUALIZE_MAX_NUMBER=c["VISUALIZE_MAX_NUMBER"]))


def _module(case, out_dir, visualize="yes"):
    loader = NS(dataset=NS(samples=case["samples"]))
    return NS(hparams=_cfg(case, out_dir, visualize), trainer=NS(current_epoch=0, val_dataloaders=[loader]))


def _assert_files(directory, expected):
    got = V.read_pngs(directory)
    assert sorted(got) == sorted(expected)
    for n, grid in expected.items():
        assert np.array_equal(got[n], grid), n


@pytest.mark.parametrize("name", CASES)
def test_r1_map_visualize_writes_the_reference_pngs(name, tmp_path):
    case = V.load_case(load_golden(f"visrank_{name}.npz"), str(tmp_path / "data"))
    nq = case["distmat"].shape[0]
    feats = torch.from_numpy(case["feats"])
    respect = case["cfg"]["USE_CENTROIDS"] and case["cfg"]["KEEP_CAMID_CENTROIDS"]
    args = (feats, case["pids"], case["camids"], respect)
    plain = R1_mAP(_module(case, tmp_path / "no", "no"), nq).compute(*args)
    metric = R1_mAP(_module(case, tmp_path / "yes"), nq)
    if case["error"]:
        with pytest.raises(AssertionError):
            metric.compute(*args)
        return
    vis = metric.compute(*args)
    assert np.array_equal(vis[0], plain[0]) and vis[1] == plain[1] and np.array_equal(vis[2], plain[2])
    assert not os.path.exists(tmp_path / "no" / "visrank")
    _assert_files(tmp_path / "yes" / "visrank", case["expected"])


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("budget", [1 << 30, 1])
def test_distmat_drop_in_writes_the_reference_pngs(name, budget, tmp_path, capsys):
    """numpy distmat, one chunk or (budget = 1 byte) one grid per chunk."""
    case = V.load_case(load_golden(f"visrank_{name}.npz"), str(tmp_path / "data"))
    c = case["cfg"]
    out = tmp_path / "out"
    kw = dict(width=c["SIZE_TEST"][1], height=c["SIZE_TEST"][0], save_dir=str(out), topk=c["VISUALIZE_TOPK"],
              memory_budget=budget)
    cfg = _cfg(case, out)
    if case["error"]:
        with pytest.raises(AssertionError):
            VR.visualize_ranked_results(case["distmat"], case["samples"], "image", cfg, **kw)
        return
    VR.visualize_ranked_results(case["distmat"], case["samples"], "image", cfg, **kw)
    _assert_files(out, case["expected"])
    assert capsys.readouterr().out.endswith(f'Done. Images have been saved to "{out}" ...\n')
    if budget == 1:
        for p in out.iterdir():
            p.unlink()
        VR.visualize_ranked_results(torch.from_numpy(case["distmat"]).cuda(), case["samples"], "image", cfg, **kw)
        _assert_files(out, case["expected"])


def test_visualize_rejects_video_and_missing_dataset(tmp_path):
    case = V.load_case(load_golden("visrank_plain.npz"), str(tmp_path))
    with pytest.raises(NotImplementedError):
        VR.visualize_ranked_results(case["distmat"], case["samples"], "video", _cfg(case, tmp_path))
    module = _module(case, tmp_path)
    module.trainer = NS(current_epoch=0)
    with pytest.raises(ValueError, match="VISUALIZE"):
        R1_mAP(module, 6)
    module.hparams.TEST.VISUALIZE = "no"
    R1_mAP(module, 6)  # the samples are only needed for the visualisation
