"""GPU: the block-parallel entropy decode of ctl_jpeg_decode (one CTA per image, subsequences brought into step by
sync rounds) on sources larger than tests/test_jpeg_gpu.py's fixtures -- ~500 px and 2000 x 1500 files at every
sampling and at q 75 / 90 / 100 with optimised tables, a scan long enough that the subsequence length grows, random
content at q100, a constant image, restart intervals of every length -- and on the fixtures the host model
(tests/jpeg_sync_model.py) finds slowest to converge, all bit for bit against Pillow; corrupt files against the status
and output of the serial decode it replaced (tests/golden/jpeg_corrupt.npz); and batch invariance, repeatability and
CUDA-graph replay."""
import functools
import hashlib
import os

import numpy as np
import pytest
import torch

import jpeg_sync_model as M
from jpeg_fixtures import GOLDEN, encode, fixtures, make_image, opencv_files, pillow_decode

pytestmark = pytest.mark.gpu

SUBS = (2, 1, 0, "L")


def _T():
    from ctl_b200.datasets import transforms as T

    return T


def _images(ragged):
    data, table = ragged.data.cpu().numpy(), ragged.table.cpu().numpy()
    return [None if h == 0 else data[o: o + h * w * 3].reshape(h, w, 3) for o, h, w in table]


def _decode(files):
    T = _T()
    return _images(T.decode_batch(T.pack_jpegs(files, pin=False).to("cuda")))


def _check(files, labels):
    got = _decode(files)
    wrong = [lab for g, f, lab in zip(got, files, labels) if not np.array_equal(g, pillow_decode(f))]
    assert not wrong, wrong[:20]


def noisy(h, w, seed, sigma=6.0):
    """smooth colour fields plus seeded Gaussian noise: a photograph's spectrum and bit rate"""
    img = make_image("smooth", h, w, seed).astype(np.float64)
    img += np.random.default_rng(seed).normal(0, sigma, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def about_500px(n, seed=0):
    rng = np.random.default_rng(seed)
    return [noisy(int(h), int(w), seed * 100 + i) for i, (h, w) in enumerate(zip(rng.integers(400, 601, n),
                                                                                rng.integers(250, 351, n)))]


@functools.lru_cache(maxsize=None)
def big():
    return noisy(1500, 2000, 11)


def scan_bits(data):
    d = M.JO.parse(data)
    segs, _ = M.segment_table(data, d, 1 << 30)
    return 8 * segs[-1][3]


@pytest.mark.parametrize("q", [75, 90, 100])
def test_about_500px_every_sampling(q):
    files, labels = [], []
    for i, img in enumerate(about_500px(6, seed=q)):
        for sub in SUBS:
            files.append(encode(img, sub, quality=q, optimize=True))
            labels.append(f"500px #{i} sub{sub} q{q}")
    _check(files, labels)


@pytest.mark.parametrize("sub", SUBS, ids=[f"sub{s}" for s in SUBS])
def test_2000x1500_every_quality(sub):
    files = [encode(big(), sub, quality=q, optimize=True) for q in (75, 90, 100)]
    _check(files, [f"2000x1500 sub{sub} q{q}" for q in (75, 90, 100)])


def test_scan_longer_than_every_subsequence_at_the_shortest_length():
    """a scan of more than T * S_MIN bits: the subsequence length grows instead of the count"""
    f = encode(big(), 0, quality=100)
    bits = scan_bits(f)
    S, nsub = M.sub_bits(bits)
    assert bits > M.T * M.S_MIN and S > M.S_MIN and nsub <= M.T
    _check([f], ["2000x1500 sub0 q100"])


def test_random_q100_and_constant_images():
    rnd = np.random.default_rng(3).integers(0, 256, (480, 640, 3), dtype=np.uint8)
    files = [encode(rnd, sub, quality=100) for sub in SUBS]
    files += [encode(np.full((1500, 2000, 3), v, np.uint8), sub) for v in (0, 200) for sub in (2, "L")]
    _check(files, [f"{i}" for i in range(len(files))])


def test_opencv_411_440_in_one_batch():
    files = opencv_files()
    _check([f for _, f in files], [lab for lab, _ in files])


@pytest.mark.parametrize("kw", [dict(restart_marker_blocks=1), dict(restart_marker_rows=1),
                                dict(restart_marker_blocks=7), dict(restart_marker_blocks=50),
                                dict(restart_marker_rows=3)],
                         ids=["blocks1", "rows1", "blocks7", "blocks50", "rows3"])
def test_restart_intervals_on_large_sources(kw):
    files, labels = [], []
    for sub in SUBS:
        files.append(encode(big(), sub, quality=90, **kw))
        labels.append(f"2000x1500 sub{sub} {kw}")
    for i, img in enumerate(about_500px(2, seed=5)):
        files.append(encode(img, (2, "L")[i], quality=95, **kw))
        labels.append(f"500px #{i} {kw}")
    _check(files, labels)


@functools.lru_cache(maxsize=None)
def worst_sync(count=24):
    """the fixtures the host model needs the most sync rounds for"""
    scored = []
    for label, data in fixtures():
        if 8 * len(data) <= M.S_MIN:  # one subsequence: nothing to synchronise
            continue
        scored.append((M.decode(data)["rounds"], label, data))
    scored.sort(key=lambda t: -t[0])
    return scored[:count]


def test_worst_sync_fixtures():
    picks = worst_sync()
    assert picks[0][0] >= 3
    _check([d for _, _, d in picks], [f"{lab} ({r} rounds)" for r, lab, _ in picks])


def test_corrupt_files_give_the_serial_decodes_status_and_output():
    z = np.load(os.path.join(GOLDEN, "jpeg_corrupt.npz"))
    data, off = z["data"], z["offsets"]
    files = [data[off[i]: off[i + 1]].tobytes() for i in range(len(off) - 1)]
    labels, want, sha = z["labels"].tolist(), z["status"], z["sha256"].tolist()
    assert (want != 0).sum() > 20 and (want == 0).sum() > 10
    T = _T()
    batch = T.pack_jpegs(files, pin=False)
    dev = batch.to("cuda")
    out = torch.full((batch.out_bytes,), 77, dtype=torch.uint8, device="cuda")
    status = torch.full((len(batch),), -1, dtype=torch.int32, device="cuda")
    ws = torch.empty(batch.workspace_bytes, dtype=torch.uint8, device="cuda")
    T._decode_enqueue(dev, out, status, ws)
    st = status.cpu().numpy()
    host = out.cpu().numpy()
    wrong = []
    for i, (o, h, w) in enumerate(batch.out_table.numpy()):
        img = host[o: o + h * w * 3]
        if st[i] != want[i] or hashlib.sha256(img.tobytes()).hexdigest() != sha[i] or (st[i] and img.any()):
            wrong.append((labels[i], int(st[i]), int(want[i])))
    assert not wrong, wrong[:20]


def _mixed_256():
    rng = np.random.default_rng(17)
    files = []
    for i in range(256):
        h, w = int(rng.integers(20, 601)), int(rng.integers(16, 401))
        files.append(encode(noisy(h, w, i) if i % 3 else make_image("random", h, w, i), SUBS[i % 4],
                            quality=(75, 90, 100)[i % 3], restart_marker_blocks=(0, 0, 5)[i % 3]))
    return files


def test_batch_of_256_mixed_sizes_equals_each_image_alone():
    files = _mixed_256()
    together = _decode(files)
    for i in range(0, 256, 5):
        assert np.array_equal(together[i], _decode([files[i]])[0]), i
    for i in range(256):
        assert np.array_equal(together[i], pillow_decode(files[i])), i


def test_repeat_and_graph_replay_are_bit_identical():
    T = _T()
    b = T.pack_jpegs(_mixed_256()[:96]).to("cuda")
    first = T.decode_batch(b).data
    second = T.decode_batch(b).data
    assert torch.equal(first, second)
    out = torch.empty_like(first)
    status = torch.ones(len(b), dtype=torch.int32, device="cuda")
    ws = torch.empty(b.workspace_bytes, dtype=torch.uint8, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        T._decode_enqueue(b, out, status, ws)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        T._decode_enqueue(b, out, status, ws)
    out.zero_()
    status.fill_(5)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, first) and not status.any()
