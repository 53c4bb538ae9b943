"""CPU: the host restatement of PIL's BILINEAR resize (oracle/resize_oracle.py) against Pillow itself, the ragged
packing of datasets/transforms.pack_images, and the host-side argument checks of ctl_resize_bilinear_u8."""
import ctypes as C

import numpy as np
import pytest
from PIL import Image

from ctl_b200 import _native as N
from ctl_b200.datasets import transforms as T
from oracle import resize_oracle as RO

PRIMES = [p for p in range(2, 132) if all(p % d for d in range(2, int(p ** 0.5) + 1))]
TARGETS = [(256, 128), (320, 320), (384, 128), (1, 1), None]  # (h, w); None: the identity


def duke_sizes(n, seed=0):
    """Seeded (h, w) between 60 x 30 and 400 x 200, the spread of DukeMTMC-reID's crops."""
    rng = np.random.default_rng(seed)
    return [(int(h), int(w)) for h, w in zip(rng.integers(60, 401, n), rng.integers(30, 201, n))]


def sweep_sources():
    src = [(h, w) for h in range(1, 10) for w in range(1, 10)]
    src += [(p, PRIMES[-1 - i]) for i, p in enumerate(PRIMES)]  # every prime as a height and as a width
    src += [(128, 64)] + duke_sizes(8) + [(2000, 1000)]
    return src


def make_image(kind, h, w, seed=0):
    if kind == "random":
        return np.random.default_rng(seed + 7 * h + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind in ("zeros", "ones"):
        return np.full((h, w, 3), 0 if kind == "zeros" else 255, dtype=np.uint8)
    ramp = (np.arange(w if kind == "hramp" else h) * 255 // max((w if kind == "hramp" else h) - 1, 1)).astype(np.uint8)
    img = np.empty((h, w, 3), dtype=np.uint8)
    img[...] = ramp[None, :, None] if kind == "hramp" else ramp[:, None, None]
    img[..., 1] = 255 - img[..., 1]
    return img


KINDS = ["random", "zeros", "ones", "hramp", "vramp"]


def pil_resize(img, oh, ow):
    return np.asarray(Image.fromarray(img, "RGB").resize((ow, oh), Image.BILINEAR))


@pytest.mark.parametrize("target", TARGETS, ids=lambda t: "identity" if t is None else f"{t[0]}x{t[1]}")
def test_oracle_equals_pil(target):
    for h, w in sweep_sources():
        oh, ow = (h, w) if target is None else target
        for kind in KINDS:
            img = make_image(kind, h, w)
            got = RO.resize_bilinear(img, oh, ow)
            ref = pil_resize(img, oh, ow)
            assert got.shape == (oh, ow, 3) and np.array_equal(got, ref), (h, w, oh, ow, kind)


def test_oracle_coefficients_sum_to_one_in_fixed_point():
    for n_in, n_out in ((64, 128), (128, 320), (2000, 256), (1, 320), (7, 3), (256, 256)):
        xmin, k = RO.axis_coeffs(n_in, n_out)
        assert (k >= 0).all() and (xmin >= 0).all()
        s = k.sum(1)
        assert (abs(s - (1 << 22)) <= k.shape[1]).all(), (n_in, n_out)  # each weight rounds by at most one half
    xmin, k = RO.axis_coeffs(256, 256)  # identity: taps {1, 0}
    assert np.array_equal(xmin, np.arange(256)) and (k[:, 0] == 1 << 22).all() and (k[:, 1:] == 0).all()


def test_pack_images_layout():
    imgs = [make_image("random", 3, 5), None, make_image("hramp", 1, 1),
            Image.fromarray(make_image("vramp", 4, 7), "RGB"), None, make_image("random", 9, 2)]
    r = T.pack_images(imgs, pin=False)
    assert len(r) == 6
    table = r.table.numpy()
    assert table.dtype == np.int64 and table.shape == (6, 3)
    sizes = [(3, 5), (0, 0), (1, 1), (4, 7), (0, 0), (9, 2)]
    off = 0
    for i, (h, w) in enumerate(sizes):
        if h == 0:
            assert table[i].tolist() == [0, 0, 0]
            continue
        assert table[i].tolist() == [off, h, w]
        a = np.asarray(imgs[i])
        assert np.array_equal(r.data.numpy()[off: off + h * w * 3].reshape(h, w, 3), a)
        off += h * w * 3
    assert r.data.numel() == off and r.rows == 3 + 1 + 4 + 9
    assert table[2, 0] == 45 and table[3, 0] == 48  # back to back: odd, unaligned offsets
    only_mock = T.pack_images([None, None], pin=False)
    assert only_mock.rows == 0 and only_mock.data.numel() == 1 and only_mock.table.numpy().tolist() == [[0, 0, 0]] * 2


@pytest.mark.parametrize("bad", [
    [],
    [np.zeros((4, 4, 3), dtype=np.float32)],
    [np.zeros((4, 4), dtype=np.uint8)],
    [np.zeros((4, 4, 4), dtype=np.uint8)],
    [np.zeros((0, 4, 3), dtype=np.uint8)],
    [Image.new("L", (4, 4))],
    [Image.new("RGBA", (4, 4))],
])
def test_pack_images_rejects(bad):
    with pytest.raises(ValueError):
        T.pack_images(bad, pin=False)


def test_workspace_bytes():
    L = N.lib()
    assert L.ctl_resize_bilinear_u8_workspace_bytes(1000, 256, 128) == 1000 * 128 * 3
    assert L.ctl_resize_bilinear_u8_workspace_bytes(7, 1, 1) == 256  # rounded up to 256 bytes
    assert L.ctl_resize_bilinear_u8_workspace_bytes(0, 256, 128) == 512  # all mock rows: one row, rounded
    for args in ((-1, 256, 128), (10, 0, 128), (10, 256, 0), (10, -5, 128), (10, 16385, 128), (10, 256, 16385)):
        assert L.ctl_resize_bilinear_u8_workspace_bytes(*args) == 0, args
    r = T.pack_images([make_image("random", 128, 64)] * 3 + [None], pin=False)
    assert T.resize_workspace_bytes(r, (256, 128)) == 3 * 128 * 128 * 3
    for size in (256, (256,), (256, 128, 3), (0, 128)):
        with pytest.raises(ValueError):
            T.resize_workspace_bytes(r, size)


def test_argument_errors_are_reported_without_a_gpu():
    L = N.lib()
    one = C.c_void_p(256)

    def call(src=one, src_bytes=1000, table=one, n=4, oh=256, ow=128, out=one, status=one, ws=one, ws_bytes=10**6):
        return L.ctl_resize_bilinear_u8(src, src_bytes, table, n, oh, ow, out, status, ws, ws_bytes, None)

    cases = [
        lambda: call(src=None), lambda: call(table=None), lambda: call(out=None), lambda: call(status=None),
        lambda: call(ws=None), lambda: call(n=0), lambda: call(n=-3), lambda: call(n=1 << 31), lambda: call(oh=0),
        lambda: call(ow=0), lambda: call(oh=16385), lambda: call(ow=20000), lambda: call(src_bytes=-1),
        lambda: call(ws_bytes=128 * 3 - 1),  # shorter than one intermediate row
    ]
    for i, c in enumerate(cases):
        rc = c()
        assert rc == -1, (i, rc, L.ctl_last_error())
        assert len(L.ctl_last_error()) > 0
        with pytest.raises(ValueError):
            N.check(rc)
