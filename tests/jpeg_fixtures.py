"""The JPEG fixture set of tests/test_jpeg_cpu.py and tests/test_jpeg_gpu.py: files Pillow encodes here from seeded
images (every size up to 17 x 17, prime sides, re-id crop sizes, one 1000 x 500 source; subsampling 4:4:4 / 4:2:2 /
4:2:0 and grayscale; quality 1 to 100, optimised Huffman tables, restart intervals, 8- and 16-bit quantisation tables),
files whose quantisation tables are raised after encoding (IDCT outputs far outside 0..255), and the OpenCV-encoded
4:1:1 / 4:4:0 files committed in tests/golden/jpeg_opencv.npz."""
from __future__ import annotations

import functools
import io
import os
import warnings

import numpy as np
from PIL import Image

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PRIMES = [p for p in range(2, 132) if all(p % d for d in range(2, int(p ** 0.5) + 1))]
SUBS = (0, 1, 2, "L")  # Pillow's subsampling 4:4:4, 4:2:2, 4:2:0; "L": grayscale
QUALITIES = (1, 50, 75, 95, 100)


def duke_sizes(n, seed=0):
    """Seeded (h, w) between 60 x 30 and 400 x 200, the spread of DukeMTMC-reID's crops."""
    rng = np.random.default_rng(seed)
    return [(int(h), int(w)) for h, w in zip(rng.integers(60, 401, n), rng.integers(30, 201, n))]


def make_image(kind, h, w, seed=0):
    if kind == "random":
        return np.random.default_rng(seed + 7 * h + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind in ("zeros", "ones"):
        return np.full((h, w, 3), 0 if kind == "zeros" else 255, dtype=np.uint8)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    if kind == "ramp":
        return np.stack([x * 255 / max(w - 1, 1), y * 255 / max(h - 1, 1), 255 - x * 255 / max(w - 1, 1)],
                        -1).astype(np.uint8)
    # smooth: low-frequency colour fields, the spectrum of a photograph more than of noise
    r = 128 + 100 * np.sin(x / 9.0 + seed) * np.cos(y / 13.0)
    g = 128 + 90 * np.cos((x + y) / 17.0 + seed)
    b = 128 + 80 * np.sin(y / 7.0 - seed) * np.sin(x / 23.0)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def encode(img, sub=2, **kw):
    """Pillow's JPEG of an RGB array; sub "L" encodes its luma as grayscale."""
    buf = io.BytesIO()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # "quantization tables are too coarse for baseline JPEG" (SOF1)
        if sub == "L":
            Image.fromarray(img, "RGB").convert("L").save(buf, "JPEG", **kw)
        else:
            Image.fromarray(img, "RGB").save(buf, "JPEG", subsampling=sub, **kw)
    return buf.getvalue()


def raise_tables(data, factor=4):
    """The file with every quantisation value multiplied by `factor` (capped at 255): its entropy-coded data is
    unchanged, and the dequantised blocks overshoot far past 0..255."""
    from jpeg_oracle import parse

    b = bytearray(data)
    d = parse(data)
    for c in range(d["ncomp"]):
        off = d["dqt"][c]
        for k in range(64):
            b[off + k] = min(255, b[off + k] * factor)
    return bytes(b)


def opencv_files():
    z = np.load(os.path.join(GOLDEN, "jpeg_opencv.npz"))
    data, off = z["data"], z["offsets"]
    return [(f"opencv {lab}", data[off[i]: off[i + 1]].tobytes()) for i, lab in enumerate(z["labels"].tolist())]


@functools.lru_cache(maxsize=None)
def fixtures():
    """[(label, file bytes)], deterministic."""
    out = []
    i = 0
    for h in range(1, 18):
        for w in range(1, 18):
            for sub in SUBS:
                kind = "random" if i % 2 == 0 else "smooth"
                q = QUALITIES[i % len(QUALITIES)]
                out.append((f"{h}x{w} sub{sub} {kind} q{q}", encode(make_image(kind, h, w, i), sub, quality=q)))
                i += 1
    for j, p in enumerate(PRIMES):
        h, w = p, PRIMES[-1 - j]
        sub = SUBS[j % 4]
        out.append((f"prime {h}x{w} sub{sub}", encode(make_image("random" if j % 3 else "smooth", h, w, j), sub)))
    for h, w in [(128, 64), (256, 128)] + duke_sizes(4):
        for sub in SUBS:
            out.append((f"{h}x{w} sub{sub} smooth", encode(make_image("smooth", h, w, h), sub, quality=90)))
    out.append(("1000x500 sub2 smooth", encode(make_image("smooth", 1000, 500, 3), 2, quality=90)))
    for q in QUALITIES:
        for sub in SUBS:
            for kind in ("random", "smooth"):
                out.append((f"37x29 sub{sub} {kind} q{q}", encode(make_image(kind, 37, 29, q), sub, quality=q)))
                out.append((f"37x29 sub{sub} {kind} q{q} optimize",
                            encode(make_image(kind, 37, 29, q), sub, quality=q, optimize=True)))
    for sub in SUBS:
        img = make_image("random", 45, 61, 5)
        out.append((f"45x61 sub{sub} rst blocks 1", encode(img, sub, restart_marker_blocks=1)))
        out.append((f"45x61 sub{sub} rst blocks 3", encode(img, sub, restart_marker_blocks=3)))
        out.append((f"45x61 sub{sub} rst rows 1", encode(img, sub, restart_marker_rows=1)))
        ramp = [min(1 + 16 * k, 1000) for k in range(64)]  # values > 255: 16-bit tables, SOF1
        out.append((f"45x61 sub{sub} 16-bit qtables", encode(img, sub, qtables=[ramp, [300] * 64])))
        out.append((f"45x61 sub{sub} 8-bit qtables", encode(img, sub, qtables=[[1 + k for k in range(64)], [7] * 64])))
        for kind in ("zeros", "ones", "ramp"):
            out.append((f"45x61 sub{sub} {kind}", encode(make_image(kind, 45, 61), sub)))
        out.append((f"24x40 sub{sub} raised tables", raise_tables(encode(make_image("random", 24, 40, 1), sub,
                                                                         quality=50))))
    out += opencv_files()
    return tuple(out)


def pillow_decode(data):
    """The reference's decode: Image.open(p).convert("RGB") (datasets/bases.py:32-33)."""
    with Image.open(io.BytesIO(data)) as im:
        return np.asarray(im.convert("RGB"))
