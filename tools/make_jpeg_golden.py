"""Writes tests/golden/jpeg_opencv.npz: OpenCV-encoded JPEGs with the 4:1:1 and 4:4:0 sampling factors Pillow's encoder
cannot write, for tests/test_jpeg_cpu.py and tests/test_jpeg_gpu.py.  OpenCV may be absent where the tests run, so
the files are committed as data.  Arrays: `data` uint8 (the files back to back), `offsets` int64 [n + 1],
`labels` str [n] ("<sampling> <h>x<w> <content> q<quality>").

    python tools/make_jpeg_golden.py
"""
import os

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(1, 1), (1, 5), (3, 2), (7, 9), (8, 8), (9, 17), (16, 32), (17, 33), (31, 4), (64, 128), (128, 64)]


def content(kind, h, w, seed):
    if kind == "random":
        return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)
    y, x = np.mgrid[0:h, 0:w]
    return np.stack([(x * 255 // max(w - 1, 1)), (y * 255 // max(h - 1, 1)), ((x + y) * 7) % 256], -1).astype(np.uint8)


def main():
    blobs, labels = [], []
    for name in ("411", "440"):
        flag = getattr(cv2, f"IMWRITE_JPEG_SAMPLING_FACTOR_{name}")
        for i, (h, w) in enumerate(SIZES):
            for kind, q in (("random", 75), ("smooth", 95)):
                ok, buf = cv2.imencode(".jpg", content(kind, h, w, i), [cv2.IMWRITE_JPEG_QUALITY, q,
                                                                        cv2.IMWRITE_JPEG_SAMPLING_FACTOR, flag])
                assert ok
                blobs.append(buf.tobytes())
                labels.append(f"{name} {h}x{w} {kind} q{q}")
    offsets = np.cumsum([0] + [len(b) for b in blobs]).astype(np.int64)
    data = np.frombuffer(b"".join(blobs), dtype=np.uint8)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "jpeg_opencv.npz"), data=data, offsets=offsets,
                        labels=np.array(labels))


if __name__ == "__main__":
    main()
