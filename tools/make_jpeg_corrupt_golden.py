"""Writes tests/golden/jpeg_corrupt.npz: seeded corruptions of JPEG fixture files and what a given build of
`ctl_jpeg_decode` makes of them, so that a later decode can be held to the same per-file status.  The corpus:
truncations at many offsets inside the scan, single bit flips in the scan, a deleted RSTn marker, an out-of-sequence
RSTn, garbage bytes (with and without a stuffed 0xFF 0x00) before an RSTn, 0xFF fill bytes before an RSTn and before
EOI, and bytes after EOI.  Arrays: `data` uint8 (the files back to back), `offsets` int64 [n + 1], `labels` str [n],
`status` int32 [n] (the decode's status word per file), `sha256` str [n] (of each file's RGB output).

    python tools/make_jpeg_corrupt_golden.py [--lib path/to/libctl_b200.so] [--out path.npz]

Needs a CUDA device.  Without --lib it uses the library built in the tree.
"""
import argparse
import ctypes as C
import hashlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import ctl_b200  # noqa: E402,F401
from ctl_b200 import _native as N  # noqa: E402
from ctl_b200.datasets import transforms as T  # noqa: E402
from jpeg_fixtures import encode, make_image  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "jpeg_corrupt.npz")


def _scan(data):
    """(first byte of the entropy-coded data, index of the EOI marker)"""
    from jpeg_oracle import parse

    return parse(data)["scan_begin"], data.rfind(b"\xff\xd9")


def _rst_positions(data):
    begin, eoi = _scan(data)
    return [i for i in range(begin, eoi - 1) if data[i] == 0xFF and 0xD0 <= data[i + 1] <= 0xD7]


def corpus(seed=0):
    """[(label, file bytes)], deterministic."""
    rng = np.random.default_rng(seed)
    bases = [
        ("45x61 sub2 random", encode(make_image("random", 45, 61, 5), 2)),
        ("128x64 sub2 smooth q90", encode(make_image("smooth", 128, 64, 3), 2, quality=90)),
        ("45x61 sub0 rst blocks 3", encode(make_image("random", 45, 61, 5), 0, restart_marker_blocks=3)),
        ("61x45 subL rst rows 1", encode(make_image("smooth", 61, 45, 2), "L", restart_marker_rows=1)),
        ("96x80 sub2 rst blocks 1", encode(make_image("random", 96, 80, 4), 2, restart_marker_blocks=1)),
    ]
    out = []
    for name, f in bases:
        begin, eoi = _scan(f)
        out.append((f"{name} intact", f))
        for cut in np.unique(np.linspace(begin, eoi + 2, 14).astype(int)):
            out.append((f"{name} cut at {cut}", f[:cut]))
        for _ in range(12):
            i = int(rng.integers(begin, eoi))
            b = bytearray(f)
            b[i] ^= 1 << int(rng.integers(0, 8))
            out.append((f"{name} flip byte {i}", bytes(b)))
        out.append((f"{name} fill before EOI", f[:eoi] + b"\xff\xff\xff" + f[eoi:]))
        out.append((f"{name} bytes after EOI", f + bytes(rng.integers(0, 256, 64, dtype=np.uint8))))
        out.append((f"{name} EOI removed", f[:eoi]))
        rst = _rst_positions(f)
        for r in (rst[:1] + rst[len(rst) // 2: len(rst) // 2 + 1]) if rst else []:
            out.append((f"{name} RST at {r} deleted", f[:r] + f[r + 2:]))
            b = bytearray(f)
            b[r + 1] = 0xD0 + ((b[r + 1] - 0xD0 + 2) & 7)
            out.append((f"{name} RST at {r} out of sequence", bytes(b)))
            out.append((f"{name} garbage before RST at {r}", f[:r] + b"\x12\x34\x56" + f[r:]))
            out.append((f"{name} stuffed garbage before RST at {r}", f[:r] + b"\x12\xff\x00\x56" + f[r:]))
            out.append((f"{name} fill before RST at {r}", f[:r] + b"\xff\xff" + f[r:]))
    return out


def library(path=None):
    """ctl_jpeg_decode of the library at `path` (default: the tree's), with the argument types of the C ABI."""
    if path is None:
        return N.lib().ctl_jpeg_decode
    fn = C.CDLL(os.path.abspath(path)).ctl_jpeg_decode
    p, i64, sz = C.c_void_p, C.c_int64, C.c_size_t
    fn.restype = C.c_int
    fn.argtypes = [p, i64, p, i64, p, p, i64, p, p, sz, p]
    return fn


def decode_with(fn, batch):
    """(status [n], RGB output bytes) of one device JpegBatch decoded by ctl_jpeg_decode `fn`."""
    out = torch.zeros(max(batch.out_bytes, 1), dtype=torch.uint8, device="cuda")
    status = torch.full((len(batch),), -1, dtype=torch.int32, device="cuda")
    ws = torch.empty(batch.workspace_bytes, dtype=torch.uint8, device="cuda")
    rc = fn(batch.data.data_ptr(), batch.data.numel(), batch.entries.data_ptr(), len(batch),
            batch.out_table.data_ptr(), out.data_ptr(), batch.out_bytes, status.data_ptr(), ws.data_ptr(), ws.numel(),
            N.stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()
    return status.cpu().numpy(), out.cpu().numpy()


def run(fn, files):
    """per file: (status, sha256 of its RGB output)"""
    batch = T.pack_jpegs(files, pin=False)
    assert not batch.fallback, batch.fallback
    st, out = decode_with(fn, batch.to("cuda"))
    table = batch.out_table.numpy()
    return st, [hashlib.sha256(out[o: o + h * w * 3].tobytes()).hexdigest() for o, h, w in table]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    ap.add_argument("--out", default=OUT)
    a = ap.parse_args()
    files = corpus()
    labels = [lab for lab, _ in files]
    blobs = [f for _, f in files]
    st, sha = run(library(a.lib), blobs)
    offsets = np.cumsum([0] + [len(b) for b in blobs]).astype(np.int64)
    np.savez_compressed(a.out, data=np.frombuffer(b"".join(blobs), dtype=np.uint8), offsets=offsets,
                        labels=np.array(labels), status=st.astype(np.int32), sha256=np.array(sha))
    print(f"{len(files)} files, {int((st != 0).sum())} with a nonzero status -> {a.out}")


if __name__ == "__main__":
    main()
