"""CPU: the host restatement of libjpeg-turbo's decode (tests/jpeg_oracle.py) against Pillow itself on the fixture set
of tests/jpeg_fixtures.py, the host parser ctl_jpeg_parse against the oracle's, the packing of
datasets/transforms.pack_jpegs, and the host-side argument checks of ctl_jpeg_decode."""
import ctypes as C
import functools
import hashlib
import io
import os
import subprocess
import sys

import numpy as np
import pytest
from PIL import Image, features

import jpeg_oracle as JO
from jpeg_fixtures import encode, fixtures, make_image, pillow_decode
from ctl_b200 import _native as N
from ctl_b200.datasets import transforms as T

HERE = os.path.dirname(os.path.abspath(__file__))


@functools.lru_cache(maxsize=None)
def oracle_run():
    """(labels of fixtures the oracle decodes differently from Pillow, edge-rule counters over the set)."""
    counters, wrong = {}, []
    for label, data in fixtures():
        if not np.array_equal(JO.decode(data, counters), pillow_decode(data)):
            wrong.append(label)
    return wrong, counters


def test_oracle_equals_pillow():
    wrong, _ = oracle_run()
    assert len(fixtures()) > 1300
    assert not wrong, wrong[:20]


def test_fixtures_reach_every_edge_rule():
    _, counters = oracle_run()
    for rule in ("idct_wrap", "narrow_fallback", "edge_right", "edge_bottom"):
        assert counters.get(rule, 0) > 0, (rule, counters)


def test_fixtures_cover_the_scope():
    kinds = set()
    for _, data in fixtures():
        d = JO.parse(data)
        kinds.add((d["ncomp"], tuple(d["hs"][: d["ncomp"]]), tuple(d["vs"][: d["ncomp"]])))
        if d["restart_interval"]:
            kinds.add("restart")
        if d["dqt16"]:
            kinds.add("dqt16")
        if b"\xff\xc1" in data[: d["scan_begin"]]:
            kinds.add("SOF1")
    for k in [(1, (1,), (1,)), (3, (1, 1, 1), (1, 1, 1)), (3, (2, 1, 1), (1, 1, 1)), (3, (2, 1, 1), (2, 1, 1)),
              (3, (1, 1, 1), (2, 1, 1)), (3, (4, 1, 1), (1, 1, 1)), "restart", "dqt16", "SOF1"]:
        assert k in kinds, k


_SIMD_PROBE = """
import hashlib, sys
sys.path.insert(0, {here!r})
from jpeg_fixtures import fixtures, pillow_decode
h = hashlib.sha256()
for label, data in fixtures():
    if "raised tables" not in label:
        h.update(pillow_decode(data).tobytes())
print(h.hexdigest())
"""


def test_pillow_decode_does_not_depend_on_the_simd_path():
    """Pillow decodes with libjpeg-turbo, and its C path (JSIMD_FORCENONE=1) gives the same bits as the SIMD path on
    every encoder-made fixture.  (The raised-table files are left out: there the SIMD IDCT saturates and the C path's
    range_limit table wraps, and Pillow -- the SIMD path -- is what the decode follows.)"""
    assert features.check_feature("libjpeg_turbo")
    h = hashlib.sha256()
    for label, data in fixtures():
        if "raised tables" not in label:
            h.update(pillow_decode(data).tobytes())
    env = dict(os.environ, JSIMD_FORCENONE="1")
    out = subprocess.run([sys.executable, "-c", _SIMD_PROBE.format(here=HERE)], env=env, capture_output=True,
                         text=True, check=True)
    assert out.stdout.strip() == h.hexdigest()


DESC_FIELDS = ("h", "w", "scan_begin", "scan_end", "restart_interval", "ncomp", "dqt16")


def desc_dict(desc):
    d = {f: getattr(desc, f) for f in DESC_FIELDS}
    for f in ("dqt", "dht_dc", "dht_ac", "hs", "vs"):
        d[f] = list(getattr(desc, f))
    return d


def test_parse_matches_oracle():
    for label, data in fixtures():
        desc, why = T.parse_jpeg(data)
        assert why is None, (label, why)
        assert desc_dict(desc) == JO.parse(data), label
    h, w = C.c_int32(), C.c_int32()
    data = fixtures()[100][1]
    assert N.lib().ctl_jpeg_parse(data, len(data), C.byref(N.JpegDesc()), C.byref(h), C.byref(w)) == 0
    assert (h.value, w.value) == (JO.parse(data)["h"], JO.parse(data)["w"])


def _patched(data, marker, offset, value):
    """data with the byte `offset` after the first occurrence of `marker` set to value"""
    b = bytearray(data)
    i = b.find(marker)
    assert i > 0
    b[i + offset] = value
    return bytes(b)


def rejected_files():
    img = make_image("random", 40, 32)
    base = encode(img, 2)
    png = io.BytesIO()
    Image.fromarray(img).save(png, "PNG")
    cmyk = io.BytesIO()
    Image.fromarray(img).convert("CMYK").save(cmyk, "JPEG")
    sos = base.find(b"\xff\xda")
    return [
        ("progressive", encode(img, 2, progressive=True), "progressive"),
        ("cmyk", cmyk.getvalue(), "CMYK"),
        ("12-bit", _patched(base, b"\xff\xc0", 4, 12), "12-bit"),          # SOF precision byte
        ("arithmetic", _patched(base, b"\xff\xc0", 1, 0xC9), "arithmetic"),  # SOF0 -> SOF9
        ("lossless", _patched(base, b"\xff\xc0", 1, 0xC3), "lossless"),
        ("truncated header", base[:sos - 7], "truncated"),
        ("no SOS", base[:sos], "truncated"),
        ("png", png.getvalue(), "not a JPEG"),
        ("empty", b"", "not a JPEG"),
        ("text", b"hello, world", "not a JPEG"),
    ]


@pytest.mark.parametrize("name,data,reason", rejected_files(), ids=[r[0] for r in rejected_files()])
def test_parse_rejects(name, data, reason):
    desc, why = T.parse_jpeg(data)
    assert desc is None and reason in why, (name, why)
    with pytest.raises(ValueError):
        JO.parse(data)


def test_parse_rejects_adobe_rgb():
    """A 3-component file without JFIF and with Adobe transform 0 is RGB, not YCbCr: out of scope."""
    base = encode(make_image("random", 16, 16), 0)
    assert base[2:4] == b"\xff\xe0"
    app0_len = base[4] << 8 | base[5]
    adobe = b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00"  # transform 0
    data = base[:2] + adobe + base[4 + app0_len:]
    desc, why = T.parse_jpeg(data)
    assert desc is None and "Adobe RGB" in why
    ycc = data.replace(adobe, adobe[:-1] + b"\x01")  # transform 1: YCbCr
    assert T.parse_jpeg(ycc)[0] is not None
    assert np.array_equal(JO.decode(ycc), pillow_decode(ycc))


def entry(batch, i):
    return N.JpegEntry.from_buffer_copy(batch.entries[i].numpy().tobytes())


def test_pack_jpegs_layout(tmp_path):
    j1 = encode(make_image("random", 13, 7), 2)
    j2 = encode(make_image("smooth", 20, 31), "L")
    prog = encode(make_image("random", 9, 5), 2, progressive=True)
    png = io.BytesIO()
    Image.fromarray(make_image("ramp", 6, 11)).save(png, "PNG")
    path = tmp_path / "a.jpg"
    path.write_bytes(j2)
    items = [j1, None, prog, str(path), png.getvalue(), None, bytearray(j1)]
    b = T.pack_jpegs(items, pin=False)
    assert len(b) == 7 and b.entries.shape == (7, C.sizeof(N.JpegEntry)) == (7, 88)
    kinds = [entry(b, i).kind for i in range(7)]
    J, R, M = N.CTL_JPEG_ENTRY_JPEG, N.CTL_JPEG_ENTRY_RAW, N.CTL_JPEG_ENTRY_MOCK
    assert kinds == [J, M, R, J, R, M, J]
    assert [i for i, _ in b.fallback] == [2, 4] and "progressive" in b.fallback[0][1]
    sizes = [(13, 7), (0, 0), (9, 5), (20, 31), (6, 11), (0, 0), (13, 7)]
    off = out = 0
    data = b.data.numpy()
    for i, (h, w) in enumerate(sizes):
        e = entry(b, i)
        assert b.out_table[i].tolist() == ([out, h, w] if h else [0, 0, 0])
        if kinds[i] == M:
            continue
        assert (e.offset, e.desc.h, e.desc.w) == (off, h, w)
        blob = data[off: off + e.nbytes].tobytes()
        if kinds[i] == J:
            assert blob == bytes(items[i]) if i != 3 else blob == j2
            assert desc_dict(e.desc) == JO.parse(blob)
        else:
            src = prog if i == 2 else png.getvalue()
            assert np.array_equal(np.frombuffer(blob, np.uint8).reshape(h, w, 3), pillow_decode(src))
        off += e.nbytes
        out += h * w * 3
    assert b.data.numel() == off and b.out_bytes == out and b.rows == 13 + 9 + 20 + 6 + 13
    assert entry(b, 6).offset % 2 == 1 or entry(b, 3).offset % 2 == 1  # back to back: unaligned offsets
    assert T.pack_jpegs([None, None], pin=False).out_bytes == 0


@pytest.mark.parametrize("bad", [[], [3], [b"not an image"], [np.zeros((4, 4, 3), np.uint8)]])
def test_pack_jpegs_rejects(bad):
    with pytest.raises(ValueError):
        T.pack_jpegs(bad, pin=False)


def test_workspace_bytes():
    items = [encode(make_image("random", 128, 64), 2), None, encode(make_image("random", 17, 9), 0),
             encode(make_image("random", 30, 21), "L"), encode(make_image("random", 5, 5), 2, progressive=True)]
    b = T.pack_jpegs(items, pin=False)
    blocks = 8 * 4 * 4 + 2 * (8 * 4)       # 4:2:0 128 x 64: 8 x 4 MCUs of 4 luma blocks + one per chroma component
    blocks += 3 * 3 * 2                     # 4:4:4 17 x 9: 3 x 2 blocks per component
    blocks += 4 * 3                         # grayscale 30 x 21: 4 x 3 blocks
    header = 256                            # 5 offsets, rounded up to 256 bytes
    want = (header + blocks * 64 * 3 + 255) // 256 * 256
    assert b.workspace_bytes == want
    L = N.lib()
    assert L.ctl_jpeg_decode_workspace_bytes(None, 3) == 0
    assert L.ctl_jpeg_decode_workspace_bytes(b.entries.data_ptr(), 0) == 0


def test_argument_errors_are_reported_without_a_gpu():
    L = N.lib()
    one = C.c_void_p(256)

    def call(src=one, src_bytes=1000, ent=one, n=4, tab=one, out=one, out_bytes=1000, status=one, ws=one,
             ws_bytes=10 ** 6):
        return L.ctl_jpeg_decode(src, src_bytes, ent, n, tab, out, out_bytes, status, ws, ws_bytes, None)

    cases = [
        lambda: call(src=None), lambda: call(ent=None), lambda: call(tab=None), lambda: call(out=None),
        lambda: call(status=None), lambda: call(ws=None), lambda: call(n=0), lambda: call(n=-1),
        lambda: call(n=1 << 31), lambda: call(src_bytes=-1), lambda: call(out_bytes=-1),
        lambda: call(ws_bytes=255), lambda: call(n=40, ws_bytes=256),  # shorter than the offset header
    ]
    for i, c in enumerate(cases):
        rc = c()
        assert rc == -1, (i, rc, L.ctl_last_error())
        assert len(L.ctl_last_error()) > 0
        with pytest.raises(ValueError):
            N.check(rc)
    assert L.ctl_jpeg_parse(None, 10, C.byref(N.JpegDesc()), None, None) == -1
    assert L.ctl_jpeg_parse(b"\xff\xd8", 2, None, None, None) == -1
    assert L.ctl_jpeg_parse(b"\xff\xd8\xff\xd9", -1, C.byref(N.JpegDesc()), None, None) == -1
