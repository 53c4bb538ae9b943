"""Host restatement of the JPEG decode of `ctl_jpeg_decode` -- libjpeg-turbo's default decompression as Pillow runs it
for `Image.open(p).convert("RGB")` -- in Python integers and numpy int64: the checker the CPU tests pin to Pillow and
the GPU tests compare the device against.

parse() mirrors ctl_jpeg_parse (marker segments up to SOS, the same descriptor fields and the same rejections) and
decode() the three device stages: Huffman decode, dequantisation + jpeg_idct_islow with its range_limit table, and
per-component upsampling + ycc_rgb_convert.  `counters` (a dict) counts how often each edge rule fires, so a test can
show that a fixture set reaches every rule.
"""
from __future__ import annotations

import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45,
                   38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])


class Unsupported(ValueError):
    """A file the device decode does not cover (Pillow decodes it on the host instead)."""


class CorruptData(ValueError):
    """Entropy-coded data that ends early or is malformed."""


def _be16(b, i):
    return b[i] << 8 | b[i + 1]


def parse(data: bytes) -> dict:
    """The fields of struct ctl_jpeg_desc, or Unsupported with the reason."""
    b = bytes(data)
    n = len(b)
    if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise Unsupported("not a JPEG: no SOI marker")
    qt, qt16, dht = {}, {}, {}
    sof = None
    jfif, adobe, ri = False, None, 0
    pos = 2
    while True:
        if pos >= n or b[pos] != 0xFF:
            raise Unsupported("truncated or corrupt JPEG header")
        while pos < n and b[pos] == 0xFF:
            pos += 1
        if pos >= n:
            raise Unsupported("truncated JPEG header: no SOS marker")
        m = b[pos]
        pos += 1
        if m == 0x01 or 0xD0 <= m <= 0xD7:
            continue
        if m in (0xD8, 0xD9):
            raise Unsupported("corrupt JPEG header: marker before SOS")
        if pos + 2 > n:
            raise Unsupported("truncated JPEG header")
        ln = _be16(b, pos)
        if ln < 2 or pos + ln > n:
            raise Unsupported("truncated JPEG header: marker segment")
        body, seg = pos + 2, b[pos + 2: pos + ln]
        pos += ln
        if m in (0xC0, 0xC1):
            if seg[0] != 8:
                raise Unsupported(f"{seg[0]}-bit JPEG samples")
            h, w, nc = _be16(seg, 1), _be16(seg, 3), seg[5]
            if h == 0:
                raise Unsupported("JPEG height defined by a DNL marker")
            if nc == 4:
                raise Unsupported("4-component (CMYK / YCCK) JPEG")
            if nc not in (1, 3):
                raise Unsupported(f"{nc}-component JPEG")
            comps = [(seg[6 + 3 * c], seg[7 + 3 * c] >> 4, seg[7 + 3 * c] & 15, seg[8 + 3 * c]) for c in range(nc)]
            sof = (h, w, comps)
        elif m in (0xC2, 0xC6, 0xCA, 0xCE):
            raise Unsupported(f"progressive JPEG (SOF{m - 0xC0})")
        elif m in (0xC3, 0xC7, 0xCB, 0xCF):
            raise Unsupported(f"lossless JPEG (SOF{m - 0xC0})")
        elif m == 0xC5:
            raise Unsupported("hierarchical JPEG (SOF5)")
        elif m in (0xC9, 0xCD, 0xCC):
            raise Unsupported("arithmetic-coded JPEG")
        elif m == 0xDB:
            i = 0
            while i < len(seg):
                pq, t = seg[i] >> 4, seg[i] & 15
                qt[t], qt16[t] = body + i + 1, pq
                i += 1 + (128 if pq else 64)
        elif m == 0xC4:
            i = 0
            while i < len(seg):
                tc, th = seg[i] >> 4, seg[i] & 15
                dht[tc, th] = body + i + 1
                i += 17 + sum(seg[i + 1: i + 17])
        elif m == 0xDD:
            ri = _be16(seg, 0)
        elif m == 0xE0 and seg[:5] == b"JFIF\0":
            jfif = True
        elif m == 0xEE and seg[:5] == b"Adobe" and len(seg) >= 12:
            adobe = seg[11]
        elif m == 0xDA:
            h, w, comps = sof
            nc = len(comps)
            ns = seg[0]
            if ns != nc:
                raise Unsupported("multi-scan sequential JPEG")
            if nc == 3:
                if not jfif and adobe == 0:
                    raise Unsupported("Adobe RGB JPEG (transform 0)")
                if not jfif and adobe is None and [c[0] for c in comps] == [82, 71, 66]:
                    raise Unsupported("RGB JPEG (component ids R, G, B)")
            d = dict(h=h, w=w, ncomp=nc, restart_interval=ri, scan_begin=pos, scan_end=n, dqt=[0] * 3,
                     dht_dc=[0] * 3, dht_ac=[0] * 3, dqt16=0, hs=[0] * 3, vs=[0] * 3)
            for c, (cid, hs, vs, tq) in enumerate(comps):
                td, ta = seg[2 + 2 * c] >> 4, seg[2 + 2 * c] & 15
                d["dqt"][c], d["dht_dc"][c], d["dht_ac"][c] = qt[tq], dht[0, td], dht[1, ta]
                d["dqt16"] |= qt16[tq] << c
                d["hs"][c], d["vs"][c] = (1, 1) if nc == 1 else (hs, vs)
            return d


def _huff_lut(b, off):
    """16-bit lookahead table: (code length << 8) | symbol, 0 where no code starts."""
    counts = b[off: off + 16]
    vals = b[off + 16: off + 16 + sum(counts)]
    lut = np.zeros(1 << 16, dtype=np.int64)
    code = k = 0
    for ln in range(1, 17):
        for _ in range(counts[ln - 1]):
            lut[code << (16 - ln): (code + 1) << (16 - ln)] = ln << 8 | vals[k]
            code += 1
            k += 1
        code <<= 1
    return lut.tolist()


def _segments(b, begin, end):
    """The entropy-coded bytes after SOS, unstuffed, split at RSTn markers -> [(rst number or None, bytes)]."""
    segs, cur, tag = [], bytearray(), None
    i = begin
    while i < end:
        j = b.find(b"\xff", i, end)
        if j < 0:
            cur += b[i:end]
            break
        cur += b[i:j]
        k = j + 1
        while k < end and b[k] == 0xFF:
            k += 1
        if k >= end:
            break
        if b[k] == 0x00 and k == j + 1:
            cur.append(0xFF)
            i = k + 1
        elif 0xD0 <= b[k] <= 0xD7:
            segs.append((tag, bytes(cur)))
            cur, tag = bytearray(), b[k] - 0xD0
            i = k + 1
        else:
            break  # EOI or another marker: the end of the scan
    segs.append((tag, bytes(cur)))
    return segs


def _windows(seg):
    """Bit windows of a segment: w[i] = the 16 bits starting at bit i (zeros past the end), and the bit count."""
    bits = np.unpackbits(np.frombuffer(seg, dtype=np.uint8)).astype(np.int64)
    nb = bits.size
    pad = 64 * 32 + 64  # one block's worth of bits read past the end before the check after it
    bits = np.concatenate([bits, np.zeros(pad + 16, dtype=np.int64)])
    w = np.zeros(nb + pad, dtype=np.int64)
    for k in range(16):
        w += bits[k: k + nb + pad] << (15 - k)
    return w.tolist(), nb


def geometry(d):
    nc = d["ncomp"]
    hs, vs = d["hs"][:nc], d["vs"][:nc]
    maxh, maxv = max(hs), max(vs)
    mcux, mcuy = -(-d["w"] // (8 * maxh)), -(-d["h"] // (8 * maxv))
    comps = []
    for c in range(nc):
        comps.append(dict(hs=hs[c], vs=vs[c], bw=mcux * hs[c], bh=mcuy * vs[c], dw=-(-d["w"] * hs[c] // maxh),
                          dh=-(-d["h"] * vs[c] // maxv), fh=maxh // hs[c], fv=maxv // vs[c]))
    return dict(maxh=maxh, maxv=maxv, mcux=mcux, mcuy=mcuy, comps=comps)


def entropy_decode(b, d, g):
    """-> per component int64 coefficients [bh, bw, 64] in natural order."""
    nc = d["ncomp"]
    coef = [np.zeros((c["bh"], c["bw"], 64), dtype=np.int64) for c in g["comps"]]
    dc = [_huff_lut(b, d["dht_dc"][c]) for c in range(nc)]
    ac = [_huff_lut(b, d["dht_ac"][c]) for c in range(nc)]
    segs = _segments(b, d["scan_begin"], d["scan_end"])
    ri = d["restart_interval"]
    mcus = g["mcux"] * g["mcuy"]
    per_seg = ri if ri else mcus
    need = -(-mcus // per_seg)
    if len(segs) < need:
        raise CorruptData("missing restart marker")
    zz = ZIGZAG.tolist()
    m = 0
    for s in range(need):
        tag, seg = segs[s]
        if s and tag != (s - 1) % 8:
            raise CorruptData("restart marker out of sequence")
        win, nb = _windows(seg)
        pos = 0
        pred = [0] * nc
        for _ in range(min(per_seg, mcus - m)):
            my, mx = divmod(m, g["mcux"])
            for c in range(nc):
                cc = g["comps"][c]
                dct, act = dc[c], ac[c]
                for v in range(cc["vs"]):
                    for h in range(cc["hs"]):
                        blk = coef[c][my * cc["vs"] + v, mx * cc["hs"] + h]
                        e = dct[win[pos]]
                        if not e:
                            raise CorruptData("bad Huffman code")
                        pos += e >> 8
                        t = e & 0xFF
                        if t > 15:
                            raise CorruptData("DC magnitude > 15")
                        diff = 0
                        if t:
                            r = win[pos] >> (16 - t)
                            pos += t
                            diff = r if r >= 1 << (t - 1) else r - (1 << t) + 1
                        pred[c] += diff
                        blk[0] = ((pred[c] + 32768) & 0xFFFF) - 32768  # stored as JCOEF (int16)
                        k = 1
                        while k < 64:
                            e = act[win[pos]]
                            if not e:
                                raise CorruptData("bad Huffman code")
                            pos += e >> 8
                            rs = e & 0xFF
                            r, sz = rs >> 4, rs & 15
                            if sz:
                                k += r
                                if k > 63:
                                    raise CorruptData("coefficient index > 63")
                                val = win[pos] >> (16 - sz)
                                pos += sz
                                blk[zz[k]] = val if val >= 1 << (sz - 1) else val - (1 << sz) + 1
                            elif r != 15:
                                break
                            else:
                                k += 15
                            k += 1
                        if pos > nb:
                            raise CorruptData("entropy-coded data ends before the last MCU")
            m += 1
    return coef


FIX = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137,
           f1961=16069, f2053=16819, f2562=20995, f3072=25172)


def _islow_1d(d):
    """jidctint.c's butterfly along the last axis of int64 d [..., 8] -> the 8 outputs before descaling."""
    F = FIX
    z2, z3 = d[..., 2], d[..., 6]
    z1 = (z2 + z3) * F["f0541"]
    tmp2 = z1 + z3 * -F["f1847"]
    tmp3 = z1 + z2 * F["f0765"]
    tmp0 = (d[..., 0] + d[..., 4]) << 13
    tmp1 = (d[..., 0] - d[..., 4]) << 13
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = d[..., 7], d[..., 5], d[..., 3], d[..., 1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * F["f1175"]
    t0, t1, t2, t3 = t0 * F["f0298"], t1 * F["f2053"], t2 * F["f3072"], t3 * F["f1501"]
    z1, z2, z3, z4 = z1 * -F["f0899"], z2 * -F["f2562"], z3 * -F["f1961"] + z5, z4 * -F["f0390"] + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    return np.stack([tmp10 + t3, tmp11 + t2, tmp12 + t1, tmp13 + t0, tmp13 - t0, tmp12 - t1, tmp11 - t2, tmp10 - t3],
                    axis=-1)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def range_limit(v):
    """The post-IDCT limit of v = sample - 128 as Pillow applies it: a saturating clamp.  libjpeg-turbo's SIMD IDCTs
    (what Pillow runs) pack with saturation; its C path's range_limit[v & 1023] agrees on [-384, 512) and wraps
    outside it, a band only crafted files reach (counted as "idct_wrap")."""
    return np.clip(v + 128, 0, 255)


def quant_table(b, d, c):
    off = d["dqt"][c]
    if d["dqt16"] >> c & 1:
        q = np.frombuffer(b[off: off + 128], dtype=">u2").astype(np.int64)
    else:
        q = np.frombuffer(b[off: off + 64], dtype=np.uint8).astype(np.int64)
    nat = np.zeros(64, dtype=np.int64)
    nat[ZIGZAG] = q
    return ((nat + 32768) & 0xFFFF) - 32768  # ISLOW_MULT_TYPE is short


def idct_plane(coef, q, counters=None):
    """int64 coefficients [bh, bw, 64] -> the uint8 component plane [bh * 8, bw * 8]."""
    bh, bw, _ = coef.shape
    d = (coef * q).reshape(bh, bw, 8, 8)                       # [.., row (vertical frequency), col]
    p1 = _descale(_islow_1d(np.swapaxes(d, -1, -2)), 11)      # per column: [.., col, row]
    p1 = ((p1 + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)           # the int workspace
    p2 = _descale(_islow_1d(np.swapaxes(p1, -1, -2)), 18)     # per row: [.., row, x]
    if counters is not None:
        counters["idct_wrap"] = counters.get("idct_wrap", 0) + int(((p2 < -384) | (p2 >= 512)).sum())
    out = range_limit(p2).astype(np.uint8)
    return out.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)


def upsample(plane, cc, h, w, counters=None):
    """Component plane -> [h, w] int64 at the output resolution (jdsample.c's method for the component's ratio)."""
    fh, fv, dw, dh = cc["fh"], cc["fv"], cc["dw"], cc["dh"]
    p = plane.astype(np.int64)
    y, x = np.arange(h), np.arange(w)
    cnt = counters if counters is not None else {}

    def bump(k, v):
        cnt[k] = cnt.get(k, 0) + int(v)

    if fh == 1 and fv == 1:
        return p[:h, :w]
    if fh in (2,) and fv in (1, 2) and dw <= 2:
        bump("narrow_fallback", 1)
    if fh == 2 and fv == 1 and dw > 2:
        i = x >> 1
        j = np.where(x & 1, np.minimum(i + 1, dw - 1), np.maximum(i - 1, 0))
        bump("edge_right", (dw % 8 != 0) and bool(((x & 1) & (i + 1 > dw - 1)).any()))
        rows = p[:h]
        return np.where(x & 1, (3 * rows[:, i] + rows[:, j] + 2) >> 2, (3 * rows[:, i] + rows[:, j] + 1) >> 2)
    if fh == 1 and fv == 2:
        r0 = y >> 1
        r1 = np.where(y & 1, np.minimum(r0 + 1, dh - 1), np.maximum(r0 - 1, 0))
        bump("edge_bottom", (dh % 8 != 0) and bool(((y & 1) & (r0 + 1 > dh - 1)).any()))
        return (3 * p[r0][:, :w] + p[r1][:, :w] + np.where(y & 1, 2, 1)[:, None]) >> 2
    if fh == 2 and fv == 2 and dw > 2:
        r0 = y >> 1
        r1 = np.where(y & 1, np.minimum(r0 + 1, dh - 1), np.maximum(r0 - 1, 0))
        bump("edge_bottom", (dh % 8 != 0) and bool(((y & 1) & (r0 + 1 > dh - 1)).any()))
        bump("edge_right", (dw % 8 != 0) and bool(((x & 1) & ((x >> 1) + 1 > dw - 1)).any()))
        cs = 3 * p[r0] + p[r1]                                   # column sums [h, bw * 8]
        i = x >> 1
        j = np.where(x & 1, np.minimum(i + 1, dw - 1), np.maximum(i - 1, 0))
        return np.where(x & 1, (3 * cs[:, i] + cs[:, j] + 7) >> 4, (3 * cs[:, i] + cs[:, j] + 8) >> 4)
    return p[(y // fv)][:, x // fh]


def decode(data: bytes, counters=None) -> np.ndarray:
    """-> uint8 [h, w, 3] == np.asarray(Image.open(BytesIO(data)).convert("RGB")).  Raises Unsupported or CorruptData."""
    b = bytes(data)
    d = parse(b)
    g = geometry(d)
    coef = entropy_decode(b, d, g)
    h, w = d["h"], d["w"]
    comps = [upsample(idct_plane(coef[c], quant_table(b, d, c), counters), g["comps"][c], h, w, counters)
             for c in range(d["ncomp"])]
    if d["ncomp"] == 1:
        return np.repeat(comps[0].astype(np.uint8)[:, :, None], 3, axis=2)
    yy, cb, cr = comps[0], comps[1] - 128, comps[2] - 128
    r = yy + ((91881 * cr + 32768) >> 16)
    gg = yy + ((-46802 * cr - 22554 * cb + 32768) >> 16)
    bb = yy + ((116130 * cb + 32768) >> 16)
    return np.clip(np.stack([r, gg, bb], axis=-1), 0, 255).astype(np.uint8)
