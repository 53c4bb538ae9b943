"""Host restatement of how `jpeg_entropy_kernel` (csrc/jpeg.cu) splits one image's entropy-coded data into
subsequences and decodes them in parallel, on top of tests/jpeg_oracle.py: the marker scan and restart-segment table,
the subsequence length rule, the speculative exits, the sync rounds to convergence, the per-subsequence block counts
and DC sums with their segmented scans, and the write pass with the serial reader's error rules.

Positions are bits in scan coordinates: the bytes after SOS with the stuffed 0x00 of every 0xFF 0x00 pair left out
(marker bytes count).  A decode state is (position, block u of the MCU, coefficient index k) plus the restart
segment j the position lies in.  `decode(data)` returns the model's result: the converged entries, the round count,
the coefficients it writes and whether the serial decode fails.
"""
from __future__ import annotations

import numpy as np

import jpeg_oracle as JO

T = 256            # threads per image: at most this many subsequences
S_MIN = 1024       # shortest subsequence, bits
TERMINAL = 1 << 62  # the state past the last restart segment


def sub_bits(bits):
    """The subsequence length S of an image whose segments end at scan bit `bits`, and the subsequence count."""
    s = (max(S_MIN, -(-bits // T)) + 31) & ~31
    return s, max(1, -(-bits // s))


def stuffed(b, i, begin):
    return i > begin and b[i] == 0 and b[i - 1] == 0xFF


def is_marker(b, i, begin, end):
    return b[i] == 0xFF and (i + 1 == end or b[i + 1] != 0) and (i == begin or b[i - 1] != 0xFF)


def segment_table(b, d, needed):
    """[(s_off, s_u, q_off, q_u, rst)] for the restart segments the data has (at most `needed`): start (file offset,
    scan byte), data end at the next marker run (file offset, scan byte) and the RSTn number after it (-1: another
    marker or the end of the data).  Also the scan byte of every file offset in the scan (for the reader's pointer)."""
    begin, end = d["scan_begin"], d["scan_end"]
    ri = d["restart_interval"]
    segs = [[begin, 0, None, None, -1]]
    u = 0
    ubyte = {}
    for i in range(begin, end):
        if stuffed(b, i, begin):
            continue
        ubyte[u] = i
        if is_marker(b, i, begin, end) and segs[-1][2] is None:
            r = i
            while r < end and b[r] == 0xFF:
                r += 1
            rst = b[r] - 0xD0 if ri and r < end and 0xD0 <= b[r] <= 0xD7 else -1
            segs[-1][2:] = [i, u, rst]
            if rst < 0 or len(segs) == needed:
                break
            segs.append([r + 1, u + (r + 1 - i), None, None, -1])
        u += 1
    if segs[-1][2] is None:
        n = sum(1 for i in range(begin, end) if not stuffed(b, i, begin))
        segs[-1][2:] = [end, n, -1]
        ubyte[n] = end
    return [tuple(s) for s in segs], ubyte


class Image:
    """One JPEG's decode context: tables, geometry, restart segments and their bit windows."""

    def __init__(self, data: bytes):
        b = self.b = bytes(data)
        d = self.d = JO.parse(b)
        g = self.g = JO.geometry(d)
        nc = d["ncomp"]
        self.comp, self.vrow, self.hcol = [], [], []
        for c, cc in enumerate(g["comps"]):
            for v in range(cc["vs"]):
                for h in range(cc["hs"]):
                    self.comp.append(c)
                    self.vrow.append(v)
                    self.hcol.append(h)
        self.bpm = len(self.comp)
        mcus = g["mcux"] * g["mcuy"]
        self.total = mcus * self.bpm
        self.ri = d["restart_interval"]
        self.needed = -(-mcus // self.ri) if self.ri else 1
        self.dc = [JO._huff_lut(b, d["dht_dc"][c]) for c in range(nc)]
        self.ac = [JO._huff_lut(b, d["dht_ac"][c]) for c in range(nc)]
        self.segs, self.ubyte = segment_table(b, d, self.needed)
        self.nseg = len(self.segs)
        self.win = []
        for s_off, s_u, q_off, q_u, _ in self.segs:
            seg = bytes(b[i] for i in range(s_off, q_off) if not stuffed(b, i, d["scan_begin"]))
            assert len(seg) == q_u - s_u
            self.win.append(JO._windows(seg)[0])
        self.bits = 8 * self.segs[-1][3]
        self.S, self.nsub = sub_bits(self.bits)

    def base(self, j):
        return j * self.ri * self.bpm if self.ri else 0

    def quota(self, j):
        return min(self.ri * self.bpm, self.total - self.base(j)) if self.ri else self.total

    def seg_end(self, j):
        return 8 * self.segs[j][3]

    def seg_of(self, p):
        j = 0
        while j + 1 < self.nseg and 8 * self.segs[j + 1][1] <= p:
            j += 1
        return j

    def window(self, j, p):
        return self.win[j][p - 8 * self.segs[j][1]]

    def step(self, j, p, u, k):
        """One symbol at p -> (new p, u, k, dc difference or None, coefficient (index, value) or None,
        'ok' | 'invalid' | 'range')."""
        c = self.comp[u]
        w = self.window(j, p)
        e = (self.ac[c] if k else self.dc[c])[w]
        if not e:
            return p, u, k, None, None, "invalid"
        ln, sym = e >> 8, e & 0xFF
        if k == 0:
            if sym > 15:
                return p, u, k, None, None, "range"
            p += ln
            diff = 0
            if sym:
                r = self.window(j, p) >> (16 - sym)
                p += sym
                diff = r if r >= 1 << (sym - 1) else r - (1 << sym) + 1
            return p, u, 1, diff, None, "ok"
        r, sz = sym >> 4, sym & 15
        if sz:
            if k + r > 63:
                return p, u, k, None, None, "range"
            p += ln
            val = self.window(j, p) >> (16 - sz)
            p += sz
            val = val if val >= 1 << (sz - 1) else val - (1 << sz) + 1
            return p, u, k + r + 1, None, (k + r, val), "ok"
        return p + ln, u, (k + 16 if r == 15 else 64), None, None, "ok"

    def walk(self, state, stop):
        """jd_walk: the speculative / sync decode from `state` = (p, j, u, k) until a step would start at or past
        `stop` -> (exit state, record (f, blocks, dc sums))."""
        p, j, u, k = state
        f, blocks, dcs = 0, 0, [0, 0, 0]
        if j >= self.nseg or p >= stop:
            return state, (f, blocks, dcs)
        while True:
            if p >= self.seg_end(j):
                f, blocks, dcs = 1, 0, [0, 0, 0]
                j += 1
                if j >= self.nseg:
                    return (TERMINAL, self.nseg, 0, 0), (f, blocks, dcs)
                blocks = self.base(j)
                p, u, k = 8 * self.segs[j][1], 0, 0
                continue
            if p >= stop:
                return (p, j, u, k), (f, blocks, dcs)
            c = self.comp[u]
            p2, u2, k2, diff, _, how = self.step(j, p, u, k)
            if how != "ok":
                p, u, k = p + 1, 0, 0
                continue
            p, u, k = p2, u2, k2
            if diff is not None:
                dcs[c] = (dcs[c] + diff) & 0xFFFFFFFF
            if k >= 64:
                k, u = 0, (u + 1) % self.bpm
                blocks += 1

    def reader_p(self, j, fill_at):
        """File offset of the serial reader's next byte after a fill at scan bit `fill_at` in segment j: it holds at
        least 57 bits past the consumed ones, or stopped at the marker."""
        return self.ubyte[min((fill_at + 57 + 7) // 8, self.segs[j][3])]

    def restart_ok(self, j, p_off):
        s_off, s_u, q_off, q_u, rst = self.segs[j]
        return rst == (j & 7) and all(self.b[i] != 0xFF for i in range(p_off, q_off))

    def write(self, state, stop, sb, pred, coef):
        """jd_write: the true path from `state` with block index sb and DC predictors pred -> True on an error."""
        p, j, u, k = state
        if j >= self.nseg or p >= stop:
            return False
        base, quota = self.base(j), self.quota(j)
        completed, fill_at = False, None
        pred = list(pred)
        g = self.g
        while True:
            done = sb - base >= quota
            if done or p >= self.seg_end(j):
                if not done:
                    return True
                if j + 1 >= self.needed:
                    return False
                if completed and not self.restart_ok(j, self.reader_p(j, fill_at)):
                    return True
                j += 1
                if j >= self.nseg:
                    return False
                base = sb = self.base(j)
                quota = self.quota(j)
                pred = [0, 0, 0]
                p, u, k = 8 * self.segs[j][1], 0, 0
                completed = False
                continue
            if p >= stop:
                return False
            completed = False
            c = self.comp[u]
            cc = g["comps"][c]
            m = sb // self.bpm
            my, mx = divmod(m, g["mcux"])
            blk = coef[c][my * cc["vs"] + self.vrow[u], mx * cc["hs"] + self.hcol[u]]
            fill_at = p
            p, u, k2, diff, val, how = self.step(j, p, u, k)
            if how != "ok":
                return True
            if diff is not None:
                pred[c] = (pred[c] + diff) & 0xFFFFFFFF
                blk[0] = ((pred[c] + 32768) & 0xFFFF) - 32768
            if val is not None:
                blk[JO.ZIGZAG[val[0]]] = val[1]
            k = k2
            if p > self.seg_end(j):
                return True
            if k >= 64:
                k, u = 0, (u + 1) % self.bpm
                sb += 1
                completed = True


def _combine(a, b):
    if b[0]:
        return b
    return (a[0], (a[1] + b[1]) & 0xFFFFFFFF, [(x + y) & 0xFFFFFFFF for x, y in zip(a[2], b[2])])


def decode(data: bytes) -> dict:
    """The kernel's decode of one file: S, nsub, the converged entry of every subsequence, the sync rounds it took
    (round 0 is the speculative pass), each subsequence's record and entry counts, the coefficients and the error."""
    im = Image(data)
    S, nsub = im.S, im.nsub
    stops = [(i + 1) * S if i + 1 < nsub else TERMINAL for i in range(nsub)]
    entries = [(i * S, im.seg_of(i * S), 0, 0) for i in range(nsub)]
    exits, recs = [None] * nsub, [None] * nsub
    for i in range(nsub):
        exits[i], recs[i] = im.walk(entries[i], stops[i])
    rounds = 0
    while True:
        incoming = [entries[0]] + exits[:-1]
        redo = [i for i in range(1, nsub) if incoming[i][0::2] + incoming[i][3:] != entries[i][0::2] + entries[i][3:]]
        if not redo:
            break
        rounds += 1
        for i in redo:
            entries[i] = incoming[i]
            exits[i], recs[i] = im.walk(entries[i], stops[i])
    prefix, acc = [], (0, 0, [0, 0, 0])
    for r in recs:
        prefix.append(acc)
        acc = _combine(acc, r)
    nc = im.d["ncomp"]
    coef = [np.zeros((c["bh"], c["bw"], 64), dtype=np.int64) for c in im.g["comps"]]
    err = False
    for i in range(nsub):
        _, sb, dcs = prefix[i]
        pred = [x - (1 << 32) if x >= 1 << 31 else x for x in dcs]
        err |= im.write(entries[i], stops[i], sb, pred, coef)
    return dict(image=im, S=S, nsub=nsub, entries=entries, exits=exits, rounds=rounds, recs=recs, prefix=prefix,
                coef=coef[:nc], err=err)


def serial_states(im: Image):
    """The true path under the same step rules from the exact start, with no subsequence stops: for every boundary
    i * S (i >= 1) the state at the first step that would start at or past it -- what the exit of subsequence i - 1
    must converge to."""
    out = []
    state = (0, 0, 0, 0)
    for i in range(1, im.nsub):
        state, _ = im.walk(state, i * im.S)
        out.append(state)
    return out
