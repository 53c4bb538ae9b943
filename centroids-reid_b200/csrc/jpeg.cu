// `Image.open(p).convert("RGB")` of the reference's loaders (datasets/bases.py:32-33, inference/inference_utils.py:33-34)
// on the device for the JPEGs its datasets contain: baseline / extended-sequential Huffman, 8-bit samples, one
// interleaved scan, grayscale or YCbCr.  Pillow decodes with libjpeg-turbo's defaults, whose arithmetic is fixed
// integer code, so this decode is bit for bit Pillow's:
//   * Huffman decode (byte stuffing, RSTn resync and DC-predictor resets) into int16 coefficients, dezigzagged;
//   * dequantisation in `short` (ISLOW_MULT_TYPE of a SIMD build: a 16-bit table value above 32767 wraps) and
//     jpeg_idct_islow (jidctint.c: CONST_BITS 13, PASS1_BITS 2, 64-bit products, an int workspace), whose output
//     x = sample - 128 is clamped to 0..255 after + 128.  That is what Pillow gives: libjpeg-turbo's SIMD IDCTs pack
//     with saturation.  Its C path's range_limit[x & 1023] (jdmaster.c prepare_range_limit_table) agrees on
//     [-384, 512) and wraps outside it, a band that encoder output does not reach (only crafted tables do);
//   * upsampling per component (jdsample.c): h2v1 and h2v2 "fancy" triangle filters when the component's downsampled
//     width is > 2 (else replication), h1v2 fancy always, replication for every other integral ratio; neighbours
//     are clamped at the component's real (not MCU-padded) width and height, and the rounding alternates
//     +1/+2 (h2v1, h1v2) and +8/+7 (h2v2);
//   * ycc_rgb_convert (jdcolor.c): SCALEBITS 16 tables with ONE_HALF rounding, then a clamp; grayscale writes
//     R = G = B = Y as convert("RGB") of an "L" image does.
// Three launches, one image per CTA row: entropy decode (one CTA per image, its Huffman tables built in shared memory
// from the file's own DHT bytes, its entropy-coded data split into up to 256 subsequences decoded in parallel and
// brought into step by sync rounds), IDCT (eight threads per 8x8 block), upsample + colour convert (one thread per
// output pixel).  The host parser below (ctl_jpeg_parse) reads the marker segments up to SOS; it is the
// only code that knows the JPEG file format, and it never reads the entropy-coded data.
#include <stdint.h>
#include <string.h>

#include <algorithm>

#include "common.h"
#include "wgmma.cuh"  // pdl_wait, pdl_launch_dependents

namespace ctl {

constexpr int JD_HEADER_ALIGN = 256;
constexpr int JD_IDCT_THREADS = 128;  // 16 blocks of 8 threads
constexpr int JD_COLOR_THREADS = 256;
constexpr int JD_MAX_SIDE = 65535;

// status bits of an entry
constexpr int JS_DATA = 1;       // entropy-coded data ends before the last MCU or is malformed
constexpr int JS_ENTRY = 2;      // entry outside the source buffer, or a descriptor the parser cannot have written
constexpr int JS_OUTPUT = 4;     // output entry of another size, or outside the output buffer
constexpr int JS_WORKSPACE = 8;  // the image's coefficients and planes do not fit in the workspace

// Geometry of a JPEG entry: MCU grid, and per component its block grid (MCU-padded) and real downsampled size.
struct JGeom {
  int nc, maxh, maxv, mcux, mcuy;
  int hs[3], vs[3], bw[3], bh[3], dw[3], dh[3];
  long long blocks;  // sum of bw * bh
};

// false for a descriptor ctl_jpeg_parse cannot have written
__host__ __device__ inline bool jpeg_geom(const ctl_jpeg_desc& d, JGeom& g) {
  if (d.ncomp != 1 && d.ncomp != 3) return false;
  if (d.h < 1 || d.w < 1 || d.h > JD_MAX_SIDE || d.w > JD_MAX_SIDE) return false;
  g.nc = d.ncomp;
  g.maxh = g.maxv = 1;
  int per_mcu = 0;
  for (int c = 0; c < g.nc; ++c) {
    g.hs[c] = g.nc == 1 ? 1 : d.hs[c];
    g.vs[c] = g.nc == 1 ? 1 : d.vs[c];
    if (g.hs[c] < 1 || g.hs[c] > 4 || g.vs[c] < 1 || g.vs[c] > 4) return false;
    g.maxh = g.hs[c] > g.maxh ? g.hs[c] : g.maxh;
    g.maxv = g.vs[c] > g.maxv ? g.vs[c] : g.maxv;
    per_mcu += g.hs[c] * g.vs[c];
  }
  if (per_mcu > 10) return false;  // libjpeg's D_MAX_BLOCKS_IN_MCU
  g.mcux = (d.w + 8 * g.maxh - 1) / (8 * g.maxh);
  g.mcuy = (d.h + 8 * g.maxv - 1) / (8 * g.maxv);
  g.blocks = 0;
  for (int c = 0; c < g.nc; ++c) {
    if (g.maxh % g.hs[c] || g.maxv % g.vs[c]) return false;  // integral upsampling only
    g.bw[c] = g.mcux * g.hs[c];
    g.bh[c] = g.mcuy * g.vs[c];
    g.dw[c] = (int)(((long long)d.w * g.hs[c] + g.maxh - 1) / g.maxh);
    g.dh[c] = (int)(((long long)d.h * g.vs[c] + g.maxv - 1) / g.maxv);
    g.blocks += (long long)g.bw[c] * g.bh[c];
  }
  return true;
}

// workspace bytes of one entry: int16 coefficients, then uint8 component planes, 16-byte aligned; 0 unless a JPEG
__host__ __device__ inline long long jpeg_region_bytes(const ctl_jpeg_entry& e) {
  JGeom g;
  if (e.kind != CTL_JPEG_ENTRY_JPEG || !jpeg_geom(e.desc, g)) return 0;
  return g.blocks * 64 * 3;  // a multiple of 64
}

__host__ __device__ inline size_t jpeg_header_bytes(long long n) {
  return ((size_t)n * sizeof(long long) + JD_HEADER_ALIGN - 1) & ~size_t(JD_HEADER_ALIGN - 1);
}

// ---------------------------------------------------------------------------------------------------------------
// entropy decode
//
// One CTA of JD_ENTROPY_THREADS threads per image, each thread one subsequence of the entropy-coded data.
// Positions are bit offsets in scan coordinates: the bytes after SOS with the stuffed 0x00 of every 0xFF 0x00 pair left
// out (marker bytes count), so a restart segment (the data between SOS or an RSTn and the next marker) is one
// contiguous range.  The image's S-bit subsequences partition them; S = max(JD_SUB_MIN_BITS, ceil(bits / T)) rounded
// to a word, so an image never has more than T subsequences.  The decode state at a position is (block u of the MCU,
// coefficient index k); restart-segment starts are exact states (0, 0).
//   1. marker scan: each thread scans T-th of the bytes for stuffing zeros and marker runs; CTA-wide scans of the
//      counts give each chunk's scan coordinate and each marker its index, and the restart-segment table (start,
//      data end, the RST number that follows) is written to the image's plane region, which the IDCT fills later.
//   2. speculative pass: thread i decodes from the start of subsequence i as if a block began there (an invalid code
//      resumes at the next bit with state (0, 0)) until it crosses into subsequence i + 1, and records that exit.
//   3. sync rounds: every thread whose predecessor's exit changed decodes again from it, until no exit changes.  The
//      decoder self-synchronises, so this takes a few rounds; round r has the first r subsequences exact, so the
//      loop ends after at most T rounds.
//   4. counts: from the converged decodes, CTA-wide segmented scans of the blocks each subsequence completes and of
//      its DC differences (32-bit wrapping sums, the low 16 bits of the serial predictors) give every subsequence its
//      first block and DC predictors; they restart at every restart segment.
//   5. write pass: each thread decodes its part of the true path again and stores the dezigzagged coefficients.
// Errors count on the true path only, before the image's last block, and are the serial reader's: an invalid code, a
// DC magnitude > 15, a coefficient index > 63, bits consumed past a marker or the end of the data (zeros are read
// there), an RSTn missing or out of sequence after an interval (the bytes the reader had not loaded before it may be
// padding without 0xFF, and 0xFF fill bytes may precede the marker).

constexpr int JD_ENTROPY_THREADS = 256;
constexpr long long JD_SUB_MIN_BITS = 1024;
constexpr long long JD_TERMINAL = 1LL << 62;  // the state past the last restart segment

struct HuffTable {
  uint16_t lut[512];  // 9-bit lookahead: (code length << 8) | symbol, 0 for a longer code
  int32_t maxcode[17];
  int32_t valoff[17];
  uint8_t val[256];
};

// restart segment j: starts at file byte s_off (scan coordinate s_u bytes), its data ends at the marker at q_off
// (q_u), which is RSTn with n = rst, or rst = -1 (another marker, or the end of the data)
struct JSeg {
  uint32_t s_off, s_u, q_off, q_u;
  int32_t rst;
};

struct BitReader {
  const uint8_t* p;  // next byte to load
  const uint8_t* end;
  uint64_t buf;      // next bits, MSB first
  int n;             // valid bits in buf
  bool marker;       // stopped at a marker: zeros from here on
  long long pos;     // scan-coordinate bit of the next unconsumed bit
  long long pu;      // scan-coordinate byte of p

  __device__ __forceinline__ void init(const uint8_t* at, const uint8_t* e, long long ubyte) {
    p = at;
    end = e;
    buf = 0;
    n = 0;
    marker = false;
    pos = ubyte * 8;
    pu = ubyte;
  }
  __device__ __forceinline__ void fill() {
    while (n <= 56) {
      uint32_t b = 0;
      if (!marker && p < end) {
        b = *p;
        if (b == 0xFF) {
          if (p + 1 < end && p[1] == 0x00) {
            p += 2;
            ++pu;
          } else {
            marker = true;  // a marker (or the end of the data) inside a stuffed pair: zeros from here on
            b = 0;
          }
        } else {
          ++p;
          ++pu;
        }
      }
      buf |= (uint64_t)b << (56 - n);
      n += 8;
    }
  }
  __device__ __forceinline__ uint32_t peek(int k) const { return (uint32_t)(buf >> (64 - k)); }
  __device__ __forceinline__ void consume(int k) {
    buf <<= k;
    n -= k;
    pos += k;
  }
  // the symbol of the code at the head of the buffer and its length (0: no code of up to 16 bits); consumes nothing
  __device__ __forceinline__ int lookup(const HuffTable& t, int& len) const {
    const uint32_t e = t.lut[peek(9)];
    if (e) {
      len = e >> 8;
      return e & 0xFF;
    }
    const uint32_t code = peek(16);
    for (int l = 10; l <= 16; ++l) {
      const int c = (int)(code >> (16 - l));
      if (c <= t.maxcode[l]) {
        len = l;
        return t.val[(t.valoff[l] + c) & 0xFF];
      }
    }
    len = 0;
    return 0;
  }
  __device__ __forceinline__ int receive_extend(int s) {
    if (s == 0) return 0;
    const int v = (int)peek(s);
    consume(s);
    return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v;
  }
  // file offset of the byte holding scan byte x <= pu (x within the data loaded so far): back from p over whole bytes
  __device__ __forceinline__ uint32_t locate(long long x, const uint8_t* file, const uint8_t* scan) const {
    const uint8_t* q = p;
    for (long long u = pu; u > x; --u) q -= (q - 2 >= scan && q[-1] == 0x00 && q[-2] == 0xFF) ? 2 : 1;
    return (uint32_t)(q - file);
  }
};

__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// false for a table whose symbols fall outside the file or whose code lengths overflow the code space; called by
// warp 0
__device__ bool build_huff(const uint8_t* file, long long nbytes, uint32_t off, HuffTable& t) {
  const int lane = threadIdx.x;
  __shared__ int ok_s;
  if (lane == 0) {
    bool ok = (long long)off + 16 <= nbytes;
    int code = 0, k = 0;
    t.maxcode[0] = -1;
    for (int l = 1; l <= 16 && ok; ++l) {
      const int cnt = file[off + l - 1];
      t.valoff[l] = k - code;
      t.maxcode[l] = cnt ? code + cnt - 1 : -1;
      k += cnt;
      code += cnt;
      if (code > (1 << l) || k > 256) ok = false;
      code <<= 1;
    }
    ok_s = ok && (long long)off + 16 + k <= nbytes ? k : -1;
  }
  __syncwarp();
  const int k = ok_s;
  __syncwarp();
  if (k < 0) return false;
  for (int i = lane; i < k; i += 32) t.val[i] = file[off + 16 + i];
  __syncwarp();
  for (int i = lane; i < 512; i += 32) {
    uint16_t e = 0;
    for (int l = 1; l <= 9; ++l) {
      const int c = i >> (9 - l);
      if (c <= t.maxcode[l]) {
        e = (uint16_t)((l << 8) | t.val[(t.valoff[l] + c) & 0xFF]);
        break;
      }
    }
    t.lut[i] = e;
  }
  __syncwarp();
  return true;
}

__device__ __forceinline__ bool in_file(uint32_t off, long long len, long long nbytes) { return (long long)off + len <= nbytes; }

// element of the CTA-wide segmented scans: f marks a restart inside the element (its v then count from it)
struct JAgg {
  int f;
  uint32_t v[4];
};

__device__ __forceinline__ JAgg jagg_combine(const JAgg& a, const JAgg& b) {
  if (b.f) return b;
  JAgg r = a;
#pragma unroll
  for (int q = 0; q < 4; ++q) r.v[q] += b.v[q];
  return r;
}

__device__ __forceinline__ JAgg jagg_shfl_up(const JAgg& a, int o) {
  JAgg r;
  r.f = __shfl_up_sync(0xffffffffu, a.f, o);
#pragma unroll
  for (int q = 0; q < 4; ++q) r.v[q] = __shfl_up_sync(0xffffffffu, a.v[q], o);
  return r;
}

// exclusive segmented scan over the CTA's threads in thread order; `tot` is shared scratch of a warp count
__device__ JAgg jagg_exclusive_scan(JAgg x, JAgg* tot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int nwarps = JD_ENTROPY_THREADS / 32;
  const JAgg zero = {0, {0, 0, 0, 0}};
  JAgg inc = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const JAgg y = jagg_shfl_up(inc, o);
    if (lane >= o) inc = jagg_combine(y, inc);
  }
  if (lane == 31) tot[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    JAgg w = lane < nwarps ? tot[lane] : zero;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const JAgg y = jagg_shfl_up(w, o);
      if (lane >= o) w = jagg_combine(y, w);
    }
    if (lane < nwarps) tot[lane] = w;
  }
  __syncthreads();
  JAgg before = jagg_shfl_up(inc, 1);
  if (lane == 0) before = zero;
  const JAgg r = warp ? jagg_combine(tot[warp - 1], before) : before;
  __syncthreads();  // tot is reused by the next scan
  return r;
}

// what the decoding threads of one image share
struct JCtx {
  const uint8_t* file;
  const uint8_t* scan;  // file + scan_begin
  const uint8_t* end;   // file + scan_end
  const JSeg* seg;      // restart-segment table (in the image's plane region)
  int nseg;             // segments the data has, at most `needed`
  int needed;           // segments the image has: ceil(MCUs / restart interval), 1 without restarts
  int ri, bpm;          // restart interval (MCUs, 0: none), blocks per MCU
  long long total;      // blocks of the image
  const HuffTable* dc;
  const HuffTable* ac;
  const uint8_t* comp;  // component of each block of an MCU
  __device__ __forceinline__ long long base(int j) const { return ri ? (long long)j * ri * bpm : 0; }
  __device__ __forceinline__ long long quota(int j) const {
    return ri ? min((long long)ri * bpm, total - base(j)) : total;
  }
  __device__ __forceinline__ long long seg_end(int j) const { return (long long)seg[j].q_u * 8; }
};

// decode state at a position: segment j, block u of the MCU, coefficient k; off = file offset of the byte of pos
struct JState {
  long long pos;
  uint32_t off;
  int j, u, k;
};

// Speculative / sync decode from s until a step would start at or past `stop`; s becomes the exit.  rec: blocks
// completed and DC differences per component since the entry, or, once a restart segment began (f = 1), its first
// block index and the differences since that start.
__device__ void jd_walk(const JCtx& cx, JState& s, long long stop, JAgg& rec) {
  rec = JAgg{0, {0, 0, 0, 0}};
  if (s.j >= cx.nseg || s.pos >= stop) return;
  BitReader br;
  br.init(cx.file + s.off, cx.end, s.pos >> 3);
  br.fill();
  br.consume((int)(s.pos & 7));
  int u = s.u, k = s.k, j = s.j;
  long long segend = cx.seg_end(j);
  for (;;) {
    if (br.pos >= segend) {  // the next restart segment starts fresh
      rec = JAgg{1, {0, 0, 0, 0}};
      if (++j >= cx.nseg) {
        s = JState{JD_TERMINAL, 0, cx.nseg, 0, 0};
        return;
      }
      rec.v[0] = (uint32_t)cx.base(j);
      u = k = 0;
      br.init(cx.file + cx.seg[j].s_off, cx.end, cx.seg[j].s_u);
      segend = cx.seg_end(j);
      continue;
    }
    if (br.pos >= stop) break;
    br.fill();
    const int c = cx.comp[u];
    int len;
    const int sym = br.lookup(k ? cx.ac[c] : cx.dc[c], len);
    if (k == 0) {
      if (!len || sym > 15) {  // not a block start: resume at the next bit
        br.consume(1);
        u = 0;
        continue;
      }
      br.consume(len);
      rec.v[1 + c] += (uint32_t)br.receive_extend(sym);
      k = 1;
    } else {
      const int r = sym >> 4, sz = sym & 15;
      if (!len || (sz && k + r > 63)) {
        br.consume(1);
        u = k = 0;
        continue;
      }
      br.consume(len);
      if (sz) {
        br.consume(sz);
        k += r + 1;
      } else {
        k = r == 15 ? k + 16 : 64;  // ZRL or end of block
      }
    }
    if (k >= 64) {
      k = 0;
      u = u + 1 == cx.bpm ? 0 : u + 1;
      ++rec.v[0];
    }
  }
  s = JState{br.pos, br.locate(br.pos >> 3, cx.file, cx.scan), j, u, k};
}

// the serial reader's check at the end of interval j: from where it stopped loading, only padding without 0xFF up to
// the marker, and the marker is RSTn with n = j mod 8
__device__ __forceinline__ bool jd_restart_ok(const JCtx& cx, int j, const uint8_t* p) {
  const JSeg sg = cx.seg[j];
  if (sg.rst != (j & 7)) return false;
  for (const uint8_t* q = p; q < cx.file + sg.q_off; ++q)
    if (*q == 0xFF) return false;
  return true;
}

// Write pass of one subsequence: the true path from s (block sb, DC predictors pred) until `stop`, storing the
// coefficients; true on an error of the serial decode.
__device__ bool jd_write(const JCtx& cx, JState s, long long stop, long long sb, int pred[3], const JGeom& g,
                         int16_t* const coef[3], const uint8_t* vrow, const uint8_t* hcol) {
  if (s.j >= cx.nseg || s.pos >= stop) return false;
  BitReader br;
  br.init(cx.file + s.off, cx.end, s.pos >> 3);
  br.fill();
  br.consume((int)(s.pos & 7));
  int u = s.u, k = s.k, j = s.j;
  long long segend = cx.seg_end(j), base = cx.base(j), quota = cx.quota(j);
  bool completed = false;  // the last step ended a block
  int16_t* blk = nullptr;
  for (;;) {
    const bool done = sb - base >= quota;
    if (done || br.pos >= segend) {
      if (!done) return true;                                          // the data ends inside the interval
      if (j + 1 >= cx.needed) return false;                            // the image's last block is written
      if (completed && !jd_restart_ok(cx, j, br.p)) return true;       // checked by the thread that ended it
      if (++j >= cx.nseg) return false;                                // (then the check above failed)
      base = sb = cx.base(j);
      quota = cx.quota(j);
      pred[0] = pred[1] = pred[2] = 0;
      u = k = 0;
      br.init(cx.file + cx.seg[j].s_off, cx.end, cx.seg[j].s_u);
      segend = cx.seg_end(j);
      completed = false;
      continue;
    }
    if (br.pos >= stop) return false;
    completed = false;
    const int c = cx.comp[u];
    if (k == 0 || !blk) {
      const long long m = sb / cx.bpm;
      const int my = (int)(m / g.mcux), mx = (int)(m % g.mcux);
      blk = coef[c] + ((size_t)(my * g.vs[c] + vrow[u]) * g.bw[c] + mx * g.hs[c] + hcol[u]) * 64;
    }
    br.fill();
    int len;
    const int sym = br.lookup(k ? cx.ac[c] : cx.dc[c], len);
    if (!len) return true;
    br.consume(len);
    if (k == 0) {
      if (sym > 15) return true;
      pred[c] = (int)((uint32_t)pred[c] + (uint32_t)br.receive_extend(sym));
      blk[0] = (int16_t)pred[c];
      k = 1;
    } else {
      const int r = sym >> 4, sz = sym & 15;
      if (sz) {
        k += r;
        if (k > 63) return true;
        blk[kZigzag[k]] = (int16_t)br.receive_extend(sz);
        ++k;
      } else {
        k = r == 15 ? k + 16 : 64;
      }
    }
    if (br.pos > segend) return true;  // bits consumed past the data
    if (k >= 64) {
      k = 0;
      u = u + 1 == cx.bpm ? 0 : u + 1;
      ++sb;
      completed = true;
    }
  }
}

// file offset of scan byte x, from the chunk table (chunk_u[c]: scan byte at file byte begin + c * csize; ~0u past
// the data): the first byte at or after the chunk start with x scan bytes before it that is not a stuffed zero
__device__ uint32_t jd_map(const uint8_t* file, uint32_t begin, uint32_t end, uint32_t csize, const uint32_t* chunk_u,
                           long long x) {
  if (begin >= end) return begin;
  int lo = 0, hi = JD_ENTROPY_THREADS - 1;  // chunk_u[0] = 0 <= x
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if ((long long)chunk_u[mid] <= x) lo = mid;
    else hi = mid - 1;
  }
  uint32_t i = begin + (uint32_t)lo * csize;
  long long u = chunk_u[lo];
  for (; i < end; ++i) {
    if (i > begin && file[i] == 0x00 && file[i - 1] == 0xFF) continue;
    if (u == x) break;
    ++u;
  }
  return i;
}

__device__ __forceinline__ bool jd_stuffed(const uint8_t* f, uint32_t i, uint32_t begin) {
  return i > begin && f[i] == 0x00 && f[i - 1] == 0xFF;
}
__device__ __forceinline__ bool jd_marker(const uint8_t* f, uint32_t i, uint32_t begin, uint32_t end) {
  return f[i] == 0xFF && (i + 1 == end || f[i + 1] != 0x00) && (i == begin || f[i - 1] != 0xFF);
}

// One CTA per entry.  Warp 0 validates the entry, its output slot and its workspace region (whose offset it records in
// the workspace header) and builds the Huffman tables; then the CTA decodes the image as described above.
__global__ void __launch_bounds__(JD_ENTROPY_THREADS, 1) jpeg_entropy_kernel(
    const uint8_t* __restrict__ src, long long src_bytes, const ctl_jpeg_entry* __restrict__ entries,
    const ctl_resize_entry* __restrict__ out_table, long long out_bytes, uint8_t* __restrict__ ws, long long ws_bytes,
    long long n, int* __restrict__ status) {
  constexpr int T = JD_ENTROPY_THREADS;
  __shared__ HuffTable dc[3], ac[3];
  __shared__ uint32_t chunk_u[T];
  __shared__ long long x_pos[T];
  __shared__ uint32_t x_off[T];
  __shared__ int x_j[T], x_uk[T];
  __shared__ JAgg tot[T / 32];
  __shared__ uint8_t comp[10], vrow[10], hcol[10];
  __shared__ long long region_s;
  __shared__ int go_s, first_other_s, err_s;
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, tid = threadIdx.x;
  const ctl_jpeg_entry e = entries[b];
  if (tid < 32) {
    const int lane = tid;
    long long region = 0;
    for (long long j = lane; j < b; j += 32) region += jpeg_region_bytes(entries[j]);
    for (int o = 16; o > 0; o >>= 1) region += __shfl_xor_sync(0xffffffffu, region, o);
    region += jpeg_header_bytes(n);
    const ctl_resize_entry o = out_table[b];
    if (lane == 0) reinterpret_cast<long long*>(ws)[b] = region;
    int st = 0;
    JGeom g;
    const bool jpeg = e.kind == CTL_JPEG_ENTRY_JPEG;
    if (e.kind == CTL_JPEG_ENTRY_MOCK) {
      if (o.h != 0 || o.w != 0) st |= JS_OUTPUT;
    } else if (!jpeg && e.kind != CTL_JPEG_ENTRY_RAW) {
      st |= JS_ENTRY;
    } else {
      if (e.offset < 0 || e.nbytes < 0 || e.offset > src_bytes || e.nbytes > src_bytes - e.offset) st |= JS_ENTRY;
      if (e.desc.h < 1 || e.desc.w < 1 || e.desc.h > JD_MAX_SIDE || e.desc.w > JD_MAX_SIDE) st |= JS_ENTRY;
      if (!jpeg && e.nbytes != (long long)e.desc.h * e.desc.w * 3) st |= JS_ENTRY;
      if (jpeg) {
        const ctl_jpeg_desc& d = e.desc;
        if (!jpeg_geom(d, g) || d.scan_begin > d.scan_end || !in_file(d.scan_end, 0, e.nbytes)) st |= JS_ENTRY;
        for (int c = 0; c < d.ncomp && c < 3; ++c)
          if (!in_file(d.dqt[c], (d.dqt16 >> c & 1) ? 128 : 64, e.nbytes)) st |= JS_ENTRY;
        if (!st && region + jpeg_region_bytes(e) > ws_bytes) st |= JS_WORKSPACE;
      }
      if (o.h != e.desc.h || o.w != e.desc.w || o.offset < 0 || o.offset > out_bytes ||
          o.h * o.w * 3 > out_bytes - o.offset)
        st |= JS_OUTPUT;
    }
    bool go = jpeg && !st;
    if (go) {
      const uint8_t* file = src + e.offset;
      bool ok = true;
      for (int c = 0; c < g.nc; ++c) {
        ok = build_huff(file, e.nbytes, e.desc.dht_dc[c], dc[c]) && ok;
        ok = build_huff(file, e.nbytes, e.desc.dht_ac[c], ac[c]) && ok;
      }
      if (!ok) st = JS_ENTRY;
      go = ok;
    }
    if (lane == 0) {
      if (!go) status[b] = st;
      region_s = region;
      go_s = go;
      first_other_s = INT32_MAX;
      err_s = 0;
      if (go) {
        int i = 0;
        for (int c = 0; c < g.nc; ++c)
          for (int v = 0; v < g.vs[c]; ++v)
            for (int h = 0; h < g.hs[c]; ++h, ++i) comp[i] = (uint8_t)c, vrow[i] = (uint8_t)v, hcol[i] = (uint8_t)h;
      }
    }
  }
  __syncthreads();
  if (!go_s) return;  // CTA-uniform

  JGeom g;
  jpeg_geom(e.desc, g);
  const long long region = region_s;
  const uint8_t* file = src + e.offset;
  const uint32_t begin = e.desc.scan_begin, end = e.desc.scan_end;
  int16_t* coef[3];
  {
    int16_t* base = reinterpret_cast<int16_t*>(ws + region);
    for (int c = 0; c < g.nc; ++c) {
      coef[c] = base;
      base += (size_t)g.bw[c] * g.bh[c] * 64;
    }
    uint4* z = reinterpret_cast<uint4*>(ws + region);  // the write pass stores only the nonzero coefficients
    for (long long i = tid; i < g.blocks * 8; i += T) z[i] = make_uint4(0, 0, 0, 0);
  }
  JSeg* seg = reinterpret_cast<JSeg*>(ws + region + g.blocks * 128);  // <= MCUs entries of 20 B in 64 B per block
  const long long mcus = (long long)g.mcux * g.mcuy;
  const int ri = e.desc.restart_interval;
  const int needed = ri ? (int)((mcus + ri - 1) / ri) : 1;

  // 1. marker scan over T chunks of the scan bytes
  const uint32_t len = end - begin, csize = (len + T - 1) / T;
  const uint32_t c0 = min(begin + (uint32_t)tid * csize, end), c1 = min(c0 + csize, end);
  JAgg cnt = {0, {0, 0, 0, 0}};
  for (uint32_t i = c0; i < c1; ++i) {
    cnt.v[0] += jd_stuffed(file, i, begin);
    cnt.v[1] += jd_marker(file, i, begin, end);
  }
  const JAgg pre = jagg_exclusive_scan(cnt, tot);
  chunk_u[tid] = c0 < end ? (uint32_t)(c0 - begin) - pre.v[0] : ~0u;
  {
    long long u = (long long)(c0 - begin) - pre.v[0];
    long long m = pre.v[1];
    for (uint32_t i = c0; i < c1 && m < needed; ++i) {
      if (jd_stuffed(file, i, begin)) continue;
      if (jd_marker(file, i, begin, end)) {
        uint32_t r = i;
        while (r < end && file[r] == 0xFF) ++r;
        const int rst = ri && r < end && file[r] >= 0xD0 && file[r] <= 0xD7 ? file[r] - 0xD0 : -1;
        seg[m].q_off = i;
        seg[m].q_u = (uint32_t)u;
        seg[m].rst = rst;
        if (rst < 0) atomicMin(&first_other_s, (int)m);
        if (rst >= 0 && m + 1 < needed) {
          seg[m + 1].s_off = r + 1;
          seg[m + 1].s_u = (uint32_t)(u + (r + 1 - i));
        }
        ++m;
      }
      ++u;
    }
  }
  if (tid == T - 1) {  // totals: the inclusive scan of the last chunk
    const uint32_t marks = pre.v[1] + cnt.v[1];
    const uint32_t bytes = len - (pre.v[0] + cnt.v[0]);
    x_off[0] = marks;  // handed to the CTA below
    x_off[1] = bytes;
  }
  if (tid == 0) {
    seg[0].s_off = begin;
    seg[0].s_u = 0;
  }
  __syncthreads();
  const uint32_t marks = x_off[0], scan_bytes = x_off[1];
  const int nseg = min(needed, min(first_other_s, marks > (uint32_t)INT32_MAX ? INT32_MAX : (int)marks) + 1);
  __syncthreads();
  if (tid == 0 && (uint32_t)(nseg - 1) >= marks) {  // the last segment runs to the end of the data
    seg[nseg - 1].q_off = end;
    seg[nseg - 1].q_u = scan_bytes;
    seg[nseg - 1].rst = -1;
  }
  __syncthreads();

  JCtx cx;
  cx.file = file;
  cx.scan = file + begin;
  cx.end = file + end;
  cx.seg = seg;
  cx.nseg = nseg;
  cx.needed = needed;
  cx.ri = ri;
  cx.bpm = (int)(g.blocks / mcus);
  cx.total = g.blocks;
  cx.dc = dc;
  cx.ac = ac;
  cx.comp = comp;

  // 2. speculative pass
  const long long bits = cx.seg_end(nseg - 1);
  const long long S = (max(JD_SUB_MIN_BITS, (bits + T - 1) / T) + 31) & ~31LL;
  const int nsub = (int)max(1LL, (bits + S - 1) / S);
  const bool live = tid < nsub;
  const long long stop = tid + 1 == nsub ? JD_TERMINAL : (tid + 1) * S;
  JState entry{0, begin, 0, 0, 0};
  JAgg rec = {0, {0, 0, 0, 0}};
  if (live) {
    const long long p0 = tid * S;
    int lo = 0, hi = nseg - 1;  // the segment holding p0: the last one starting at or before it
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if ((long long)seg[mid].s_u * 8 <= p0) lo = mid;
      else hi = mid - 1;
    }
    entry = JState{p0, jd_map(file, begin, end, csize, chunk_u, p0 >> 3), lo, 0, 0};
    JState s = entry;
    jd_walk(cx, s, stop, rec);
    x_pos[tid] = s.pos;
    x_off[tid] = s.off;
    x_j[tid] = s.j;
    x_uk[tid] = s.u | s.k << 8;
  }
  // 3. sync rounds
  for (;;) {
    __syncthreads();
    JState in = entry;
    if (live && tid > 0) in = JState{x_pos[tid - 1], x_off[tid - 1], x_j[tid - 1], x_uk[tid - 1] & 0xFF, x_uk[tid - 1] >> 8};
    const bool redo = live && (in.pos != entry.pos || in.u != entry.u || in.k != entry.k);
    __syncthreads();
    if (redo) {
      entry = in;
      JState s = in;
      jd_walk(cx, s, stop, rec);
      x_pos[tid] = s.pos;
      x_off[tid] = s.off;
      x_j[tid] = s.j;
      x_uk[tid] = s.u | s.k << 8;
    }
    if (!__syncthreads_or(redo)) break;
  }
  // 4. counts
  const JAgg at = jagg_exclusive_scan(rec, tot);
  // 5. write pass
  if (live) {
    int pred[3] = {(int)at.v[1], (int)at.v[2], (int)at.v[3]};
    if (jd_write(cx, entry, stop, (long long)at.v[0], pred, g, coef, vrow, hcol)) err_s = 1;
  }
  __syncthreads();
  if (tid == 0) status[b] = err_s ? JS_DATA : 0;
}

// ---------------------------------------------------------------------------------------------------------------
// dequantisation + jpeg_idct_islow

constexpr long long FIX_0_298631336 = 2446, FIX_0_390180644 = 3196, FIX_0_541196100 = 4433, FIX_0_765366865 = 6270,
                    FIX_0_899976223 = 7373, FIX_1_175875602 = 9633, FIX_1_501321110 = 12299,
                    FIX_1_847759065 = 15137, FIX_1_961570560 = 16069, FIX_2_053119869 = 16819,
                    FIX_2_562915447 = 20995, FIX_3_072711026 = 25172;

__device__ __forceinline__ long long descale(long long x, int n) { return (x + (1LL << (n - 1))) >> n; }

// the 1-D islow butterfly of jidctint.c on d[0..7] (already dequantised / from the workspace); out[k] before descale
__device__ __forceinline__ void islow_1d(const long long d[8], long long out[8]) {
  long long z2 = d[2], z3 = d[6];
  long long z1 = (z2 + z3) * FIX_0_541196100;
  long long tmp2 = z1 + z3 * -FIX_1_847759065;
  long long tmp3 = z1 + z2 * FIX_0_765366865;
  long long tmp0 = (d[0] + d[4]) * (1LL << 13);
  long long tmp1 = (d[0] - d[4]) * (1LL << 13);
  const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = d[7];
  tmp1 = d[5];
  tmp2 = d[3];
  tmp3 = d[1];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  long long z4 = tmp1 + tmp3;
  const long long z5 = (z3 + z4) * FIX_1_175875602;
  tmp0 *= FIX_0_298631336;
  tmp1 *= FIX_2_053119869;
  tmp2 *= FIX_3_072711026;
  tmp3 *= FIX_1_501321110;
  z1 *= -FIX_0_899976223;
  z2 *= -FIX_2_562915447;
  z3 *= -FIX_1_961570560;
  z4 *= -FIX_0_390180644;
  z3 += z5;
  z4 += z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  out[0] = tmp10 + tmp3;
  out[7] = tmp10 - tmp3;
  out[1] = tmp11 + tmp2;
  out[6] = tmp11 - tmp2;
  out[2] = tmp12 + tmp1;
  out[5] = tmp12 - tmp1;
  out[3] = tmp13 + tmp0;
  out[4] = tmp13 - tmp0;
}

// the post-IDCT limit of x = sample - 128 as libjpeg-turbo's SIMD IDCTs apply it: saturation
__device__ __forceinline__ uint8_t idct_limit(long long v) { return (uint8_t)(v < -128 ? 0 : v > 127 ? 255 : v + 128); }

__global__ void __launch_bounds__(JD_IDCT_THREADS) jpeg_idct_kernel(const uint8_t* __restrict__ src,
                                                                    const ctl_jpeg_entry* __restrict__ entries,
                                                                    uint8_t* __restrict__ ws,
                                                                    const int* __restrict__ status) {
  __shared__ int16_t qt[3][64];  // natural order
  __shared__ int32_t work[JD_IDCT_THREADS / 8][64];
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const ctl_jpeg_entry& e = entries[b];
  if (e.kind != CTL_JPEG_ENTRY_JPEG || status[b] != 0) return;  // block-uniform
  JGeom g;
  jpeg_geom(e.desc, g);
  const uint8_t* file = src + e.offset;
  for (int i = threadIdx.x; i < g.nc * 64; i += blockDim.x) {
    const int c = i >> 6, k = i & 63;
    const uint8_t* q = file + e.desc.dqt[c];
    const int v = (e.desc.dqt16 >> c & 1) ? (q[2 * k] << 8 | q[2 * k + 1]) : q[k];
    qt[c][kZigzag[k]] = (int16_t)v;  // ISLOW_MULT_TYPE is short
  }
  __syncthreads();
  const long long region = reinterpret_cast<const long long*>(ws)[b];
  const int16_t* coef = reinterpret_cast<const int16_t*>(ws + region);
  uint8_t* planes = ws + region + g.blocks * 128;
  const int slot = threadIdx.x >> 3, t = threadIdx.x & 7;
  for (long long base = (long long)blockIdx.y * (JD_IDCT_THREADS / 8); base < g.blocks;
       base += (long long)gridDim.y * (JD_IDCT_THREADS / 8)) {
    const long long blk = base + slot;
    const bool live = blk < g.blocks;
    int c = 0;
    long long first = 0;  // first block of component c
    while (c + 1 < g.nc && blk >= first + (long long)g.bw[c] * g.bh[c]) first += (long long)g.bw[c] * g.bh[c], ++c;
    if (live) {  // pass 1: column t
      const int16_t* in = coef + blk * 64;
      long long d[8], r[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) d[k] = (int)in[k * 8 + t] * (int)qt[c][k * 8 + t];
      islow_1d(d, r);
#pragma unroll
      for (int k = 0; k < 8; ++k) work[slot][k * 8 + t] = (int32_t)descale(r[k], 13 - 2);
    }
    __syncthreads();
    if (live) {  // pass 2: row t
      long long d[8], r[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) d[k] = work[slot][t * 8 + k];
      islow_1d(d, r);
      uint8_t px[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) px[k] = idct_limit(descale(r[k], 13 + 2 + 3));
      const long long local = blk - first;
      const int by = (int)(local / g.bw[c]), bx = (int)(local % g.bw[c]);
      uint8_t* plane = planes + first * 64;
      const size_t stride = (size_t)g.bw[c] * 8;
      uint2 v;
      v.x = px[0] | px[1] << 8 | px[2] << 16 | (uint32_t)px[3] << 24;
      v.y = px[4] | px[5] << 8 | px[6] << 16 | (uint32_t)px[7] << 24;
      *reinterpret_cast<uint2*>(plane + (size_t)(by * 8 + t) * stride + bx * 8) = v;
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------------
// upsampling + colour conversion

// component c's sample at output pixel (y, x): jdsample.c's method for its ratio, read from its plane
__device__ __forceinline__ int upsample(const JGeom& g, int c, const uint8_t* plane, int y, int x) {
  const int fh = g.maxh / g.hs[c], fv = g.maxv / g.vs[c], dw = g.dw[c], dh = g.dh[c];
  const size_t s = (size_t)g.bw[c] * 8;
  if (fh == 1 && fv == 1) return plane[(size_t)y * s + x];
  if (fh == 2 && fv == 1 && dw > 2) {  // h2v1_fancy_upsample
    const uint8_t* row = plane + (size_t)y * s;
    const int i = x >> 1, a = 3 * row[i];
    return (x & 1) ? (a + row[min(i + 1, dw - 1)] + 2) >> 2 : (a + row[max(i - 1, 0)] + 1) >> 2;
  }
  if (fh == 1 && fv == 2) {  // h1v2_fancy_upsample
    const int r0 = y >> 1, r1 = (y & 1) ? min(r0 + 1, dh - 1) : max(r0 - 1, 0);
    return (3 * plane[(size_t)r0 * s + x] + plane[(size_t)r1 * s + x] + ((y & 1) ? 2 : 1)) >> 2;
  }
  if (fh == 2 && fv == 2 && dw > 2) {  // h2v2_fancy_upsample: column sums of the nearer and the further row
    const int r0 = y >> 1, r1 = (y & 1) ? min(r0 + 1, dh - 1) : max(r0 - 1, 0);
    const uint8_t *p0 = plane + (size_t)r0 * s, *p1 = plane + (size_t)r1 * s;
    const int i = x >> 1, j = (x & 1) ? min(i + 1, dw - 1) : max(i - 1, 0);
    const int here = 3 * p0[i] + p1[i], there = 3 * p0[j] + p1[j];
    return (x & 1) ? (3 * here + there + 7) >> 4 : (3 * here + there + 8) >> 4;
  }
  return plane[(size_t)(y / fv) * s + x / fh];  // h2v1 / h2v2 with a width <= 2, int_upsample
}

__device__ __forceinline__ uint8_t clamp255(int v) { return (uint8_t)min(max(v, 0), 255); }

__global__ void __launch_bounds__(JD_COLOR_THREADS) jpeg_color_kernel(const uint8_t* __restrict__ src,
                                                                      const ctl_jpeg_entry* __restrict__ entries,
                                                                      const ctl_resize_entry* __restrict__ out_table,
                                                                      const uint8_t* __restrict__ ws,
                                                                      uint8_t* __restrict__ out,
                                                                      const int* __restrict__ status) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const ctl_jpeg_entry& e = entries[b];
  const int st = status[b];
  if (e.kind == CTL_JPEG_ENTRY_MOCK || (st & JS_OUTPUT) || (e.kind != CTL_JPEG_ENTRY_JPEG && e.kind != CTL_JPEG_ENTRY_RAW))
    return;
  const ctl_resize_entry o = out_table[b];
  uint8_t* dst = out + o.offset;
  const long long bytes = o.h * o.w * 3;
  const long long stride = (long long)gridDim.y * blockDim.x;
  const long long first = (long long)blockIdx.y * blockDim.x + threadIdx.x;
  if (st) {  // zeros
    for (long long i = first; i < bytes; i += stride) dst[i] = 0;
    return;
  }
  if (e.kind == CTL_JPEG_ENTRY_RAW) {
    const uint8_t* s = src + e.offset;
    for (long long i = first; i < bytes; i += stride) dst[i] = s[i];
    return;
  }
  JGeom g;
  jpeg_geom(e.desc, g);
  const long long region = reinterpret_cast<const long long*>(ws)[b];
  const uint8_t* planes[3];
  {
    const uint8_t* p = ws + region + g.blocks * 128;
    for (int c = 0; c < g.nc; ++c) {
      planes[c] = p;
      p += (size_t)g.bw[c] * g.bh[c] * 64;
    }
  }
  const int w = (int)o.w;
  for (long long i = first; i < o.h * o.w; i += stride) {
    const int y = (int)(i / w), x = (int)(i % w);
    uint8_t* d = dst + i * 3;
    const int yy = upsample(g, 0, planes[0], y, x);
    if (g.nc == 1) {
      d[0] = d[1] = d[2] = (uint8_t)yy;
      continue;
    }
    const int cb = upsample(g, 1, planes[1], y, x) - 128, cr = upsample(g, 2, planes[2], y, x) - 128;
    // jdcolor.c build_ycc_rgb_table: FIX(1.40200) = 91881, FIX(1.77200) = 116130, FIX(0.71414) = 46802,
    // FIX(0.34414) = 22554, ONE_HALF = 1 << 15; >> is arithmetic (RIGHT_SHIFT)
    d[0] = clamp255(yy + ((91881 * cr + 32768) >> 16));
    d[1] = clamp255(yy + ((-46802 * cr - 22554 * cb + 32768) >> 16));
    d[2] = clamp255(yy + ((116130 * cb + 32768) >> 16));
  }
}

static unsigned jd_grid_y(long long units, int per_cta) {
  return (unsigned)std::min<long long>(std::max<long long>((units + per_cta - 1) / per_cta, 1), 65535);
}

// ---------------------------------------------------------------------------------------------------------------
// host parser

struct Cursor {
  const uint8_t* p;
  long long n;
};

static int be16(const uint8_t* p) { return p[0] << 8 | p[1]; }

#define JP_REJECT(code, ...)       \
  do {                             \
    ::ctl::set_error(__VA_ARGS__); \
    return code;                   \
  } while (0)

static int jpeg_parse(const uint8_t* f, long long nbytes, ctl_jpeg_desc* d, int32_t* out_h, int32_t* out_w) {
  if (nbytes < 4 || f[0] != 0xFF || f[1] != 0xD8) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "not a JPEG: no SOI marker");
  if (nbytes > (long long)UINT32_MAX) JP_REJECT(CTL_ERR_UNSUPPORTED, "JPEG of %lld bytes: at most 4 GiB", nbytes);
  int64_t qt_off[4] = {-1, -1, -1, -1}, dht_off[2][4] = {{-1, -1, -1, -1}, {-1, -1, -1, -1}};
  int qt16[4] = {0, 0, 0, 0};
  bool sof = false, jfif = false;
  int adobe = -1;
  int nc = 0, ids[4] = {0, 0, 0, 0}, hv[4] = {0, 0, 0, 0}, tq[4] = {0, 0, 0, 0};
  int h = 0, w = 0, ri = 0;
  long long pos = 2;
  for (;;) {
    if (pos >= nbytes || f[pos] != 0xFF) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "truncated or corrupt JPEG header at byte %lld", pos);
    while (pos < nbytes && f[pos] == 0xFF) ++pos;  // fill bytes
    if (pos >= nbytes) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "truncated JPEG header: no SOS marker");
    const int m = f[pos++];
    if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;  // standalone markers
    if (m == 0xD8 || m == 0xD9) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt JPEG header: marker 0x%02X before SOS", m);
    if (pos + 2 > nbytes) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "truncated JPEG header at byte %lld", pos);
    const int len = be16(f + pos);
    if (len < 2 || pos + len > nbytes) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "truncated JPEG header: marker 0x%02X segment", m);
    const uint8_t* s = f + pos + 2;
    const long long body = pos + 2, L = len - 2;
    pos += len;
    switch (m) {
      case 0xC0:
      case 0xC1: {
        if (sof) JP_REJECT(CTL_ERR_UNSUPPORTED, "JPEG with two frame headers");
        if (L < 6) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt SOF segment");
        if (s[0] != 8) JP_REJECT(CTL_ERR_UNSUPPORTED, "%d-bit JPEG samples: only 8-bit is decoded on the device", s[0]);
        h = be16(s + 1);
        w = be16(s + 3);
        nc = s[5];
        if (h == 0) JP_REJECT(CTL_ERR_UNSUPPORTED, "JPEG height defined by a DNL marker");
        if (w == 0) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt SOF segment: width 0");
        if (nc == 4) JP_REJECT(CTL_ERR_UNSUPPORTED, "4-component (CMYK / YCCK) JPEG");
        if (nc != 1 && nc != 3) JP_REJECT(CTL_ERR_UNSUPPORTED, "%d-component JPEG: only grayscale and YCbCr", nc);
        if (L < 6 + 3 * nc) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt SOF segment");
        for (int c = 0; c < nc; ++c) {
          ids[c] = s[6 + 3 * c];
          hv[c] = s[7 + 3 * c];
          tq[c] = s[8 + 3 * c];
          const int hs = hv[c] >> 4, vs = hv[c] & 15;
          if (hs < 1 || hs > 4 || vs < 1 || vs > 4 || tq[c] > 3)
            JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt SOF segment: component %d", c);
        }
        sof = true;
        break;
      }
      case 0xC2:
      case 0xC6:
      case 0xCA:
      case 0xCE:
        JP_REJECT(CTL_ERR_UNSUPPORTED, "progressive JPEG (SOF%d)", m - 0xC0);
      case 0xC3:
      case 0xC7:
      case 0xCB:
      case 0xCF:
        JP_REJECT(CTL_ERR_UNSUPPORTED, "lossless JPEG (SOF%d)", m - 0xC0);
      case 0xC5:
        JP_REJECT(CTL_ERR_UNSUPPORTED, "hierarchical JPEG (SOF5)");
      case 0xC9:
      case 0xCD:
        JP_REJECT(CTL_ERR_UNSUPPORTED, "arithmetic-coded JPEG (SOF%d)", m - 0xC0);
      case 0xC8:
        JP_REJECT(CTL_ERR_UNSUPPORTED, "JPEG extension frame (JPG marker)");
      case 0xDB:  // DQT
        for (long long i = 0; i < L;) {
          const int pq = s[i] >> 4, t = s[i] & 15;
          const long long sz = pq ? 128 : 64;
          if (pq > 1 || t > 3 || i + 1 + sz > L) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt DQT segment");
          qt_off[t] = body + i + 1;
          qt16[t] = pq;
          i += 1 + sz;
        }
        break;
      case 0xC4:  // DHT
        for (long long i = 0; i < L;) {
          const int tc = s[i] >> 4, th = s[i] & 15;
          if (tc > 1 || th > 3 || i + 17 > L) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt DHT segment");
          int total = 0, code = 0;
          for (int l = 1; l <= 16; ++l) {
            total += s[i + l];
            code += s[i + l];
            if (code > (1 << l)) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt DHT segment: code lengths overflow");
            code <<= 1;
          }
          if (total > 256 || i + 17 + total > L) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt DHT segment");
          dht_off[tc][th] = body + i + 1;
          i += 17 + total;
        }
        break;
      case 0xCC:
        JP_REJECT(CTL_ERR_UNSUPPORTED, "arithmetic-coded JPEG (DAC marker)");
      case 0xDD:  // DRI
        if (L < 2) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt DRI segment");
        ri = be16(s);
        break;
      case 0xE0:
        if (L >= 5 && !memcmp(s, "JFIF", 5)) jfif = true;
        break;
      case 0xEE:
        if (L >= 12 && !memcmp(s, "Adobe", 5)) adobe = s[11];
        break;
      case 0xDA: {  // SOS: the end of the header
        if (!sof) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt JPEG header: SOS before SOF");
        if (L < 1) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt SOS segment");
        const int ns = s[0];
        if (L < 4 + 2 * ns) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt SOS segment");
        if (ns != nc) JP_REJECT(CTL_ERR_UNSUPPORTED, "multi-scan sequential JPEG (%d of %d components in the first scan)", ns, nc);
        const uint8_t* sp = s + 1 + 2 * ns;
        if (sp[0] != 0 || sp[1] != 63 || sp[2] != 0)
          JP_REJECT(CTL_ERR_UNSUPPORTED, "JPEG scan with spectral selection or successive approximation");
        if (nc == 3) {
          if (jfif) {
          } else if (adobe == 0) {
            JP_REJECT(CTL_ERR_UNSUPPORTED, "Adobe RGB JPEG (transform 0)");
          } else if (adobe < 0 && ids[0] == 'R' && ids[1] == 'G' && ids[2] == 'B') {
            JP_REJECT(CTL_ERR_UNSUPPORTED, "RGB JPEG (component ids R, G, B)");
          }
          int maxh = 1, maxv = 1, blocks = 0;
          for (int c = 0; c < 3; ++c) {
            maxh = std::max(maxh, hv[c] >> 4);
            maxv = std::max(maxv, hv[c] & 15);
            blocks += (hv[c] >> 4) * (hv[c] & 15);
          }
          for (int c = 0; c < 3; ++c)
            if (maxh % (hv[c] >> 4) || maxv % (hv[c] & 15))
              JP_REJECT(CTL_ERR_UNSUPPORTED, "JPEG sampling factors that need non-integral upsampling");
          if (blocks > 10) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt SOF segment: %d blocks per MCU", blocks);
        }
        memset(d, 0, sizeof(*d));
        d->h = h;
        d->w = w;
        d->ncomp = (uint8_t)nc;
        d->restart_interval = (uint16_t)ri;
        for (int c = 0; c < nc; ++c) {
          if (s[1 + 2 * c] != ids[c]) JP_REJECT(CTL_ERR_UNSUPPORTED, "JPEG scan with its components out of frame order");
          const int td = s[2 + 2 * c] >> 4, ta = s[2 + 2 * c] & 15;
          if (td > 3 || ta > 3 || dht_off[0][td] < 0 || dht_off[1][ta] < 0)
            JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt JPEG header: undefined Huffman table");
          if (qt_off[tq[c]] < 0) JP_REJECT(CTL_ERR_INVALID_ARGUMENT, "corrupt JPEG header: undefined quantisation table");
          d->dqt[c] = (uint32_t)qt_off[tq[c]];
          d->dqt16 |= (uint8_t)(qt16[tq[c]] << c);
          d->dht_dc[c] = (uint32_t)dht_off[0][td];
          d->dht_ac[c] = (uint32_t)dht_off[1][ta];
          d->hs[c] = nc == 1 ? 1 : (uint8_t)(hv[c] >> 4);
          d->vs[c] = nc == 1 ? 1 : (uint8_t)(hv[c] & 15);
        }
        d->scan_begin = (uint32_t)pos;
        d->scan_end = (uint32_t)nbytes;
        if (out_h) *out_h = h;
        if (out_w) *out_w = w;
        return 0;
      }
      default:  // APPn, COM, DNL, ...: skipped
        break;
    }
  }
}

}  // namespace ctl

using namespace ctl;

extern "C" {

int ctl_jpeg_parse(const void* bytes, int64_t nbytes, ctl_jpeg_desc* desc, int32_t* h, int32_t* w) {
  CTL_CHECK_ARG(bytes && desc, "null pointer");
  CTL_CHECK_ARG(nbytes >= 0, "nbytes < 0");
  return jpeg_parse(static_cast<const uint8_t*>(bytes), nbytes, desc, h, w);
}

size_t ctl_jpeg_decode_workspace_bytes(const ctl_jpeg_entry* entries_host, int64_t n) {
  if (!entries_host || n < 1 || n > INT32_MAX) return 0;
  size_t bytes = jpeg_header_bytes(n);
  for (int64_t i = 0; i < n; ++i) bytes += (size_t)jpeg_region_bytes(entries_host[i]);
  return (bytes + 255) & ~size_t(255);
}

int ctl_jpeg_decode(const void* src, int64_t src_bytes, const void* entries_device, int64_t n,
                    const void* out_table_device, void* out_u8, int64_t out_bytes, int32_t* status, void* workspace,
                    size_t workspace_bytes, ctl_stream_t stream) {
  CTL_CHECK_ARG(src && entries_device && out_table_device && out_u8 && status && workspace, "null pointer");
  CTL_CHECK_ARG(n >= 1 && n <= INT32_MAX, "n = %lld: expected 1 <= n < 2^31", (long long)n);
  CTL_CHECK_ARG(src_bytes >= 0 && out_bytes >= 0, "negative buffer size");
  CTL_CHECK_ARG(workspace_bytes >= jpeg_header_bytes(n),
                "workspace of %zu bytes is shorter than its %zu-byte header (ctl_jpeg_decode_workspace_bytes)",
                workspace_bytes, jpeg_header_bytes(n));
  int rc = ctl_device_check();
  if (rc) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  const auto* entries = static_cast<const ctl_jpeg_entry*>(entries_device);
  const auto* table = static_cast<const ctl_resize_entry*>(out_table_device);
  auto* ws = static_cast<uint8_t*>(workspace);
  auto* s = static_cast<const uint8_t*>(src);
  int* stat = reinterpret_cast<int*>(status);
  // the later launches loop over an image's blocks / pixels; sized for the mean image the buffers were planned for
  const long long mean_blocks = (long long)((workspace_bytes - jpeg_header_bytes(n)) / (64 * 3)) / n;
  const long long mean_pixels = out_bytes / 3 / n;
  CTL_CUDA(launch_k(jpeg_entropy_kernel, dim3((unsigned)n), dim3(JD_ENTROPY_THREADS), 0, st, s, (long long)src_bytes,
                    entries, table, (long long)out_bytes, ws, (long long)workspace_bytes, (long long)n, stat));
  CTL_CUDA(launch_k(jpeg_idct_kernel, dim3((unsigned)n, jd_grid_y(mean_blocks, JD_IDCT_THREADS / 8)),
                    dim3(JD_IDCT_THREADS), 0, st, s, entries, ws, (const int*)stat));
  CTL_CUDA(launch_k(jpeg_color_kernel, dim3((unsigned)n, jd_grid_y(mean_pixels, JD_COLOR_THREADS)),
                    dim3(JD_COLOR_THREADS), 0, st, s, entries, table, (const uint8_t*)ws, static_cast<uint8_t*>(out_u8),
                    (const int*)stat));
  return 0;
}

}  // extern "C"
