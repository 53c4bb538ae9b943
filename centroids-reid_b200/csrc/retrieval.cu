// Query x gallery distances on Hopper tensor cores (wgmma) with streamed top-k / CMC / mAP epilogues.
//
// Replaces utils/reid_metric.py:25-33,51-59,112-136, utils/eval_reid.py:25-92 and
// inference/get_similar.py:104-128 of the reference (see include/ctl_b200.h).
//
// Arithmetic.  The reference computes q.g in fp32.  Here every fp32 row x is split to within 2^-23 |x s| as
//     x * s = hi + 2^-11 * lo        (s: per-row power of two, hi/lo: fp16; exact for rows of <= 20 significant bits)
// and q.g = (hi_q.hi_g + 2^-11 (hi_q.lo_g + lo_q.hi_g)) / (s_q s_g): three fp16 wgmma
// passes with fp32 accumulation into TWO register accumulators (the 2^-11 terms never get swamped
// by the leading term).  Dropped: 2^-22 lo.lo -- i.e. >= 22 significant bits per product,
// fp32-equivalent, and EXACT whenever the operands have <= 11 significant bits (the
// dyadic-grid fixtures on which rank parity is asserted bit-exact).
//
// One persistent CTA per SM, 3 warpgroups: a TMA producer and two consumers; 2-stage smem ring of
// {q_hi, q_lo, g_hi, g_lo} 128x64 fp16 tiles (SWIZZLE_128B).  Consumer warpgroup wg multiplies
// query rows [64 wg, 64 wg + 64) of the tile (two m64n128 accumulators in registers), folds them
// into one fp32 dot product per element, stages its rows in shared memory and runs the epilogue
// on them, one thread per (query row, 64-column half); the producer fills the ring meanwhile.
#include <limits.h>
#include <math_constants.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "common.h"
#include "wgmma.cuh"

namespace ctl {

static constexpr int BM = 128;      // queries per tile (2 consumer warpgroups x 64 rows)
static constexpr int BN = 128;      // gallery rows per tile
static constexpr int BK = 64;       // fp16 elements per k-block = one 128-byte swizzle row
static constexpr int STAGES = 2;
static constexpr int TILE_BYTES = BM * BK * 2;          // 16 KiB
static constexpr int STAGE_BYTES = 4 * TILE_BYTES;      // q_hi, q_lo, g_hi, g_lo
static constexpr int GEMM_THREADS = 384;  // producer warpgroup + 2 consumer warpgroups
static constexpr uint32_t GEMM_PRODUCER_REGS = 40, GEMM_CONSUMER_REGS = 232;
static constexpr int ACC_BYTES = BM * BN * 4;  // the tile's fp32 dot products, one 512-byte row per query
static constexpr int GROUP_W = 16;                      // columns per group-min
static constexpr int META_BYTES = 2 * BN * (4 + 4 + 4 + 8 + 4);  // double-buffered per-tile column metadata
static constexpr int THR_MAX = 32, THR_STRIDE = 36;         // positives per query held in shared memory (16-byte rows)
static constexpr int THR_BYTES = BM * THR_STRIDE * 4;
static constexpr int CNT_STRIDE = THR_MAX / 2 + 1;          // bucket counters of one query row: 2 x 16 bit per word
static constexpr int CNT_BYTES = BM * CNT_STRIDE * 4;
static constexpr int FAR_LEVELS = 1;  // buckets of the count pass resolved by plain compares against the farthest positives
                                      // (config 3 retrieval step on one H100: none 5.57 ms, 1 level 5.51 ms, 2 levels 5.79 ms)
static constexpr size_t GEMM_SMEM = STAGES * STAGE_BYTES + ACC_BYTES + META_BYTES + THR_BYTES + CNT_BYTES + 1024 /*align*/ + 256 /*barriers*/;
static_assert(GEMM_SMEM <= 227 * 1024, "dist_gemm_kernel shared memory");
static_assert(BN < 65536, "16-bit bucket counters of a tile");

// ---------------------------------------------------------------------------------------
// (distance, index) keys: ascending uint64 order == ascending (distance, index)
// ---------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t float_orderable(float f) {
#ifdef __CUDA_ARCH__
  uint32_t b = __float_as_uint(f);
#else
  uint32_t b;
  memcpy(&b, &f, 4);
#endif
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ __forceinline__ float orderable_float(uint32_t u) {
  uint32_t b = (u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u;
#ifdef __CUDA_ARCH__
  return __uint_as_float(b);
#else
  float f;
  memcpy(&f, &b, 4);
  return f;
#endif
}
__host__ __device__ __forceinline__ uint64_t make_key(float d, uint32_t idx) {
  return (static_cast<uint64_t>(float_orderable(d)) << 32) | idx;
}

// ---------------------------------------------------------------------------------------
// planes layout
// ---------------------------------------------------------------------------------------
struct PlanesView {
  const __half* hi;
  const __half* lo;
  const float* sq;
  const float* inv_scale;
};
static size_t planes_off_lo(int64_t n, int32_t d) { return ((size_t)n * d * 2 + 255) & ~size_t(255); }
static size_t planes_off_sq(int64_t n, int32_t d) { return 2 * planes_off_lo(n, d); }
static size_t planes_off_is(int64_t n, int32_t d) { return planes_off_sq(n, d) + (((size_t)n * 4 + 255) & ~size_t(255)); }
static size_t planes_total(int64_t n, int32_t d) { return planes_off_is(n, d) + (((size_t)n * 4 + 255) & ~size_t(255)); }
static PlanesView planes_view(const void* p, int64_t n, int32_t d) {
  const char* c = static_cast<const char*>(p);
  PlanesView v;
  v.hi = reinterpret_cast<const __half*>(c);
  v.lo = reinterpret_cast<const __half*>(c + planes_off_lo(n, d));
  v.sq = reinterpret_cast<const float*>(c + planes_off_sq(n, d));
  v.inv_scale = reinterpret_cast<const float*>(c + planes_off_is(n, d));
  return v;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One warp per row.  n_norm sequential L2 normalisations x <- x / max(|x|, 1e-12)
// (F.normalize, reid_metric.py:113-115; cosine_similarity, reid_metric.py:43-46), then the
// hi/lo split (DESIGN.md section 2: the bound) and the fp32 squared norm of the (normalised) row.
__global__ void __launch_bounds__(128) planes_build_kernel(const float* __restrict__ x, int64_t n, int d, int n_norm,
                                                           __half* __restrict__ hi, __half* __restrict__ lo,
                                                           float* __restrict__ sq, float* __restrict__ inv_scale) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= n) return;
  const float* xr = x + row * d;
  float denom[2] = {1.f, 1.f};
  for (int t = 0; t < n_norm; ++t) {
    float ss = 0.f;
    for (int i = lane; i < d; i += 32) {
      float v = xr[i];
      if (t > 0) v = __fdiv_rn(v, denom[0]);
      ss = __fmaf_rn(v, v, ss);
    }
    ss = warp_sum(ss);
    denom[t] = fmaxf(__fsqrt_rn(ss), 1e-12f);
  }
  float ss = 0.f, mx = 0.f;
  for (int i = lane; i < d; i += 32) {
    float v = xr[i];
    if (n_norm > 0) v = __fdiv_rn(v, denom[0]);
    if (n_norm > 1) v = __fdiv_rn(v, denom[1]);
    ss = __fmaf_rn(v, v, ss);
    mx = fmaxf(mx, fabsf(v));
  }
  ss = warp_sum(ss);
  mx = warp_max(mx);
  int sexp = 0;
  if (mx > 0.f && mx < CUDART_INF_F) {
    int e;
    frexpf(mx, &e);            // mx = m * 2^e, m in [0.5, 1)
    sexp = min(14 - e, 120);   // mx * 2^sexp in [2^13, 2^14)
  }
  const float scale = scalbnf(1.f, sexp);
  for (int i = lane; i < d; i += 32) {
    float v = xr[i];
    if (n_norm > 0) v = __fdiv_rn(v, denom[0]);
    if (n_norm > 1) v = __fdiv_rn(v, denom[1]);
    const float vs = v * scale;  // exact (power of two)
    const __half h = __float2half_rn(vs);
    const float r = vs - __half2float(h);  // exact remainder
    hi[row * d + i] = h;
    lo[row * d + i] = __float2half_rn(r * 2048.f);  // one bit more than fp16 holds: off by <= 2^-23 |vs|
  }
  if (lane == 0) {
    sq[row] = ss;
    inv_scale[row] = scalbnf(1.f, -sexp);
  }
}

// ---------------------------------------------------------------------------------------
// the GEMM pass
// ---------------------------------------------------------------------------------------
struct GemmPass {
  int nq, ng, d;
  int m_tiles, n_tiles;
  int cosine;
  long long g_off;
  const float* q_sq;
  const float* q_is;
  const float* g_sq;
  const float* g_is;
  // full matrix
  float* dist_out;
  long long ld_out;
  // group minima (pass A of top-k)
  float* gmin;
  int n_groups;
  // candidates <= tau (pass B of top-k)
  const float* tau;
  unsigned long long* cand_keys;
  int* cand_count;
  int cand_cap;
  // identities (eval)
  const int* q_pid;
  const int* q_cam;
  const int* g_pid;
  const unsigned long long* g_mask;
  unsigned long long* pos_keys;  // collect
  int* pos_count;
  int max_pos;
  const unsigned long long* thr_keys;  // count
  const int* thr_count;
  int* buckets;
  int* overflow;
  // optional tile list (ctl_dist_worklist): work[0] = number of tiles to run, work[1..] their ids in ascending order.
  // A pass that only collects the positives and a threshold needs the tiles that can hold a positive plus a subset for
  // the group minima -- with both operands stored in identity order that is a fraction of the matrix.
  const int* work;
  const int* g_map;     // optional: gallery row -> index written into the keys (rows stored in another order)
};

struct GemmMaps {
  CUtensorMap q_hi, q_lo, g_hi, g_lo;
};

// The ONE place a distance is formed from the accumulators (dot_from_acc, then dist_from_dot): every
// pass must produce bit-identical values for the same (query, gallery) pair.
// d[j] for a runtime j without spilling the array to local memory: a 4-level select tree (15 FSEL)
__device__ __forceinline__ float select16(const float (&d)[16], int j) {
  float a[8], b[4], c[2];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = (j & 1) ? d[2 * i + 1] : d[2 * i];
#pragma unroll
  for (int i = 0; i < 4; ++i) b[i] = (j & 2) ? a[2 * i + 1] : a[2 * i];
#pragma unroll
  for (int i = 0; i < 2; ++i) c[i] = (j & 4) ? b[2 * i + 1] : b[2 * i];
  return (j & 8) ? c[1] : c[0];
}

__device__ __forceinline__ float dot_from_acc(float acc0, float acc1) {
  return __fmaf_rn(acc1, 4.8828125e-4f /* 2^-11 */, acc0);
}
__device__ __forceinline__ float dist_from_dot(float dot, float q_is, float g_is, float qq, float gg, int cosine) {
  dot = __fmul_rn(__fmul_rn(dot, q_is), g_is);
  if (cosine & 1) return fmaxf(fabsf(__fsub_rn(1.f, dot)), 1e-12f);
  const float sqd = __fmaf_rn(-2.f, dot, __fadd_rn(qq, gg));
  // CTL_DIST_SQRT: losses/triplet_loss.py:40  dist.clamp(min=1e-12).sqrt()
  return (cosine & 4) ? __fsqrt_rn(fmaxf(sqd, 1e-12f)) : sqd;
}

// exact (distance, index) search in the sorted positives of one query: first entry > key (entry npos-1 is > key)
__device__ __noinline__ int bucket_search_global(const unsigned long long* __restrict__ thr, int npos,
                                                 unsigned long long key) {
  int lo = 0, hi = npos - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (thr[mid] > key) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// Work item w of a pass -> query tile mt, gallery tile nt; tile id = nt * m_tiles + mt.
//   full pass: tile id w, query tiles fastest -- the CTAs that run concurrently touch ~5 gallery tiles x all query
//              tiles, so each operand tile is fetched from HBM about once.  One tile per work item in every pass: longer
//              items for the count pass (the per-row thresholds and counters set up and flushed once per several gallery
//              tiles) gave no gain (config 3 retrieval step on one H100, measured while the epilogue still spilled
//              registers: 5.51 ms (1 tile), 5.50 ms (2), 5.74 ms (4));
//   tile list: the listed tile work[1 + w].
__device__ __forceinline__ void tile_coords(const GemmPass& p, int w, int& mt, int& nt) {
  const int id = p.work ? p.work[1 + w] : w;
  nt = id / p.m_tiles;
  mt = id - nt * p.m_tiles;
}

// Shared-memory word of element (row, col) of the staged dot-product tile: 16-byte chunks of a row XOR-swizzled by
// (2 row + chunk / 16) & 7, so neither the accumulator stores nor the epilogue's row reads conflict on a bank.
__device__ __forceinline__ int acc_word(int row, int col) {
  const int chunk = col >> 2;
  return row * BN + ((chunk ^ ((2 * row + (chunk >> 4)) & 7)) << 2) + (col & 3);
}

__global__ void __launch_bounds__(GEMM_THREADS, 1)
    dist_gemm_kernel(const __grid_constant__ GemmMaps maps, const GemmPass p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t acc_base = smem_base + STAGES * STAGE_BYTES;
  const uint32_t meta_base = acc_base + ACC_BYTES;
  const uint32_t thr_base = meta_base + META_BYTES;
  const uint32_t bar_base = thr_base + THR_BYTES + CNT_BYTES;
  // barriers: full[STAGES], empty[STAGES]
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // every role walks the same sequence of work items (tile_coords)
  const int num_work = p.work ? p.work[0] : p.m_tiles * p.n_tiles;
  const int k_blocks = (p.d + BK - 1) / BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
    tma_prefetch_desc(&maps.q_hi);
    tma_prefetch_desc(&maps.q_lo);
    tma_prefetch_desc(&maps.g_hi);
    tma_prefetch_desc(&maps.g_lo);
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<GEMM_PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
        int mt, nt;
        tile_coords(p, w, mt, nt);
        for (int kb = 0; kb < k_blocks; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t dst = smem_base + stage * STAGE_BYTES;
          mbar_arrive_expect_tx(full_bar(stage), STAGE_BYTES);
          tma_load_2d(dst + 0 * TILE_BYTES, &maps.q_hi, full_bar(stage), kb * BK, mt * BM);
          tma_load_2d(dst + 1 * TILE_BYTES, &maps.q_lo, full_bar(stage), kb * BK, mt * BM);
          tma_load_2d(dst + 2 * TILE_BYTES, &maps.g_hi, full_bar(stage), kb * BK, nt * BN);
          tma_load_2d(dst + 3 * TILE_BYTES, &maps.g_lo, full_bar(stage), kb * BK, nt * BN);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
  } else {
    // ===================== consumers: MMA + epilogue, one thread per (query row, 64-column half) =====
    // Per-tile column metadata (|g|^2, 1/scale, pid, camera mask of the 128 gallery rows) is staged
    // once in shared memory; every thread then reads it by broadcast instead of 4 global loads per
    // element.
    setmaxnreg_inc<GEMM_CONSUMER_REGS>();
    const int wg = (threadIdx.x >> 7) - 1;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const int wrow0 = 64 * wg + 16 * (warp & 3);  // first of the 16 tile rows this warp multiplies and drains
    float* acc_s = reinterpret_cast<float*>(smem_raw + (acc_base - smem_u32(smem_raw)));
    int stage = 0;
    uint32_t phase = 0;
    const int ew = warp - 4;          // 0..7
    const int et = threadIdx.x - 128;  // 0..255
    const int chalf = lane & 1;       // columns [64*chalf, 64*chalf + 64) of the tile
    const int row_in_tile = wrow0 + (lane >> 1);
    float* cm_sq = reinterpret_cast<float*>(smem_raw + (meta_base - smem_u32(smem_raw)));  // [2][128]
    float* cm_is = cm_sq + 2 * BN;
    int* cm_pid = reinterpret_cast<int*>(cm_is + 2 * BN);
    unsigned long long* cm_mask = reinterpret_cast<unsigned long long*>(cm_pid + 2 * BN);
    unsigned int* cm_idx = reinterpret_cast<unsigned int*>(cm_mask + 2 * BN);  // index written into the keys
    uint32_t* thr_s = reinterpret_cast<uint32_t*>(smem_raw + (thr_base - smem_u32(smem_raw)));
    int it = 0;
    uint32_t* cnt_s = thr_s + BM * THR_STRIDE;  // [BM][CNT_STRIDE]: 2 x 16-bit bucket counters per word
    const bool thr_in_smem = p.buckets != nullptr;
    const int n_stage = min(p.max_pos, THR_MAX);
    uint32_t* thr_row = thr_s + row_in_tile * THR_STRIDE;
    uint32_t* cnt_row = cnt_s + row_in_tile * CNT_STRIDE;
    if (thr_in_smem)  // the counters start at zero; every flush leaves them at zero again
      for (int i = et; i < BM * CNT_STRIDE; i += 256) cnt_s[i] = 0u;
    for (int w = blockIdx.x; w < num_work; w += gridDim.x, ++it) {
      int mt, nt;
      tile_coords(p, w, mt, nt);
      // ---- per work item: the state of this thread's query row ----
      const int row = mt * BM + row_in_tile;
      const bool row_ok = row < p.nq;
      float qq = 0.f, qis = 0.f, tau = -CUDART_INF_F;
      int qpid = -1, qcam = 0, npos = 0;
      unsigned long long maxkey = 0ull;
      // distance parts of the FAR_LEVELS + 1 farthest positives of this row, farthest first (0 where there is none)
      uint32_t tf[FAR_LEVELS + 1];
#pragma unroll
      for (int l = 0; l <= FAR_LEVELS; ++l) tf[l] = 0u;
      if (row_ok) {
        qq = p.q_sq[row];
        qis = p.q_is[row];
        if (p.tau) tau = p.tau[row];
        if (p.q_pid) {
          qpid = p.q_pid[row];
          qcam = p.q_cam[row];
        }
        if (p.buckets) {
          npos = p.thr_count[row];
          if (npos > 0) maxkey = p.thr_keys[(size_t)row * p.max_pos + npos - 1];
#pragma unroll
          for (int l = 0; l <= FAR_LEVELS; ++l)
            if (npos > l) tf[l] = (uint32_t)(p.thr_keys[(size_t)row * p.max_pos + npos - 1 - l] >> 32);
        }
      }
      // The distance halves of each row's first THR_MAX sorted positives are staged in shared memory (row stride 36
      // words: 16-byte rows, conflict-free LDS.128), so the bucket of a gallery row comes from shared memory instead of a
      // dependent chain of L2 loads; deeper positives (rare) and exact distance ties use the 64-bit global search.  The
      // metadata barrier publishes the staged rows.
      if (thr_in_smem) {
        const int rows_here = min(BM, p.nq - mt * BM);
        const unsigned long long* src = p.thr_keys + (size_t)mt * BM * p.max_pos;
        // warp `ew` stages rows ew, ew+8, ...: coalesced along the sorted entries, and all loads of a thread are issued
        // before the first shared store (one memory latency per work item, not one per row)
        const uint32_t* src_hi = reinterpret_cast<const uint32_t*>(src) + 1;  // distance half of a key
        // slots at and beyond a row's own count hold 0xFFFFFFFF (the key rows are only defined up to their count)
        uint32_t v0[BM / 8];
        int cn[BM / 8];
#pragma unroll
        for (int i = 0; i < BM / 8; ++i) {
          const int r = ew + 8 * i;
          cn[i] = r < rows_here ? min(p.thr_count[mt * BM + r], n_stage) : 0;
        }
#pragma unroll
        for (int i = 0; i < BM / 8; ++i) {
          const int r = ew + 8 * i;
          const size_t o = 2 * ((size_t)r * p.max_pos + lane);
          v0[i] = lane < cn[i] ? src_hi[o] : 0xFFFFFFFFu;
        }
#pragma unroll
        for (int i = 0; i < BM / 8; ++i) thr_s[(ew + 8 * i) * THR_STRIDE + lane] = v0[i];
      }
      const int mb = (it & 1) * BN;  // double-buffered metadata slice
      if (et < BN) {
        const int col = nt * BN + et;
        const bool ok = col < p.ng;
        cm_sq[mb + et] = ok ? p.g_sq[col] : 0.f;
        cm_is[mb + et] = ok ? p.g_is[col] : 0.f;
        cm_idx[mb + et] = (ok && p.g_map) ? static_cast<unsigned int>(p.g_map[col]) : static_cast<unsigned int>(col + p.g_off);
        if (p.q_pid) {
          cm_pid[mb + et] = ok ? p.g_pid[col] : -2;
          cm_mask[mb + et] = ok ? p.g_mask[col] : 0ull;
        }
      }
      const int nps = min(npos, THR_MAX);
      {
        // acc0 = q_hi.g_hi, acc1 = q_hi.g_lo + q_lo.g_hi over this warpgroup's 64 query rows x 128 gallery rows
        float acc0[BN / 2], acc1[BN / 2];
        int held = -1;  // ring slot still read by the wgmma group in flight
        for (int kb = 0; kb < k_blocks; ++kb) {
          mbar_wait(full_bar(stage), phase);
          const uint32_t base = smem_base + stage * STAGE_BYTES;
          const uint64_t d_qh = make_sw128_kmajor_desc(base + 0 * TILE_BYTES + wg * (TILE_BYTES / 2));
          const uint64_t d_ql = make_sw128_kmajor_desc(base + 1 * TILE_BYTES + wg * (TILE_BYTES / 2));
          const uint64_t d_gh = make_sw128_kmajor_desc(base + 2 * TILE_BYTES);
          const uint64_t d_gl = make_sw128_kmajor_desc(base + 3 * TILE_BYTES);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) {
            const uint32_t acc = (kb > 0 || k > 0) ? 1u : 0u;
            wgmma_f16<BN>(acc0, desc_advance_k(d_qh, k), desc_advance_k(d_gh, k), acc);
            wgmma_f16<BN>(acc1, desc_advance_k(d_qh, k), desc_advance_k(d_gl, k), acc);
            wgmma_f16<BN>(acc1, desc_advance_k(d_ql, k), desc_advance_k(d_gh, k), 1u);
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (held >= 0 && wg_leader) mbar_arrive(empty_bar(held));
          held = stage;
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1u;
          }
        }
        wgmma_wait<0>();
        if (held >= 0 && wg_leader) mbar_arrive(empty_bar(held));
        // this warp's 16 rows -> shared memory (only this warp reads them back)
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = wrow0 + (lane >> 2) + 8 * h, col = 8 * j + 2 * (lane & 3);
            *reinterpret_cast<float2*>(acc_s + acc_word(r, col)) =
                make_float2(dot_from_acc(acc0[4 * j + 2 * h], acc1[4 * j + 2 * h]),
                            dot_from_acc(acc0[4 * j + 2 * h + 1], acc1[4 * j + 2 * h + 1]));
          }
        __syncwarp();
      }
      named_bar_sync(1, 256);  // metadata slice published
#pragma unroll 1
      for (int c = 0; c < 4; ++c) {
        float r0[16];
#pragma unroll
        for (int q4 = 0; q4 < 4; ++q4) {
          const float4 v = *reinterpret_cast<const float4*>(acc_s + acc_word(row_in_tile, chalf * 64 + c * 16 + 4 * q4));
          r0[4 * q4] = v.x; r0[4 * q4 + 1] = v.y; r0[4 * q4 + 2] = v.z; r0[4 * q4 + 3] = v.w;
        }
        const int cl0 = chalf * 64 + c * 16;  // column inside the tile
        const int col0 = nt * BN + cl0;
        // ---- phase 1, branch-free: the 16 distances and the masks of the (rare) elements that need more ----
        float dist[16];
        uint32_t m_valid = 0, m_cand = 0, m_pos = 0, m_cnt = 0;
        uint32_t m_far[FAR_LEVELS];
#pragma unroll
        for (int l = 0; l < FAR_LEVELS; ++l) m_far[l] = 0u;
        float gmin = CUDART_INF_F;
        {
          const float4* sqv = reinterpret_cast<const float4*>(cm_sq + mb + cl0);
          const float4* isv = reinterpret_cast<const float4*>(cm_is + mb + cl0);
          float gsq[16], gis[16];
#pragma unroll
          for (int q4 = 0; q4 < 4; ++q4) {
            const float4 a4 = sqv[q4], b4 = isv[q4];
            gsq[4 * q4] = a4.x; gsq[4 * q4 + 1] = a4.y; gsq[4 * q4 + 2] = a4.z; gsq[4 * q4 + 3] = a4.w;
            gis[4 * q4] = b4.x; gis[4 * q4 + 1] = b4.y; gis[4 * q4 + 2] = b4.z; gis[4 * q4 + 3] = b4.w;
          }
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            dist[j] = dist_from_dot(r0[j], qis, gis[j], qq, gsq[j], p.cosine);
            const bool ok = row_ok && (col0 + j < p.ng);
            m_valid |= (ok ? 1u : 0u) << j;
            gmin = fminf(gmin, ok ? dist[j] : CUDART_INF_F);
            m_cand |= ((ok && dist[j] <= tau) ? 1u : 0u) << j;
          }
          if (p.q_pid) {
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              const bool same = cm_pid[mb + cl0 + j] == qpid;
              const bool junk = same && ((cm_mask[mb + cl0 + j] >> qcam) & 1ull);
              const bool ok = (m_valid >> j) & 1u;
              m_pos |= ((ok && same && !junk) ? 1u : 0u) << j;
              // kept rows at or before the farthest positive are counted.  A row strictly between two of the FAR_LEVELS + 1
              // farthest positives (for a query with a few far positives: almost everything that is counted) has its
              // bucket without a search -> m_far[l], one popc per chunk and level; the rest (nearer rows and distance
              // ties) take the per-row path of phase 2.
              const uint32_t kdj = float_orderable(dist[j]);
              const bool cnt = ok && !junk && npos > 0 && kdj <= tf[0];
              bool fast = false;
#pragma unroll
              for (int l = 0; l < FAR_LEVELS; ++l) {
                const bool f = cnt && kdj > tf[l + 1] && kdj < tf[l];
                m_far[l] |= (f ? 1u : 0u) << j;
                fast = fast || f;
              }
              m_cnt |= ((cnt && !fast) ? 1u : 0u) << j;
            }
          }
        }
        if (!p.cand_keys) m_cand = 0;
        if (!p.pos_keys) m_pos = 0;
        if (!p.buckets) m_cnt = 0;
        if (p.buckets) {
#pragma unroll
          for (int l = 0; l < FAR_LEVELS; ++l)
            if (m_far[l]) {  // (tf[l + 1] < kd < tf[l] needs positive npos - 1 - l to exist: the bucket index is >= 0)
              const int b = npos - 1 - l, c = __popc(m_far[l]);
              if (b < THR_MAX) atomicAdd(cnt_row + (b >> 1), (uint32_t)c << ((b & 1) * 16));
              else atomicAdd(p.buckets + (size_t)row * (p.max_pos + 1) + b, c);
            }
        }
        // ---- phase 2: full-matrix output (dense) and the rare per-element actions ----
        if (p.dist_out) {
#pragma unroll
          for (int j = 0; j < 16; ++j)
            if ((m_valid >> j) & 1u) p.dist_out[(size_t)row * p.ld_out + col0 + j] = dist[j];
        }
        // One rolled loop over the set bits (the code of the rare actions is emitted once, and a warp iterates
        // max-popcount times instead of visiting all 16 column positions).
        uint32_t m_any = m_cand | m_pos | m_cnt;
        {
#pragma unroll 1
          while (m_any) {
            const int j = __ffs(m_any) - 1;
            const uint32_t bit = 1u << j;
            m_any &= ~bit;
            const float dj = select16(dist, j);
            const unsigned int gidx = cm_idx[mb + cl0 + j];
            const unsigned long long key = make_key(dj, gidx);
            if (m_cand & bit) {
              const int slot = atomicAdd(p.cand_count + row, 1);
              if (slot < p.cand_cap) p.cand_keys[(size_t)row * p.cand_cap + slot] = key; else *p.overflow = 1;
            }
            if (m_pos & bit) {
              const int slot = atomicAdd(p.pos_count + row, 1);
              if (slot < p.max_pos) p.pos_keys[(size_t)row * p.max_pos + slot] = key; else *p.overflow = 1;
            }
            if ((m_cnt & bit) && key < maxkey) {
              // index of the first positive that sorts strictly after this gallery row
              int lo_i;
              bool exact = true;
              const uint32_t kd = (uint32_t)(key >> 32);
              if (nps == npos || kd < thr_row[nps - 1]) {
                // lo = number of staged positives whose distance is <= kd = index of the first LARGER one.  Branch-free
                // over all THR_MAX slots (unused ones hold 0xFFFFFFFF): 8 independent LDS.128 + 32 compares -- the
                // binary search this replaces was a chain of 5 dependent shared-memory loads per counted row, and with
                // ~half the gallery counted for a query with one far positive it made the count pass epilogue-bound.
                int lo = 0;
#pragma unroll
                for (int t4 = 0; t4 < THR_MAX / 4; ++t4) {
                  const uint4 v = *reinterpret_cast<const uint4*>(thr_row + 4 * t4);
                  lo += (v.x <= kd ? 1 : 0) + (v.y <= kd ? 1 : 0) + (v.z <= kd ? 1 : 0) + (v.w <= kd ? 1 : 0);
                }
                lo_i = lo;
                // a positive with the SAME distance needs the 64-bit (distance, index) comparison
                exact = lo > 0 && thr_row[lo - 1] == kd;
              }
              if (exact) lo_i = bucket_search_global(p.thr_keys + (size_t)row * p.max_pos, npos, key);
              // buckets below THR_MAX: 16-bit counters of this row in shared memory (flushed once per work item) instead
              // of one global RED per counted row (tens of millions per pass at config 3)
              if (lo_i < THR_MAX) atomicAdd(cnt_row + (lo_i >> 1), 1u << ((lo_i & 1) * 16));
              else atomicAdd(p.buckets + (size_t)row * (p.max_pos + 1) + lo_i, 1);
            }
          }
        }
        if (p.gmin && row_ok && col0 < p.ng) p.gmin[(size_t)row * p.n_groups + (col0 >> 4)] = gmin;
      }
      __syncwarp();  // this warp's staged rows are read: the next tile may overwrite them
      if (thr_in_smem) {
        named_bar_sync(2, 256);  // every warp is done with this work item's thresholds and counters
        // flush: the two threads of a row take alternate counter words of the row and leave them zero.  The next
        // work item's metadata barrier orders these writes (and the new thresholds) before any use.
        if (row_ok) {
          int* dst = p.buckets + (size_t)row * (p.max_pos + 1);
          for (int wd = chalf; wd < THR_MAX / 2; wd += 2) {
            const uint32_t v = cnt_row[wd];
            if (v) {
              cnt_row[wd] = 0u;
              if (v & 0xFFFFu) atomicAdd(dst + 2 * wd, (int)(v & 0xFFFFu));
              if (v >> 16) atomicAdd(dst + 2 * wd + 1, (int)(v >> 16));
            }
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------
// small kernels: k-th smallest group minimum, key-row sort, top-k emit, AP finalize
// ---------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void bitonic_sort_smem(T* s, int n_pow2) {
  for (int k = 2; k <= n_pow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n_pow2; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const T a = s[i], b = s[ixj];
          const bool up = (i & k) == 0;
          if ((a > b) == up) {
            s[i] = b;
            s[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  }
}

// tau[q] = k-th smallest of the (merged) group minima: an upper bound of the k-th smallest
// distance, with at most merge*GROUP_W*(k-1) rows strictly below it.
// Radix select on the order-preserving uint32 keys (4 passes of 8 bits, shared-memory histogram + warp scan): the k-th
// smallest needs no sort (a bitonic network over all n_merged keys takes 55 block-wide stages for 1024 keys).
__global__ void __launch_bounds__(256) select_tau_kernel(const float* __restrict__ gmin, int n_groups, int merge, int k,
                                                         int n_pow2, float* __restrict__ tau) {
  extern __shared__ uint32_t skeys[];
  __shared__ int hist[256];
  __shared__ int s_bucket, s_k;
  const float* g = gmin + (size_t)blockIdx.x * n_groups;
  const int n_merged = (n_groups + merge - 1) / merge;
  for (int i = threadIdx.x; i < n_merged; i += blockDim.x) {
    float m = CUDART_INF_F;
    for (int t = 0; t < merge; ++t) {
      const int gi = i * merge + t;
      if (gi < n_groups) m = fminf(m, g[gi]);
    }
    skeys[i] = float_orderable(m);
  }
  uint32_t prefix = 0, mask = 0;
  int kk = k;  // 1-based rank inside the keys that match `prefix` under `mask`
  for (int shift = 24; shift >= 0; shift -= 8) {
    hist[threadIdx.x] = 0;
    __syncthreads();  // also publishes skeys on the first pass
    for (int i = threadIdx.x; i < n_merged; i += blockDim.x) {
      const uint32_t key = skeys[i];
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1);
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      const int lane = threadIdx.x;
      int local[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        local[j] = hist[lane * 8 + j];
        sum += local[j];
      }
      int incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      const int before = incl - sum;
      if (kk > before && kk <= incl) {  // exactly one lane
        int cum = before;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (kk <= cum + local[j]) {
            s_bucket = lane * 8 + j;
            s_k = kk - cum;
            break;
          }
          cum += local[j];
        }
      }
    }
    __syncthreads();
    prefix |= (uint32_t)s_bucket << shift;
    mask |= 255u << shift;
    kk = s_k;
    __syncthreads();
  }
  if (threadIdx.x == 0) tau[blockIdx.x] = orderable_float(prefix);
}

// Tile list of a collect / threshold pass (ONE block): a tile is kept if the identity ranges of its 128 query rows and
// its 128 gallery rows intersect (it may hold a positive) or if its gallery tile index is a multiple of `keep_stride`
// (the subset of the matrix the group minima -- hence tau -- are taken from; 0: none).  Phase 1: {min, max} pid of every
// row tile into shared memory; phase 2: the kept tile ids in ascending order (block-wide prefix sums), work[0] = count.
static constexpr int WL_THREADS = 1024;
static constexpr int WL_MAX_ROW_TILES = 5632;  // int2 each: 44 KiB of shared memory

__global__ void __launch_bounds__(WL_THREADS) dist_worklist_kernel(const int* __restrict__ q_pid, int nq, int m_tiles,
                                                                   const int* __restrict__ g_pid, int ng, int n_tiles,
                                                                   int keep_stride, int* __restrict__ work) {
  extern __shared__ int2 s_rng[];  // [m_tiles + n_tiles]
  __shared__ int s_warp[WL_THREADS / 32];
  __shared__ int s_base;
  for (int t = threadIdx.x; t < m_tiles + n_tiles; t += blockDim.x) {
    const bool is_q = t < m_tiles;
    const int* pid = is_q ? q_pid : g_pid;
    const int n = is_q ? nq : ng;
    const int r0 = (is_q ? t : t - m_tiles) * BM, r1 = min(n, r0 + BM);
    int lo = INT_MAX, hi = INT_MIN;
    if (pid)
      for (int r = r0; r < r1; ++r) {
        const int v = pid[r];
        lo = min(lo, v);
        hi = max(hi, v);
      }
    s_rng[t] = make_int2(lo, hi);
  }
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  const int num_tiles = m_tiles * n_tiles;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t0 = 0; t0 < num_tiles; t0 += blockDim.x) {
    const int tile = t0 + threadIdx.x;
    int keep = 0;
    if (tile < num_tiles) {
      const int nt = tile / m_tiles, mt = tile - nt * m_tiles;  // tile id = nt * m_tiles + mt (tile_coords)
      const int2 a = s_rng[mt], b = s_rng[m_tiles + nt];
      keep = (!(b.y < a.x || b.x > a.y)) || (keep_stride > 0 && nt % keep_stride == 0);
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    int before = 0;
    for (int w2 = 0; w2 < warp; ++w2) before += s_warp[w2];
    const int base = s_base;
    if (keep) work[1 + base + before + __popc(ballot & ((1u << lane) - 1u))] = tile;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) s_base = base + before + __popc(ballot);
    __syncthreads();
  }
  if (threadIdx.x == 0) work[0] = s_base;
}

__global__ void sort_key_rows_kernel(unsigned long long* __restrict__ keys, const int* __restrict__ counts,
                                     int row_stride, int n_pow2) {
  extern __shared__ unsigned long long lkeys[];
  unsigned long long* row = keys + (size_t)blockIdx.x * row_stride;
  const int cnt = min(counts[blockIdx.x], row_stride);
  if (cnt <= 1) return;
  int np2 = 2;
  while (np2 < cnt) np2 <<= 1;  // block-uniform
  for (int i = threadIdx.x; i < np2; i += blockDim.x) lkeys[i] = (i < cnt) ? row[i] : ~0ull;
  __syncthreads();
  bitonic_sort_smem(lkeys, np2);
  for (int i = threadIdx.x; i < cnt; i += blockDim.x) row[i] = lkeys[i];
}

__global__ void topk_emit_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ counts, int cap,
                                 int k, int64_t nq, long long* __restrict__ out_idx, float* __restrict__ out_dist,
                                 int* __restrict__ overflow) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq * k) return;
  const int64_t q = i / k;
  const int j = (int)(i - q * k);
  if (j >= counts[q]) {  // cannot happen (count(<= tau) >= k by construction)
    *overflow = 2;
    out_idx[i] = -1;
    out_dist[i] = CUDART_INF_F;
    return;
  }
  const unsigned long long key = keys[(size_t)q * cap + j];
  out_idx[i] = (long long)(key & 0xFFFFFFFFull);
  out_dist[i] = orderable_float((uint32_t)(key >> 32));
}

// `packed` (optional, [nq + 1][3] doubles): per query (AP, first-hit rank, #positives) and, in the last row, the
// overflow flag -- everything the host reduction of eval_func needs, in ONE device->host copy
__global__ void eval_finalize_kernel(const int* __restrict__ buckets, const int* __restrict__ pos_count, int64_t nq,
                                     int max_pos, int* __restrict__ ranks, double* __restrict__ ap,
                                     double* __restrict__ packed, const int* __restrict__ overflow) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q == 0 && packed != nullptr) {
    packed[nq * 3] = overflow ? (double)*overflow : 0.0;
    packed[nq * 3 + 1] = packed[nq * 3 + 2] = 0.0;
  }
  if (q >= nq) return;
  const int n = min(pos_count[q], max_pos);
  const int* b = buckets + (size_t)q * (max_pos + 1);
  int* r = ranks + (size_t)q * max_pos;
  long long before = 0;
  double acc = 0.0;
  for (int j = 0; j < n; ++j) {
    before += b[j];
    const int rank = (int)before + 1;  // kept rows strictly before positive j, plus itself
    r[j] = rank;
    acc += (double)(j + 1) / (double)rank;  // utils/eval_reid.py:75-79
  }
  for (int j = n; j < max_pos; ++j) r[j] = -1;
  const double a = n > 0 ? acc / (double)n : CUDART_NAN;
  ap[q] = a;
  if (packed != nullptr) {
    packed[q * 3] = a;
    packed[q * 3 + 1] = n > 0 ? (double)r[0] : -1.0;
    packed[q * 3 + 2] = (double)pos_count[q];
  }
}

// ---------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------
static int make_plane_maps(GemmMaps* m, const PlanesView& q, int64_t nq, const PlanesView& g, int64_t ng, int32_t d) {
  const uint64_t qd[2] = {(uint64_t)d, (uint64_t)nq};
  const uint64_t gd[2] = {(uint64_t)d, (uint64_t)ng};
  const uint64_t st[2] = {2, (uint64_t)d * 2};
  const uint32_t box[2] = {BK, BM};
  int rc;
  if ((rc = encode_tensor_map(&m->q_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 2, q.hi, qd, st, box, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = encode_tensor_map(&m->q_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 2, q.lo, qd, st, box, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = encode_tensor_map(&m->g_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 2, g.hi, gd, st, box, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = encode_tensor_map(&m->g_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 2, g.lo, gd, st, box, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  return 0;
}

// rows [r0, ...) of a planes view: every plane is row-major, so the slice is a pointer offset (r0 d halves stay 16-byte
// aligned for TMA because d % 8 == 0)
static PlanesView planes_rows(const PlanesView& v, int64_t r0, int32_t d) {
  PlanesView s;
  s.hi = v.hi + (size_t)r0 * d;
  s.lo = v.lo + (size_t)r0 * d;
  s.sq = v.sq + r0;
  s.inv_scale = v.inv_scale + r0;
  return s;
}

static int launch_gemm_views(const PlanesView& q, int64_t nq, const PlanesView& g, int64_t ng, int32_t d, int32_t flags,
                             GemmPass p, cudaStream_t stream);

static int launch_gemm_pass(const void* q_planes, int64_t nq, const void* g_planes, int64_t ng, int32_t d, int32_t flags,
                            GemmPass p, cudaStream_t stream) {
  CTL_CHECK_ARG(q_planes && g_planes, "null planes");
  CTL_CHECK_ARG(nq > 0 && ng > 0 && nq < (1ll << 31) && ng < (1ll << 31), "nq/ng out of range (%lld, %lld)", (long long)nq, (long long)ng);
  CTL_CHECK_ARG(d > 0 && d % 8 == 0, "feature dim %d must be a positive multiple of 8", d);
  int rc = ctl_device_check();
  if (rc) return rc;
  return launch_gemm_views(planes_view(q_planes, nq, d), nq, planes_view(g_planes, ng, d), ng, d, flags, p, stream);
}

// Distances of rows [r0, r0 + rows) against rows [c0, c0 + cols) of ONE planes buffer of n rows, into out [rows, ld_out].
// The GEMM runs the same plan and k-order for every shape, so an element depends only on its two rows: a row block is
// bit-identical to the same rows of the full matrix (tests/test_rerank_blocked_gpu.py asserts it).
int dist_matrix_rows(const void* planes, int64_t n, int32_t d, int32_t flags, int64_t r0, int64_t rows, int64_t c0,
                     int64_t cols, float* out, int64_t ld_out, cudaStream_t stream) {
  CTL_CHECK_ARG(planes && out, "null pointer");
  CTL_CHECK_ARG(n > 0 && n < (1ll << 31) && d > 0 && d % 8 == 0, "bad planes n=%lld d=%d", (long long)n, d);
  CTL_CHECK_ARG(r0 >= 0 && rows > 0 && r0 + rows <= n && c0 >= 0 && cols > 0 && c0 + cols <= n && ld_out >= cols,
                "bad row block r0=%lld rows=%lld c0=%lld cols=%lld n=%lld ld=%lld", (long long)r0, (long long)rows,
                (long long)c0, (long long)cols, (long long)n, (long long)ld_out);
  int rc = ctl_device_check();
  if (rc) return rc;
  const PlanesView all = planes_view(planes, n, d);
  GemmPass p = {};
  p.dist_out = out;
  p.ld_out = ld_out;
  return launch_gemm_views(planes_rows(all, r0, d), rows, planes_rows(all, c0, d), cols, d, flags, p, stream);
}

static int launch_gemm_views(const PlanesView& q, int64_t nq, const PlanesView& g, int64_t ng, int32_t d, int32_t flags,
                             GemmPass p, cudaStream_t stream) {
  int rc;
  GemmMaps maps;
  if ((rc = make_plane_maps(&maps, q, nq, g, ng, d))) return rc;
  p.nq = (int)nq;
  p.ng = (int)ng;
  p.d = d;
  p.m_tiles = (int)((nq + BM - 1) / BM);
  p.n_tiles = (int)((ng + BN - 1) / BN);
  p.cosine = flags & (CTL_DIST_COSINE | CTL_DIST_SQRT);
  p.q_sq = q.sq;
  p.q_is = q.inv_scale;
  p.g_sq = g.sq;
  p.g_is = g.inv_scale;
  static bool attr_set = false;
  if (!attr_set) {
    CTL_CUDA(cudaFuncSetAttribute(dist_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GEMM_SMEM));
    attr_set = true;
  }
  const long long items = (long long)p.m_tiles * p.n_tiles;
  const int grid = (int)std::min<long long>(items, sm_count());
  dist_gemm_kernel<<<grid, GEMM_THREADS, GEMM_SMEM, stream>>>(maps, p);
  CTL_LAUNCH_CHECK();
  return 0;
}

__global__ void fill_f32_kernel(float* p, int64_t n, float v) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

static constexpr int SORT_MAX = 16384;  // keys per row the smem bitonic sort accepts

static int sort_rows(unsigned long long* keys, const int* counts, int64_t rows, int row_stride, cudaStream_t stream) {
  if (row_stride > SORT_MAX) {
    set_error("key rows of %d entries exceed the sort capacity %d", row_stride, SORT_MAX);
    return CTL_ERR_UNSUPPORTED;
  }
  static bool attr_set = false;
  if (!attr_set) {
    CTL_CUDA(cudaFuncSetAttribute(sort_key_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SORT_MAX * 8));
    attr_set = true;
  }
  int np2 = 2;
  while (np2 < row_stride) np2 <<= 1;
  // 256 threads whatever the capacity: the rows are mostly short (config 3: ~130 of 4096 candidate slots used) and the
  // bitonic network is barrier-bound -- 1024-thread blocks spent 70 us per launch synchronising idle warps
  const int threads = np2 >= 512 ? 256 : 64;
  sort_key_rows_kernel<<<(unsigned)rows, threads, (size_t)np2 * 8, stream>>>(keys, counts, row_stride, np2);
  CTL_LAUNCH_CHECK();
  return 0;
}

static int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

static constexpr long long WORK_MAX_TILES = 1 << 20;  // beyond this the single-block list builder is not worth it
static size_t worklist_ints(int64_t nq, int64_t ng) {
  const long long tiles = ((nq + BM - 1) / BM) * ((ng + BN - 1) / BN);
  return (size_t)std::min<long long>(tiles, WORK_MAX_TILES) + 1;
}
// every `stride`-th gallery tile leaves >= ~2.5 k merged groups for the k-th smallest group minimum
static int subset_stride(int n_tiles, int merge, int k) {
  if (merge > 1) return 1;  // merged groups span tiles (galleries > 131 072 rows): keep every tile
  const long long groups_per_tile = BN / GROUP_W;
  const long long want = (5LL * k + 1) / 2;
  const long long tiles_needed = (want + groups_per_tile - 1) / groups_per_tile;
  return (int)std::max<long long>(1, n_tiles / std::max<long long>(1, tiles_needed));
}
static int launch_worklist(const int* q_pid, int64_t nq, const int* g_pid, int64_t ng, int keep_stride, int* work, cudaStream_t stream) {
  const int m_tiles = (int)((nq + BM - 1) / BM), n_tiles = (int)((ng + BN - 1) / BN);
  if ((long long)m_tiles * n_tiles > WORK_MAX_TILES || m_tiles + n_tiles > WL_MAX_ROW_TILES) {
    set_error("tile list: %d x %d tiles exceed the list builder (run the pass without a list)", m_tiles, n_tiles);
    return CTL_ERR_UNSUPPORTED;
  }
  const size_t smem = (size_t)(m_tiles + n_tiles) * sizeof(int2);
  static bool attr_set = false;
  if (!attr_set) {
    CTL_CUDA(cudaFuncSetAttribute(dist_worklist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(WL_MAX_ROW_TILES * sizeof(int2))));
    attr_set = true;
  }
  dist_worklist_kernel<<<1, WL_THREADS, smem, stream>>>(q_pid, (int)nq, m_tiles, g_pid, (int)ng, n_tiles, keep_stride, work);
  CTL_LAUNCH_CHECK();
  return 0;
}

struct TopkPlan {
  bool emit_all;
  int n_groups;   // GROUP_W-wide groups
  int merge;      // groups merged per selection slot
  int cap;        // candidate capacity per query
};
static constexpr int EMIT_ALL_MAX = 4096;
static constexpr int SELECT_MAX = 8192;
static constexpr int CAP_MAX = SORT_MAX;

static int plan_topk(int64_t ng, int k, TopkPlan* pl) {
  pl->n_groups = (int)((ng + GROUP_W - 1) / GROUP_W);
  if (ng <= EMIT_ALL_MAX) {
    pl->emit_all = true;
    pl->merge = 1;
    pl->cap = next_pow2((int)ng);
    return 0;
  }
  pl->emit_all = false;
  pl->merge = (pl->n_groups + SELECT_MAX - 1) / SELECT_MAX;
  const int n_merged = (pl->n_groups + pl->merge - 1) / pl->merge;
  if (n_merged < k) {
    set_error("k=%d needs at least k column groups (have %d); use ctl_dist_matrix for k this large", k, n_merged);
    return CTL_ERR_UNSUPPORTED;
  }
  long long cap = (long long)pl->merge * GROUP_W * (k - 1) + 512;  // strict bound + room for ties at tau
  cap = next_pow2((int)std::min<long long>(cap, (long long)ng));
  if (cap > CAP_MAX) {
    set_error("top-k candidate capacity %lld exceeds %d (k=%d, ng=%lld)", cap, CAP_MAX, k, (long long)ng);
    return CTL_ERR_UNSUPPORTED;
  }
  pl->cap = (int)cap;
  return 0;
}

}  // namespace ctl

using namespace ctl;

extern "C" {

size_t ctl_planes_bytes(int64_t n, int32_t d) { return planes_total(n, d); }

int ctl_planes_build(const float* x, int64_t n, int32_t d, int32_t flags, void* planes, ctl_stream_t stream) {
  CTL_CHECK_ARG(x && planes, "null pointer");
  CTL_CHECK_ARG(n > 0 && d > 0 && d % 8 == 0, "bad shape n=%lld d=%d (d must be a multiple of 8)", (long long)n, d);
  int rc = ctl_device_check();
  if (rc) return rc;
  char* c = static_cast<char*>(planes);
  const int n_norm = ((flags & CTL_FLAG_NORMALIZE) ? 1 : 0) + ((flags & CTL_DIST_COSINE) ? 1 : 0);
  planes_build_kernel<<<(unsigned)((n + 3) / 4), 128, 0, (cudaStream_t)stream>>>(
      x, n, d, n_norm, reinterpret_cast<__half*>(c), reinterpret_cast<__half*>(c + planes_off_lo(n, d)),
      reinterpret_cast<float*>(c + planes_off_sq(n, d)), reinterpret_cast<float*>(c + planes_off_is(n, d)));
  CTL_LAUNCH_CHECK();
  return 0;
}

int ctl_dist_matrix(const void* q_planes, int64_t nq, const void* g_planes, int64_t ng, int32_t d, int32_t flags,
                    float* out, int64_t ld_out, ctl_stream_t stream) {
  CTL_CHECK_ARG(out && ld_out >= ng, "bad output (ld_out=%lld, ng=%lld)", (long long)ld_out, (long long)ng);
  GemmPass p = {};
  p.dist_out = out;
  p.ld_out = ld_out;
  return launch_gemm_pass(q_planes, nq, g_planes, ng, d, flags, p, (cudaStream_t)stream);
}

int ctl_sort_key_rows(uint64_t* keys, const int32_t* counts, int64_t rows, int32_t row_stride, ctl_stream_t stream) {
  CTL_CHECK_ARG(keys && counts && rows > 0 && row_stride > 0, "bad arguments");
  int rc = ctl_device_check();
  if (rc) return rc;
  return sort_rows(reinterpret_cast<unsigned long long*>(keys), counts, rows, row_stride, (cudaStream_t)stream);
}

int ctl_eval_finalize_packed(const int32_t* buckets, const int32_t* pos_count, int64_t nq, int32_t max_pos, int32_t* ranks,
                             double* ap, double* packed, const int32_t* overflow, ctl_stream_t stream) {
  CTL_CHECK_ARG(buckets && pos_count && ranks && ap && nq > 0 && max_pos >= 1, "bad arguments");
  int rc = ctl_device_check();
  if (rc) return rc;
  eval_finalize_kernel<<<(unsigned)((nq + 127) / 128), 128, 0, (cudaStream_t)stream>>>(buckets, pos_count, nq, max_pos,
                                                                                       ranks, ap, packed, overflow);
  CTL_LAUNCH_CHECK();
  return 0;
}

int ctl_dist_pass(const void* q_planes, int64_t nq, const void* g_planes, int64_t ng, int32_t d, int32_t flags,
                  const ctl_pass_desc* desc, ctl_stream_t stream) {
  CTL_CHECK_ARG(desc != nullptr, "null pass descriptor");
  const ctl_pass_desc& e = *desc;
  GemmPass p = {};
  p.dist_out = e.dist_out;
  p.ld_out = e.ld_out;
  CTL_CHECK_ARG(!e.dist_out || e.ld_out >= ng, "ld_out too small");
  p.gmin = e.gmin;
  p.n_groups = (int)((ng + GROUP_W - 1) / GROUP_W);
  p.tau = e.tau;
  p.cand_keys = reinterpret_cast<unsigned long long*>(e.cand_keys);
  p.cand_count = e.cand_count;
  p.cand_cap = e.cand_cap;
  CTL_CHECK_ARG(!e.cand_keys || (e.tau && e.cand_count && e.cand_cap > 0 && e.overflow), "candidate output needs tau, counts, capacity, overflow");
  p.q_pid = e.q_pid;
  p.q_cam = e.q_cam;
  p.g_pid = e.g_pid;
  p.g_mask = reinterpret_cast<const unsigned long long*>(e.g_cammask);
  CTL_CHECK_ARG(!(e.pos_keys || e.buckets) || (e.q_pid && e.q_cam && e.g_pid && e.g_cammask && e.max_pos >= 1),
                "evaluation epilogues need the identity arrays and max_pos");
  p.pos_keys = reinterpret_cast<unsigned long long*>(e.pos_keys);
  p.pos_count = e.pos_count;
  CTL_CHECK_ARG(!e.pos_keys || (e.pos_count && e.overflow), "collect needs pos_count and overflow");
  p.max_pos = e.max_pos;
  p.thr_keys = reinterpret_cast<const unsigned long long*>(e.thr_keys);
  p.thr_count = e.thr_count;
  p.buckets = e.buckets;
  CTL_CHECK_ARG(!e.buckets || (e.thr_keys && e.thr_count), "count needs the sorted positives");
  p.overflow = e.overflow;
  p.g_off = e.g_index_offset;
  CTL_CHECK_ARG(e.g_index_offset >= 0 && e.g_index_offset + ng < (1ll << 32), "gallery index out of uint32 range");
  CTL_CHECK_ARG(!e.tile_list || !(e.dist_out || e.cand_keys || e.buckets),
                "a tile list drops tiles: not for the full matrix, the candidates or the bucket counts");
  p.work = e.tile_list;
  p.g_map = e.g_index_map;
  if (!p.pos_keys && !p.buckets) p.q_pid = nullptr;  // identities unused
  return launch_gemm_pass(q_planes, nq, g_planes, ng, d, flags, p, (cudaStream_t)stream);
}

int ctl_topk_plan(int64_t ng, int32_t k, int32_t* emit_all, int32_t* n_groups, int32_t* merge, int32_t* cand_cap) {
  CTL_CHECK_ARG(emit_all && n_groups && merge && cand_cap && k >= 1 && k <= ng, "bad arguments (k=%d ng=%lld)", k, (long long)ng);
  TopkPlan pl;
  int rc = plan_topk(ng, k, &pl);
  if (rc) return rc;
  *emit_all = pl.emit_all ? 1 : 0;
  *n_groups = pl.n_groups;
  *merge = pl.merge;
  *cand_cap = pl.cap;
  return 0;
}

int ctl_select_tau(const float* gmin, int64_t nq, int32_t n_groups, int32_t merge, int32_t k, float* tau,
                   ctl_stream_t stream) {
  CTL_CHECK_ARG(gmin && tau && nq > 0 && n_groups > 0 && merge >= 1 && k >= 1, "bad arguments");
  const int n_merged = (n_groups + merge - 1) / merge;
  CTL_CHECK_ARG(n_merged >= k && n_merged <= SELECT_MAX, "need k <= merged groups <= %d (have %d)", SELECT_MAX, n_merged);
  int rc = ctl_device_check();
  if (rc) return rc;
  const int np2 = next_pow2(n_merged);
  select_tau_kernel<<<(unsigned)nq, 256, np2 * sizeof(uint32_t), (cudaStream_t)stream>>>(gmin, n_groups, merge, k, np2, tau);
  CTL_LAUNCH_CHECK();
  return 0;
}

size_t ctl_dist_worklist_bytes(int64_t nq, int64_t ng) {
  if (nq < 1 || ng < 1) return 0;
  return worklist_ints(nq, ng) * sizeof(int);
}

int ctl_dist_subset_stride(int64_t ng, int32_t k) {
  TopkPlan pl;
  if (ng < 1 || k < 1 || k > ng || plan_topk(ng, k, &pl) || pl.emit_all) return 1;
  return subset_stride((int)((ng + BN - 1) / BN), pl.merge, k);
}

int ctl_dist_worklist(const int32_t* q_pid, int64_t nq, const int32_t* g_pid, int64_t ng, int32_t keep_stride, int32_t* tile_list,
                      ctl_stream_t stream) {
  CTL_CHECK_ARG(tile_list && nq > 0 && ng > 0 && nq < (1ll << 31) && ng < (1ll << 31) && keep_stride >= 0, "bad arguments");
  CTL_CHECK_ARG((q_pid == nullptr) == (g_pid == nullptr), "q_pid and g_pid come together");
  CTL_CHECK_ARG(q_pid || keep_stride > 0, "an empty selection: give identities and / or a stride");
  int rc = ctl_device_check();
  if (rc) return rc;
  return launch_worklist(q_pid, nq, g_pid, ng, keep_stride, tile_list, (cudaStream_t)stream);
}

int ctl_fill_f32(float* p, int64_t n, float value, ctl_stream_t stream) {
  CTL_CHECK_ARG(p && n > 0, "bad arguments");
  int rc = ctl_device_check();
  if (rc) return rc;
  fill_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p, n, value);
  CTL_LAUNCH_CHECK();
  return 0;
}

int ctl_topk_emit(const uint64_t* cand_keys_sorted, const int32_t* cand_count, int64_t nq, int32_t cand_cap, int32_t k,
                  int64_t* out_idx, float* out_dist, int32_t* overflow, ctl_stream_t stream) {
  CTL_CHECK_ARG(cand_keys_sorted && cand_count && out_idx && out_dist && overflow && nq > 0 && k >= 1 && k <= cand_cap, "bad arguments");
  int rc = ctl_device_check();
  if (rc) return rc;
  const int64_t total = nq * k;
  topk_emit_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const unsigned long long*>(cand_keys_sorted), cand_count, cand_cap, k, nq, (long long*)out_idx,
      out_dist, overflow);
  CTL_LAUNCH_CHECK();
  return 0;
}

uint64_t ctl_key_encode(float dist, uint32_t index) { return make_key(dist, index); }
void ctl_key_decode(uint64_t key, float* dist, uint32_t* index) {
  if (dist) *dist = orderable_float((uint32_t)(key >> 32));
  if (index) *index = (uint32_t)(key & 0xFFFFFFFFull);
}

}  // extern "C"
