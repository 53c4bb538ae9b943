// k-reciprocal re-ranking (Zhong, Zheng, Cao, Li, CVPR 2017) of a query x gallery problem, and CMC / mAP passes over a
// materialised distance matrix.
//
// Replaces the re_ranking(probFea, galFea, k1, k2, lambda_value) function of the reid-strong-baseline lineage that the
// reference's utils/reid_metric.py credits (the CTL reference dropped it), and -- for matrices the caller computed -- the
// per-query loop of utils/eval_reid.py:25-92.  Semantics: include/ctl_b200.h, DESIGN.md section 4.
//
// Pipeline over F = [q; g], N = Q + G rows (one stream, no host synchronisation, no data-dependent allocation):
//   D      = ctl_dist_matrix(F, F)                 [N, N] fp32, squared euclidean, unclamped
//   rank   : nd = D / rowmax (in place), rank[i, :kr] = first kr columns by (nd, column)   one CTA per row
//   expand : E(i) = R(i) + every R_h(c), c in R(i), with |R_h(c) & R(i)| > 2/3 |R_h(c)|;
//            V[i, E(i)] = softmax(-nd[i, E(i)])                                           one warp per row
//   qe     : V[i] <- mean_{t < k2} V[rank[i, t]]                                          one CTA per row
//   invert : CSC of the gallery rows of V (column -> gallery rows, values)
//   jaccard: out[i, j] = (1 - lambda) (1 - s / (2 - s)) + lambda nd[i, Q + j], s = sum_c min(V[i, c], V[Q + j, c])
// V rows are row-padded (index, value) lists in ascending column order, capacities fixed by (k1, k2): see plan_rerank.
// ctl_rerank_topk runs the same kernels over [block_rows, N] row blocks of D (rank, then expand in a second sweep, then
// Jaccard + top-k per query block), so only a block of the matrix is alive, with bit-identical results.
#include <limits.h>
#include <math_constants.h>
#include <math.h>

#include <algorithm>

#include "common.h"

namespace ctl {
namespace {

constexpr int KR_MAX = 128;         // rank columns kept per row: max(k1 + 1, k2)
constexpr int RK_THREADS = 256;
constexpr int EX_WARPS = 4;         // rows per CTA of the expansion kernel
constexpr int EX_BUF_MAX = 8192;    // expansion candidates per row (pow2 of (k1 + 1)(h + 2))
constexpr int QE_MAX = 16384;       // query-expansion entries per row (pow2 of k2 (k1 + 1)(h + 2))
constexpr int QE_THREADS = 256;
constexpr int JC_THREADS = 256;
constexpr int JC_TILE = 16384;      // gallery rows per Jaccard CTA (64 KiB accumulator)
constexpr int EM_THREADS = 256;
constexpr int EM_HIST_MAX = 8192;   // bucket counters of a row held in shared memory by the count pass

__device__ __forceinline__ uint32_t f2ord(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ unsigned long long key_of(float d, uint32_t idx) {
  return (static_cast<unsigned long long>(f2ord(d)) << 32) | idx;
}
__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float wmax(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
int pow2_at_least(long long v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

template <typename T>
__device__ void block_bitonic(T* s, int n_pow2) {
  for (int k = 2; k <= n_pow2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n_pow2; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const T a = s[i], b = s[ixj];
          if ((a > b) == ((i & k) == 0)) {
            s[i] = b;
            s[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
}

__device__ void warp_bitonic(int* s, int n_pow2) {
  const int lane = threadIdx.x & 31;
  for (int k = 2; k <= n_pow2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < n_pow2; i += 32) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const int a = s[i], b = s[ixj];
          if ((a > b) == ((i & k) == 0)) {
            s[i] = b;
            s[ixj] = a;
          }
        }
      }
      __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------
// steps 2 + 3: nd = D / rowmax in place, rank[i, :kr] by (nd, column)
// ---------------------------------------------------------------------------------------
// The kr-th smallest orderable key comes from a 4 x 8-bit radix select; the selected set is every key below it plus the
// first ties in column order (a block-wide ordered scan), so exactly min(kr, n) entries, sorted as (value, column) keys.
// One CTA per row of a [rows, ld] block (the whole matrix, or a row block of it: rank / rowmax point at the block's
// first row).
//   NORMALISE: row maximum (exact, so independent of the block) -> rowmax (when given), nd = D / max in place, rank;
//   otherwise: the first kr columns of the row as it is -> out_idx (int64) / out_dist, the top-k of the final distances.
__device__ __forceinline__ float normalise_nd(float v, float mx) { return __fadd_rn(__fdiv_rn(v, mx), 0.f); }  // no -0

template <bool NORMALISE>
__global__ void __launch_bounds__(RK_THREADS) rerank_rank_kernel(float* __restrict__ d, int n, long long ld, int kr,
                                                                 int* __restrict__ rank, float* __restrict__ rowmax,
                                                                 int* __restrict__ status, long long* __restrict__ out_idx,
                                                                 float* __restrict__ out_dist) {
  __shared__ float s_red[RK_THREADS / 32];
  __shared__ int hist[256];
  __shared__ int s_bucket, s_k, s_cnt, s_eq;
  __shared__ int s_warp[RK_THREADS / 32];
  __shared__ unsigned long long s_keys[KR_MAX];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float* r = d + (size_t)blockIdx.x * ld;
  if (NORMALISE) {
    float mx = -CUDART_INF_F;
    for (int j = tid; j < n; j += RK_THREADS) mx = fmaxf(mx, r[j]);
    mx = wmax(mx);
    if (lane == 0) s_red[warp] = mx;
    __syncthreads();
    mx = s_red[0];
    for (int w = 1; w < RK_THREADS / 32; ++w) mx = fmaxf(mx, s_red[w]);
    if (!(mx > 0.f) && tid == 0) atomicOr(status, 1);
    for (int j = tid; j < n; j += RK_THREADS) r[j] = normalise_nd(r[j], mx);
    __syncthreads();  // the row is re-read by other threads of the block
  }

  const int k = min(kr, n);
  uint32_t prefix = 0, mask = 0;
  int kk = k;  // 1-based rank among the keys matching `prefix` under `mask`
  for (int shift = 24; shift >= 0; shift -= 8) {
    hist[tid] = 0;
    __syncthreads();
    for (int j = tid; j < n; j += RK_THREADS) {
      const uint32_t u = f2ord(r[j]);
      if ((u & mask) == prefix) atomicAdd(&hist[(u >> shift) & 255u], 1);
    }
    __syncthreads();
    if (tid < 32) {
      int local[8], sum = 0;
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        local[t] = hist[lane * 8 + t];
        sum += local[t];
      }
      int incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      const int before = incl - sum;
      if (kk > before && kk <= incl) {
        int cum = before;
        for (int t = 0; t < 8; ++t) {
          if (kk <= cum + local[t]) {
            s_bucket = lane * 8 + t;
            s_k = kk - cum;
            break;
          }
          cum += local[t];
        }
      }
    }
    __syncthreads();
    prefix |= (uint32_t)s_bucket << shift;
    mask |= 255u << shift;
    kk = s_k;
    __syncthreads();
  }
  // keys < prefix: k - kk of them; keys == prefix: the first kk in column order
  if (tid == 0) {
    s_cnt = 0;
    s_eq = 0;
  }
  __syncthreads();
  for (int j0 = 0; j0 < n; j0 += RK_THREADS) {
    const int j = j0 + tid;
    const uint32_t u = j < n ? f2ord(r[j]) : 0xFFFFFFFFu;
    const bool eq = j < n && u == prefix;
    const unsigned b = __ballot_sync(0xffffffffu, eq);
    if (lane == 0) s_warp[warp] = __popc(b);
    __syncthreads();
    int before = s_eq;
    for (int w = 0; w < warp; ++w) before += s_warp[w];
    const int eq_rank = before + __popc(b & ((1u << lane) - 1u));
    if (j < n && (u < prefix || (eq && eq_rank < kk))) s_keys[atomicAdd(&s_cnt, 1)] = ((unsigned long long)u << 32) | (uint32_t)j;
    __syncthreads();
    if (tid == 0)
      for (int w = 0; w < RK_THREADS / 32; ++w) s_eq += s_warp[w];
    __syncthreads();
  }
  for (int t = k + tid; t < KR_MAX; t += RK_THREADS) s_keys[t] = ~0ull;
  __syncthreads();
  block_bitonic(s_keys, KR_MAX);
  if (NORMALISE) {
    for (int t = tid; t < kr; t += RK_THREADS)
      rank[(size_t)blockIdx.x * kr + t] = t < k ? (int)(uint32_t)(s_keys[t] & 0xFFFFFFFFull) : -1;
    if (rowmax && tid == 0) {  // the maximum again from s_red (kept out of the select's registers)
      float mx = s_red[0];
      for (int w = 1; w < RK_THREADS / 32; ++w) mx = fmaxf(mx, s_red[w]);
      rowmax[blockIdx.x] = mx;
    }
  } else {  // kr <= n (checked by the host): every slot holds a column
    for (int t = tid; t < kr; t += RK_THREADS) {
      const int j = (int)(uint32_t)(s_keys[t] & 0xFFFFFFFFull);
      out_idx[(size_t)blockIdx.x * kr + t] = j;
      out_dist[(size_t)blockIdx.x * kr + t] = r[j];
    }
  }
}

// nd = D / rowmax of a [rows, cols] block whose row maxima were stored by the NORMALISE rank sweep: the same division
// as that sweep, so the block equals the same rows (and columns) of the dense nd bit for bit
__global__ void rerank_normalise_kernel(float* __restrict__ d, int cols, long long ld, const float* __restrict__ rowmax) {
  float* r = d + (size_t)blockIdx.x * ld;
  const float mx = rowmax[blockIdx.x];
  for (int j = blockIdx.y * blockDim.x + threadIdx.x; j < cols; j += gridDim.y * blockDim.x) r[j] = normalise_nd(r[j], mx);
}

// ---------------------------------------------------------------------------------------
// step 4: k-reciprocal sets, expansion, weights -- one warp per row
// ---------------------------------------------------------------------------------------
// Shared memory per warp: buf[buf_pow2] (candidates, then the sorted unique set), R[KR_MAX], T[KR_MAX].
// Rows r0 .. r0 + rows - 1 of the n: the global row i indexes rank and V, the local row i - r0 the nd block.
__global__ void __launch_bounds__(EX_WARPS * 32) rerank_expand_kernel(const float* __restrict__ nd, int n, long long ld,
                                                                      int r0, int rows,
                                                                      const int* __restrict__ rank, int kr, int k1, int h,
                                                                      int* __restrict__ v_idx, float* __restrict__ v_val,
                                                                      int* __restrict__ v_cnt, int v_cap, int buf_pow2) {
  extern __shared__ int ex_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int local = blockIdx.x * EX_WARPS + warp;
  if (local >= rows) return;  // warp-uniform; no block-wide barrier below
  const int i = r0 + local;
  int* buf = ex_smem + warp * (buf_pow2 + 2 * KR_MAX);
  int* R = buf + buf_pow2;
  int* T = R + KR_MAX;
  const unsigned below = (1u << lane) - 1u;
  const int nf = min(k1 + 1, n), nh = min(h + 1, n);
  const int* ri = rank + (size_t)i * kr;
  // R(i): forward neighbours j of i that have i among their own nf nearest (forward order kept)
  int nR = 0;
  for (int t0 = 0; t0 < nf; t0 += 32) {
    const int t = t0 + lane;
    bool rec = false;
    int j = -1;
    if (t < nf) {
      j = ri[t];
      const int* rj = rank + (size_t)j * kr;
      for (int u = 0; u < nf; ++u) rec |= rj[u] == i;
    }
    const unsigned b = __ballot_sync(0xffffffffu, rec);
    if (rec) R[nR + __popc(b & below)] = j;
    nR += __popc(b);
  }
  __syncwarp();
  for (int t = lane; t < nR; t += 32) buf[t] = R[t];
  int nb = nR;
  for (int ci = 0; ci < nR; ++ci) {
    const int c = R[ci];
    const int* rc = rank + (size_t)c * kr;
    int len = 0, inter = 0;
    for (int f0 = 0; f0 < nh; f0 += 32) {
      const int f = f0 + lane;
      bool rec = false, in_r = false;
      int m = -1;
      if (f < nh) {
        m = rc[f];
        const int* rm = rank + (size_t)m * kr;
        for (int u = 0; u < nh; ++u) rec |= rm[u] == c;
        if (rec)
          for (int u = 0; u < nR; ++u) in_r |= R[u] == m;
      }
      const unsigned b = __ballot_sync(0xffffffffu, rec);
      if (rec) T[len + __popc(b & below)] = m;
      len += __popc(b);
      inter += __popc(__ballot_sync(0xffffffffu, in_r));
    }
    __syncwarp();
    if (3 * inter > 2 * len) {  // |R_h(c) & R(i)| > 2/3 |R_h(c)|, in integers
      for (int t = lane; t < len; t += 32) buf[nb + t] = T[t];
      nb += len;
    }
    __syncwarp();
  }
  for (int t = nb + lane; t < buf_pow2; t += 32) buf[t] = INT_MAX;
  __syncwarp();
  warp_bitonic(buf, buf_pow2);
  // unique, compacted in place (writes never pass the chunk being read)
  int ne = 0, prev = -1;
  for (int t0 = 0; t0 < nb; t0 += 32) {
    const int t = t0 + lane;
    const int v = t < nb ? buf[t] : INT_MAX;
    int left = __shfl_up_sync(0xffffffffu, v, 1);
    if (lane == 0) left = prev;
    const bool keep = t < nb && v != left;
    const unsigned b = __ballot_sync(0xffffffffu, keep);
    prev = __shfl_sync(0xffffffffu, v, 31);
    __syncwarp();
    if (keep) buf[ne + __popc(b & below)] = v;
    ne += __popc(b);
    __syncwarp();
  }
  const float* ndi = nd + (size_t)local * ld;
  float s = 0.f;
  for (int t = lane; t < ne; t += 32) s += expf(-ndi[buf[t]]);
  s = wsum(s);
  for (int t = lane; t < ne; t += 32) {
    v_idx[(size_t)i * v_cap + t] = buf[t];
    v_val[(size_t)i * v_cap + t] = __fdiv_rn(expf(-ndi[buf[t]]), s);
  }
  if (lane == 0) v_cnt[i] = ne;
}

// ---------------------------------------------------------------------------------------
// step 5: query expansion -- one CTA per row: the (column, source) keys of the k2 source rows, sorted; each column's
// values summed in source order and divided by the number of sources
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(QE_THREADS) rerank_qe_kernel(const int* __restrict__ rank, int n, int kr, int k2,
                                                               const int* __restrict__ v_idx, const float* __restrict__ v_val,
                                                               const int* __restrict__ v_cnt, int v_cap,
                                                               int* __restrict__ q_idx, float* __restrict__ q_val,
                                                               int* __restrict__ q_cnt, int q_cap) {
  extern __shared__ unsigned long long qk[];
  __shared__ int s_off[KR_MAX + 1], s_row[KR_MAX], s_warp[QE_THREADS / 32];
  const int i = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int m = min(k2, n);
  if (tid == 0) {
    int off = 0;
    for (int t = 0; t < m; ++t) {
      const int r = rank[(size_t)i * kr + t];
      s_row[t] = r;
      s_off[t] = off;
      off += v_cnt[r];
    }
    s_off[m] = off;
  }
  __syncthreads();
  const int total = s_off[m];
  for (int t = 0; t < m; ++t) {
    const int r = s_row[t], c = s_off[t + 1] - s_off[t];
    for (int e = tid; e < c; e += QE_THREADS)
      qk[s_off[t] + e] = ((unsigned long long)(uint32_t)v_idx[(size_t)r * v_cap + e] << 32) | (uint32_t)(t * v_cap + e);
  }
  int p2 = 2;
  while (p2 < total) p2 <<= 1;
  for (int t = total + tid; t < p2; t += QE_THREADS) qk[t] = ~0ull;
  __syncthreads();
  block_bitonic(qk, p2);
  const float m_f = (float)m;
  int base = 0;
  for (int p0 = 0; p0 < total; p0 += QE_THREADS) {
    const int p = p0 + tid;
    const uint32_t col = p < total ? (uint32_t)(qk[p] >> 32) : 0u;
    const bool head = p < total && (p == 0 || (uint32_t)(qk[p - 1] >> 32) != col);
    const unsigned b = __ballot_sync(0xffffffffu, head);
    if (lane == 0) s_warp[warp] = __popc(b);
    __syncthreads();
    int before = base;
    for (int w = 0; w < warp; ++w) before += s_warp[w];
    if (head) {
      float s = 0.f;
      for (int q = p; q < total && (uint32_t)(qk[q] >> 32) == col; ++q) {
        const uint32_t src = (uint32_t)(qk[q] & 0xFFFFFFFFull);
        const int t = (int)(src / (uint32_t)v_cap), e = (int)(src % (uint32_t)v_cap);
        s += v_val[(size_t)s_row[t] * v_cap + e];
      }
      const int slot = before + __popc(b & ((1u << lane) - 1u));
      q_idx[(size_t)i * q_cap + slot] = (int)col;
      q_val[(size_t)i * q_cap + slot] = __fdiv_rn(s, m_f);
    }
    for (int w = 0; w < QE_THREADS / 32; ++w) base += s_warp[w];
    __syncthreads();
  }
  if (tid == 0) q_cnt[i] = base;
}

// ---------------------------------------------------------------------------------------
// inverted index of the gallery rows of V: col_ptr[N + 1], inv_row (gallery-local row), inv_val
// ---------------------------------------------------------------------------------------
__global__ void rerank_colcount_kernel(const int* __restrict__ idx, const int* __restrict__ cnt, int cap, int nq, int ng,
                                       int* __restrict__ colcnt) {
  const int j = blockIdx.x;  // gallery row
  const int r = nq + j;
  const int c = cnt[r];
  for (int e = threadIdx.x; e < c; e += blockDim.x) atomicAdd(colcnt + idx[(size_t)r * cap + e], 1);
}

// single CTA: exclusive scan of colcnt[n] -> col_ptr[n + 1]; cursor[c] = col_ptr[c] (cursor may be colcnt itself: each
// thread reads an entry of its own range before it overwrites it)
__global__ void __launch_bounds__(1024) rerank_colscan_kernel(const int* colcnt, int n, int* __restrict__ col_ptr,
                                                              int* cursor) {
  __shared__ int s_part[1024];
  const int tid = threadIdx.x;
  const int per = (n + 1023) / 1024;
  const int lo = min(n, tid * per), hi = min(n, lo + per);
  int sum = 0;
  for (int c = lo; c < hi; ++c) sum += colcnt[c];
  s_part[tid] = sum;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const int v = tid >= o ? s_part[tid - o] : 0;
    __syncthreads();
    s_part[tid] += v;
    __syncthreads();
  }
  int run = s_part[tid] - sum;
  for (int c = lo; c < hi; ++c) {
    const int v = colcnt[c];
    col_ptr[c] = run;
    cursor[c] = run;
    run += v;
  }
  if (tid == 1023) col_ptr[n] = s_part[1023];
}

__global__ void rerank_colfill_kernel(const int* __restrict__ idx, const float* __restrict__ val, const int* __restrict__ cnt,
                                      int cap, int nq, int* __restrict__ cursor, int* __restrict__ inv_row,
                                      float* __restrict__ inv_val) {
  const int j = blockIdx.x;
  const int r = nq + j;
  const int c = cnt[r];
  for (int e = threadIdx.x; e < c; e += blockDim.x) {
    const int pos = atomicAdd(cursor + idx[(size_t)r * cap + e], 1);
    inv_row[pos] = j;
    inv_val[pos] = val[(size_t)r * cap + e];
  }
}

// ---------------------------------------------------------------------------------------
// step 6: Jaccard + blend.  CTA (query i, gallery tile y).  The query's columns are walked in ascending order; inside one
// column every gallery row is distinct, so the shared-memory adds of one column need no atomics, and the barrier after
// each column fixes the accumulation order of every gallery row (ascending column).
// CTA x handles query q0 + x (its V row), and row x of nd (gallery columns from nd_col0) and of out.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(JC_THREADS) rerank_jaccard_kernel(int q0, int nd_col0, int ng, const int* __restrict__ q_idx,
                                                                    const float* __restrict__ q_val,
                                                                    const int* __restrict__ q_cnt, int q_cap,
                                                                    const int* __restrict__ col_ptr,
                                                                    const int* __restrict__ inv_row,
                                                                    const float* __restrict__ inv_val,
                                                                    const float* __restrict__ nd, long long ld_nd,
                                                                    float lambda, float* __restrict__ out,
                                                                    long long ld_out, int tile) {
  extern __shared__ float acc[];
  __shared__ int s_lo[JC_THREADS], s_hi[JC_THREADS];
  __shared__ float s_v[JC_THREADS];
  const int i = q0 + blockIdx.x, tid = threadIdx.x;
  const int t0 = blockIdx.y * tile, tw = min(tile, ng - t0);
  for (int t = tid; t < tw; t += JC_THREADS) acc[t] = 0.f;
  const int cnt = q_cnt[i];
  for (int e0 = 0; e0 < cnt; e0 += JC_THREADS) {
    __syncthreads();  // the previous chunk's columns are consumed
    if (e0 + tid < cnt) {
      const int c = q_idx[(size_t)i * q_cap + e0 + tid];
      s_v[tid] = q_val[(size_t)i * q_cap + e0 + tid];
      s_lo[tid] = col_ptr[c];
      s_hi[tid] = col_ptr[c + 1];
    }
    __syncthreads();
    const int ce = min(JC_THREADS, cnt - e0);
    for (int e = 0; e < ce; ++e) {
      const float v = s_v[e];
      for (int p = s_lo[e] + tid; p < s_hi[e]; p += JC_THREADS) {
        const int jl = inv_row[p] - t0;
        if ((unsigned)jl < (unsigned)tw) acc[jl] += fminf(v, inv_val[p]);
      }
      __syncthreads();
    }
  }
  __syncthreads();
  const float a = __fsub_rn(1.f, lambda);
  const float* ndr = nd + (size_t)blockIdx.x * ld_nd + nd_col0 + t0;
  float* o = out + (size_t)blockIdx.x * ld_out + t0;
  for (int t = tid; t < tw; t += JC_THREADS) {
    const float s = acc[t];
    const float jac = __fsub_rn(1.f, __fdiv_rn(s, __fsub_rn(2.f, s)));
    o[t] = __fadd_rn(__fmul_rn(jac, a), __fmul_rn(ndr[t], lambda));
  }
}

// ---------------------------------------------------------------------------------------
// CMC / mAP over a materialised [nq, ld] matrix: the collect and count passes of ctl_dist_pass, same identity encoding,
// junk rule and (distance, column) keys
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(EM_THREADS) eval_matrix_collect_kernel(
    const float* __restrict__ dist, int ng, long long ld, const int* __restrict__ q_pid, const int* __restrict__ q_cam,
    const int* __restrict__ g_pid, const unsigned long long* __restrict__ g_mask, int max_pos,
    unsigned long long* __restrict__ pos_keys, int* __restrict__ pos_count, int* __restrict__ overflow) {
  const int row = blockIdx.x;
  const int qp = q_pid[row], qc = q_cam[row];
  const float* d = dist + (size_t)row * ld;
  for (int j = threadIdx.x; j < ng; j += EM_THREADS) {
    if (g_pid[j] != qp || ((g_mask[j] >> qc) & 1ull)) continue;
    const int slot = atomicAdd(pos_count + row, 1);
    if (slot < max_pos) pos_keys[(size_t)row * max_pos + slot] = key_of(d[j], (uint32_t)j);
    else *overflow = 1;
  }
}

__global__ void __launch_bounds__(EM_THREADS) eval_matrix_count_kernel(
    const float* __restrict__ dist, int ng, long long ld, const int* __restrict__ q_pid, const int* __restrict__ q_cam,
    const int* __restrict__ g_pid, const unsigned long long* __restrict__ g_mask, int max_pos,
    const unsigned long long* __restrict__ thr_keys, const int* __restrict__ thr_count, int* __restrict__ buckets) {
  extern __shared__ int hist[];  // [max_pos + 1] when it fits (smem_hist)
  const int row = blockIdx.x;
  const int npos = min(thr_count[row], max_pos);
  if (npos == 0) return;  // block-uniform
  const bool smem_hist = max_pos + 1 <= EM_HIST_MAX;
  if (smem_hist)
    for (int b = threadIdx.x; b <= npos; b += EM_THREADS) hist[b] = 0;
  __syncthreads();
  const int qp = q_pid[row], qc = q_cam[row];
  const float* d = dist + (size_t)row * ld;
  const unsigned long long* thr = thr_keys + (size_t)row * max_pos;
  const unsigned long long maxkey = thr[npos - 1];
  int* gb = buckets + (size_t)row * (max_pos + 1);
  for (int j = threadIdx.x; j < ng; j += EM_THREADS) {
    if (g_pid[j] == qp && ((g_mask[j] >> qc) & 1ull)) continue;  // junk
    const unsigned long long key = key_of(d[j], (uint32_t)j);
    if (key >= maxkey) continue;
    int lo = 0, hi = npos - 1;  // first positive that sorts after this row (thr[npos - 1] > key)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (thr[mid] > key) hi = mid; else lo = mid + 1;
    }
    if (smem_hist) atomicAdd(hist + lo, 1); else atomicAdd(gb + lo, 1);
  }
  if (smem_hist) {
    __syncthreads();
    for (int b = threadIdx.x; b <= npos; b += EM_THREADS)
      if (hist[b]) atomicAdd(gb + b, hist[b]);
  }
}

// ---------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------
struct RerankPlan {
  int kr;        // rank columns kept: max(k1 + 1, k2)
  int h;         // round-half-even(k1 / 2)
  int v_cap;     // (k1 + 1)(h + 2): bound of |E(i)|
  int q_cap;     // k2 v_cap (k2 > 1), else v_cap: bound of a row of the expanded V
  int buf_pow2;  // expansion buffer per warp
};

int plan_rerank(int64_t nq, int64_t ng, int k1, int k2, RerankPlan* pl) {
  if (k1 < 1 || k2 < 1 || nq < 1 || ng < 1) return CTL_ERR_INVALID_ARGUMENT;
  const int64_t n = nq + ng;
  if (n < 2) return CTL_ERR_INVALID_ARGUMENT;
  pl->kr = std::max(k1 + 1, k2);
  // numpy's around: half to even
  pl->h = (k1 % 2 == 0) ? k1 / 2 : ((k1 / 2) % 2 == 0 ? k1 / 2 : k1 / 2 + 1);
  if (pl->kr > KR_MAX || pl->h + 1 > KR_MAX) return CTL_ERR_UNSUPPORTED;
  const long long v_cap = (long long)(k1 + 1) * (pl->h + 2);
  const long long q_cap = k2 > 1 ? (long long)k2 * v_cap : v_cap;
  if (pow2_at_least(v_cap) > EX_BUF_MAX || (k2 > 1 && pow2_at_least(q_cap) > QE_MAX)) return CTL_ERR_UNSUPPORTED;
  if (n >= (1ll << 31) || ng * q_cap >= (1ll << 31)) return CTL_ERR_UNSUPPORTED;
  pl->v_cap = (int)v_cap;
  pl->q_cap = (int)q_cap;
  pl->buf_pow2 = pow2_at_least(v_cap);
  return 0;
}

struct RerankBuffers {
  float* nd;
  int* rank;
  int *v_idx, *v_cnt;
  float* v_val;
  int *q_idx, *q_cnt;
  float* q_val;
  int *col_ptr, *cursor, *inv_row;
  float* inv_val;
};

size_t rerank_layout(int64_t nq, int64_t ng, int k2, const RerankPlan& pl, void* base, size_t bytes, RerankBuffers* b) {
  const int64_t n = nq + ng;
  Workspace ws(base, bytes);
  b->nd = ws.take<float>((size_t)n * n);
  b->rank = ws.take<int>((size_t)n * pl.kr);
  b->v_idx = ws.take<int>((size_t)n * pl.v_cap);
  b->v_val = ws.take<float>((size_t)n * pl.v_cap);
  b->v_cnt = ws.take<int>((size_t)n);
  if (k2 > 1) {
    b->q_idx = ws.take<int>((size_t)n * pl.q_cap);
    b->q_val = ws.take<float>((size_t)n * pl.q_cap);
    b->q_cnt = ws.take<int>((size_t)n);
  } else {
    b->q_idx = b->v_idx;
    b->q_val = b->v_val;
    b->q_cnt = b->v_cnt;
  }
  b->col_ptr = ws.take<int>((size_t)n + 1);
  b->cursor = ws.take<int>((size_t)n);
  b->inv_row = ws.take<int>((size_t)ng * pl.q_cap);
  b->inv_val = ws.take<float>((size_t)ng * pl.q_cap);
  return ws.off;
}

int set_smem(const void* fn, size_t bytes) {
  if (bytes > 48 * 1024) CTL_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return 0;
}

// rows of a [rows, n] block (the first of them: rank / rowmax point there); rowmax may be null
int launch_rank(float* d, int64_t rows, int64_t n, int64_t ld, int kr, int* rank, float* rowmax, int* status,
                cudaStream_t st) {
  rerank_rank_kernel<true><<<(unsigned)rows, RK_THREADS, 0, st>>>(d, (int)n, ld, kr, rank, rowmax, status, nullptr,
                                                                  nullptr);
  CTL_LAUNCH_CHECK();
  return 0;
}

// the k <= min(KR_MAX, n) smallest (value, column) of each row of a [rows, n] block, as they are
int launch_topk(float* d, int64_t rows, int64_t n, int64_t ld, int k, long long* out_idx, float* out_dist,
                cudaStream_t st) {
  rerank_rank_kernel<false><<<(unsigned)rows, RK_THREADS, 0, st>>>(d, (int)n, ld, k, nullptr, nullptr, nullptr, out_idx,
                                                                   out_dist);
  CTL_LAUNCH_CHECK();
  return 0;
}

int launch_normalise(float* d, int64_t rows, int64_t cols, int64_t ld, const float* rowmax, cudaStream_t st) {
  const dim3 grid((unsigned)rows, (unsigned)std::min<int64_t>((cols + 1023) / 1024, 64));
  rerank_normalise_kernel<<<grid, 256, 0, st>>>(d, (int)cols, ld, rowmax);
  CTL_LAUNCH_CHECK();
  return 0;
}

// rows [r0, r0 + rows) of the n; nd is the block of those rows
int launch_expand(const float* nd, int64_t r0, int64_t rows, int64_t n, int64_t ld, const int* rank, int k1,
                  const RerankPlan& pl, int* v_idx, float* v_val, int* v_cnt, cudaStream_t st) {
  const size_t smem = (size_t)EX_WARPS * (pl.buf_pow2 + 2 * KR_MAX) * sizeof(int);
  int rc = set_smem((const void*)rerank_expand_kernel, smem);
  if (rc) return rc;
  rerank_expand_kernel<<<(unsigned)((rows + EX_WARPS - 1) / EX_WARPS), EX_WARPS * 32, smem, st>>>(
      nd, (int)n, ld, (int)r0, (int)rows, rank, pl.kr, k1, pl.h, v_idx, v_val, v_cnt, pl.v_cap, pl.buf_pow2);
  CTL_LAUNCH_CHECK();
  return 0;
}

int launch_qe(const int* rank, int64_t n, int k2, const RerankPlan& pl, const int* v_idx, const float* v_val,
              const int* v_cnt, int* q_idx, float* q_val, int* q_cnt, cudaStream_t st) {
  const size_t smem = (size_t)std::max(2, pow2_at_least(pl.q_cap)) * sizeof(unsigned long long);
  int rc = set_smem((const void*)rerank_qe_kernel, smem);
  if (rc) return rc;
  rerank_qe_kernel<<<(unsigned)n, QE_THREADS, smem, st>>>(rank, (int)n, pl.kr, k2, v_idx, v_val, v_cnt, pl.v_cap, q_idx,
                                                          q_val, q_cnt, pl.q_cap);
  CTL_LAUNCH_CHECK();
  return 0;
}

int launch_invert(int64_t nq, int64_t ng, const int* idx, const float* val, const int* cnt, int cap, int* col_ptr,
                  int* cursor, int* inv_row, float* inv_val, cudaStream_t st) {
  const int64_t n = nq + ng;
  CTL_CUDA(cudaMemsetAsync(cursor, 0, (size_t)n * sizeof(int), st));
  rerank_colcount_kernel<<<(unsigned)ng, 128, 0, st>>>(idx, cnt, cap, (int)nq, (int)ng, cursor);
  CTL_LAUNCH_CHECK();
  // the counts move to col_ptr's scan, then the cursors restart at each column's start
  rerank_colscan_kernel<<<1, 1024, 0, st>>>(cursor, (int)n, col_ptr, cursor);
  CTL_LAUNCH_CHECK();
  rerank_colfill_kernel<<<(unsigned)ng, 128, 0, st>>>(idx, val, cnt, cap, (int)nq, cursor, inv_row, inv_val);
  CTL_LAUNCH_CHECK();
  return 0;
}

// queries [q0, q0 + rows): nd and out are blocks of those rows, nd's gallery columns start at nd_col0
int launch_jaccard(int64_t q0, int64_t rows, int64_t ng, const int* q_idx, const float* q_val, const int* q_cnt,
                   int q_cap, const int* col_ptr, const int* inv_row, const float* inv_val, const float* nd,
                   int64_t nd_col0, int64_t ld_nd, float lambda, float* out, int64_t ld_out, cudaStream_t st) {
  const int tile = (int)std::min<int64_t>(ng, JC_TILE);
  const size_t smem = (size_t)tile * sizeof(float);
  int rc = set_smem((const void*)rerank_jaccard_kernel, (size_t)JC_TILE * sizeof(float));
  if (rc) return rc;
  const dim3 grid((unsigned)rows, (unsigned)((ng + tile - 1) / tile));
  rerank_jaccard_kernel<<<grid, JC_THREADS, smem, st>>>((int)q0, (int)nd_col0, (int)ng, q_idx, q_val, q_cnt, q_cap,
                                                        col_ptr, inv_row, inv_val, nd, ld_nd, lambda, out, ld_out, tile);
  CTL_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------
// row-blocked re-ranking (ctl_rerank_topk): the N x N matrix is never held, only a [block, N] slice of it
// ---------------------------------------------------------------------------------------
struct BlockedBuffers {
  int* rank;
  float* rowmax;
  int *v_idx, *v_cnt;
  float* v_val;
  int *q_idx, *q_cnt;
  float* q_val;
  int *col_ptr, *cursor, *inv_row;
  float* inv_val;
  float* blk;  // [R, N]: sweeps A and B; [Rq, G] nd rows in sweep C
  float* fin;  // [Rq, G] final distances of sweep C
};

int plan_blocked(int64_t nq, int64_t ng, int32_t d, int k1, int k2, int k, int64_t block_rows, RerankPlan* pl) {
  int rc = plan_rerank(nq, ng, k1, k2, pl);
  if (rc) return rc;
  if (d < 8 || d % 8 || k < 1 || k > std::min<int64_t>(KR_MAX, ng) || block_rows < 1) return CTL_ERR_INVALID_ARGUMENT;
  return 0;
}

size_t blocked_layout(int64_t nq, int64_t ng, int k2, int64_t block_rows, const RerankPlan& pl, void* base, size_t bytes,
                      BlockedBuffers* b) {
  const int64_t n = nq + ng;
  const int64_t r = std::min(block_rows, n), rq = std::min(block_rows, nq);
  Workspace ws(base, bytes);
  b->rank = ws.take<int>((size_t)n * pl.kr);
  b->rowmax = ws.take<float>((size_t)n);
  b->v_idx = ws.take<int>((size_t)n * pl.v_cap);
  b->v_val = ws.take<float>((size_t)n * pl.v_cap);
  b->v_cnt = ws.take<int>((size_t)n);
  if (k2 > 1) {
    b->q_idx = ws.take<int>((size_t)n * pl.q_cap);
    b->q_val = ws.take<float>((size_t)n * pl.q_cap);
    b->q_cnt = ws.take<int>((size_t)n);
  } else {
    b->q_idx = b->v_idx;
    b->q_val = b->v_val;
    b->q_cnt = b->v_cnt;
  }
  b->col_ptr = ws.take<int>((size_t)n + 1);
  b->cursor = ws.take<int>((size_t)n);
  b->inv_row = ws.take<int>((size_t)ng * pl.q_cap);
  b->inv_val = ws.take<float>((size_t)ng * pl.q_cap);
  b->blk = ws.take<float>((size_t)r * n);
  b->fin = ws.take<float>((size_t)rq * ng);
  return ws.off;
}

}  // namespace
}  // namespace ctl

using namespace ctl;

extern "C" {

int ctl_rerank_plan(int64_t nq, int64_t ng, int32_t k1, int32_t k2, int32_t* kr, int32_t* h, int32_t* v_cap,
                    int32_t* q_cap) {
  CTL_CHECK_ARG(kr && h && v_cap && q_cap, "null output");
  RerankPlan pl;
  const int rc = plan_rerank(nq, ng, k1, k2, &pl);
  if (rc == CTL_ERR_INVALID_ARGUMENT) {
    set_error("re-ranking needs k1 >= 1, k2 >= 1, nq >= 1, ng >= 1 (k1=%d k2=%d nq=%lld ng=%lld)", k1, k2, (long long)nq,
              (long long)ng);
    return rc;
  }
  if (rc) {
    set_error("re-ranking plan (k1=%d, k2=%d, ng=%lld) exceeds the kernels' capacities", k1, k2, (long long)ng);
    return rc;
  }
  *kr = pl.kr;
  *h = pl.h;
  *v_cap = pl.v_cap;
  *q_cap = pl.q_cap;
  return 0;
}

size_t ctl_rerank_workspace_bytes(int64_t nq, int64_t ng, int32_t k1, int32_t k2) {
  RerankPlan pl;
  if (plan_rerank(nq, ng, k1, k2, &pl)) return 0;
  RerankBuffers b;
  return rerank_layout(nq, ng, k2, pl, nullptr, 0, &b);
}

int ctl_rerank_rank(float* dist, int64_t n, int64_t ld, int32_t kr, int32_t* rank, int32_t* status, ctl_stream_t stream) {
  CTL_CHECK_ARG(dist && rank && status, "null pointer");
  CTL_CHECK_ARG(n >= 2 && n < (1ll << 31) && ld >= n, "bad shape n=%lld ld=%lld", (long long)n, (long long)ld);
  CTL_CHECK_ARG(kr >= 1 && kr <= KR_MAX, "kr=%d must be in [1, %d]", kr, KR_MAX);
  int rc = ctl_device_check();
  if (rc) return rc;
  return launch_rank(dist, n, n, ld, kr, rank, nullptr, status, (cudaStream_t)stream);
}

int ctl_rerank_expand(const float* nd, int64_t n, int64_t ld, const int32_t* rank, int32_t k1, int32_t k2,
                      int32_t* v_idx, float* v_val, int32_t* v_cnt, ctl_stream_t stream) {
  CTL_CHECK_ARG(nd && rank && v_idx && v_val && v_cnt, "null pointer");
  CTL_CHECK_ARG(n >= 2 && ld >= n, "bad shape n=%lld ld=%lld", (long long)n, (long long)ld);
  RerankPlan pl;
  CTL_CHECK_ARG(plan_rerank(1, n - 1, k1, k2, &pl) == 0, "unsupported k1=%d k2=%d", k1, k2);
  int rc = ctl_device_check();
  if (rc) return rc;
  return launch_expand(nd, 0, n, n, ld, rank, k1, pl, v_idx, v_val, v_cnt, (cudaStream_t)stream);
}

int ctl_rerank_qe(const int32_t* rank, int64_t n, int32_t k1, int32_t k2, const int32_t* v_idx, const float* v_val,
                  const int32_t* v_cnt, int32_t* q_idx, float* q_val, int32_t* q_cnt, ctl_stream_t stream) {
  CTL_CHECK_ARG(rank && v_idx && v_val && v_cnt && q_idx && q_val && q_cnt, "null pointer");
  CTL_CHECK_ARG(n >= 2, "bad shape n=%lld", (long long)n);
  RerankPlan pl;
  CTL_CHECK_ARG(plan_rerank(1, n - 1, k1, k2, &pl) == 0, "unsupported k1=%d k2=%d", k1, k2);
  CTL_CHECK_ARG(k2 > 1, "query expansion needs k2 > 1 (k2 = 1 uses V as it is)");
  int rc = ctl_device_check();
  if (rc) return rc;
  return launch_qe(rank, n, k2, pl, v_idx, v_val, v_cnt, q_idx, q_val, q_cnt, (cudaStream_t)stream);
}

int ctl_rerank_invert(int64_t nq, int64_t ng, const int32_t* idx, const float* val, const int32_t* cnt, int32_t cap,
                      int32_t* col_ptr, int32_t* cursor, int32_t* inv_row, float* inv_val, ctl_stream_t stream) {
  CTL_CHECK_ARG(idx && val && cnt && col_ptr && cursor && inv_row && inv_val, "null pointer");
  CTL_CHECK_ARG(nq >= 1 && ng >= 1 && nq + ng < (1ll << 31) && cap >= 1 && ng * cap < (1ll << 31), "bad shape");
  int rc = ctl_device_check();
  if (rc) return rc;
  return launch_invert(nq, ng, idx, val, cnt, cap, col_ptr, cursor, inv_row, inv_val, (cudaStream_t)stream);
}

int ctl_rerank_jaccard(int64_t nq, int64_t ng, const int32_t* idx, const float* val, const int32_t* cnt, int32_t cap,
                       const int32_t* col_ptr, const int32_t* inv_row, const float* inv_val, const float* nd,
                       int64_t ld_nd, float lambda_value, float* out, int64_t ld_out, ctl_stream_t stream) {
  CTL_CHECK_ARG(idx && val && cnt && col_ptr && inv_row && inv_val && nd && out, "null pointer");
  CTL_CHECK_ARG(nq >= 1 && ng >= 1 && nq + ng < (1ll << 31) && ld_nd >= nq + ng && ld_out >= ng && cap >= 1, "bad shape");
  int rc = ctl_device_check();
  if (rc) return rc;
  return launch_jaccard(0, nq, ng, idx, val, cnt, cap, col_ptr, inv_row, inv_val, nd, nq, ld_nd, lambda_value, out,
                        ld_out, (cudaStream_t)stream);
}

int ctl_rerank(const void* planes, int64_t nq, int64_t ng, int32_t d, int32_t flags, int32_t k1, int32_t k2,
               float lambda_value, float* out, int64_t ld_out, int32_t* status, void* workspace, size_t workspace_bytes,
               ctl_stream_t stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  CTL_CHECK_ARG(planes && out && status && workspace, "null pointer");
  CTL_CHECK_ARG(ld_out >= ng, "ld_out=%lld < ng=%lld", (long long)ld_out, (long long)ng);
  CTL_CHECK_ARG(!(flags & (CTL_DIST_COSINE | CTL_DIST_SQRT)), "re-ranking starts from squared euclidean distances");
  RerankPlan pl;
  int rc = plan_rerank(nq, ng, k1, k2, &pl);
  if (rc) {
    int32_t a, b, c, e;
    return ctl_rerank_plan(nq, ng, k1, k2, &a, &b, &c, &e);  // the same status, with its message
  }
  RerankBuffers bf;
  const size_t need = rerank_layout(nq, ng, k2, pl, workspace, workspace_bytes, &bf);
  if (need > workspace_bytes) {
    set_error("workspace too small: need %zu bytes, have %zu", need, workspace_bytes);
    return CTL_ERR_WORKSPACE;
  }
  const int64_t n = nq + ng;
  CTL_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
  if ((rc = ctl_dist_matrix(planes, n, planes, n, d, flags, bf.nd, n, stream_))) return rc;
  if ((rc = launch_rank(bf.nd, n, n, n, pl.kr, bf.rank, nullptr, status, st))) return rc;
  if ((rc = launch_expand(bf.nd, 0, n, n, n, bf.rank, k1, pl, bf.v_idx, bf.v_val, bf.v_cnt, st))) return rc;
  if (k2 > 1 && (rc = launch_qe(bf.rank, n, k2, pl, bf.v_idx, bf.v_val, bf.v_cnt, bf.q_idx, bf.q_val, bf.q_cnt, st)))
    return rc;
  const int cap = k2 > 1 ? pl.q_cap : pl.v_cap;
  if ((rc = launch_invert(nq, ng, bf.q_idx, bf.q_val, bf.q_cnt, cap, bf.col_ptr, bf.cursor, bf.inv_row, bf.inv_val, st)))
    return rc;
  return launch_jaccard(0, nq, ng, bf.q_idx, bf.q_val, bf.q_cnt, cap, bf.col_ptr, bf.inv_row, bf.inv_val, bf.nd, nq, n,
                        lambda_value, out, ld_out, st);
}

static int check_matrix_ids(const float* dist, int64_t nq, int64_t ng, int64_t ld, const int32_t* q_pid,
                            const int32_t* q_cam, const int32_t* g_pid, const uint64_t* g_cammask, int32_t max_pos) {
  CTL_CHECK_ARG(dist && q_pid && q_cam && g_pid && g_cammask, "null pointer");
  CTL_CHECK_ARG(nq >= 1 && ng >= 1 && nq < (1ll << 31) && ng < (1ll << 31) && ld >= ng, "bad shape nq=%lld ng=%lld ld=%lld",
                (long long)nq, (long long)ng, (long long)ld);
  CTL_CHECK_ARG(max_pos >= 1, "max_pos must be >= 1");
  return ctl_device_check();
}

int ctl_eval_matrix_collect(const float* dist, int64_t nq, int64_t ng, int64_t ld, const int32_t* q_pid,
                            const int32_t* q_cam, const int32_t* g_pid, const uint64_t* g_cammask, int32_t max_pos,
                            uint64_t* pos_keys, int32_t* pos_count, int32_t* overflow, ctl_stream_t stream) {
  CTL_CHECK_ARG(pos_keys && pos_count && overflow, "null output");
  int rc = check_matrix_ids(dist, nq, ng, ld, q_pid, q_cam, g_pid, g_cammask, max_pos);
  if (rc) return rc;
  eval_matrix_collect_kernel<<<(unsigned)nq, EM_THREADS, 0, (cudaStream_t)stream>>>(
      dist, (int)ng, ld, q_pid, q_cam, g_pid, reinterpret_cast<const unsigned long long*>(g_cammask), max_pos,
      reinterpret_cast<unsigned long long*>(pos_keys), pos_count, overflow);
  CTL_LAUNCH_CHECK();
  return 0;
}

int ctl_eval_matrix_count(const float* dist, int64_t nq, int64_t ng, int64_t ld, const int32_t* q_pid,
                          const int32_t* q_cam, const int32_t* g_pid, const uint64_t* g_cammask, int32_t max_pos,
                          const uint64_t* pos_keys_sorted, const int32_t* pos_count, int32_t* buckets,
                          ctl_stream_t stream) {
  CTL_CHECK_ARG(pos_keys_sorted && pos_count && buckets, "null pointer");
  int rc = check_matrix_ids(dist, nq, ng, ld, q_pid, q_cam, g_pid, g_cammask, max_pos);
  if (rc) return rc;
  const size_t smem = max_pos + 1 <= EM_HIST_MAX ? (size_t)(max_pos + 1) * sizeof(int) : 0;
  eval_matrix_count_kernel<<<(unsigned)nq, EM_THREADS, smem, (cudaStream_t)stream>>>(
      dist, (int)ng, ld, q_pid, q_cam, g_pid, reinterpret_cast<const unsigned long long*>(g_cammask), max_pos,
      reinterpret_cast<const unsigned long long*>(pos_keys_sorted), pos_count, buckets);
  CTL_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------
// row-blocked re-ranking: stage entry points over row blocks, and the one-call ctl_rerank_topk
// ---------------------------------------------------------------------------------------
size_t ctl_rerank_topk_workspace_bytes(int64_t nq, int64_t ng, int32_t d, int32_t k1, int32_t k2, int32_t k,
                                       int64_t block_rows) {
  RerankPlan pl;
  if (plan_blocked(nq, ng, d, k1, k2, k, block_rows, &pl)) return 0;
  BlockedBuffers b;
  return blocked_layout(nq, ng, k2, block_rows, pl, nullptr, 0, &b);
}

int ctl_rerank_dist_rows(const void* planes, int64_t n, int32_t d, int32_t flags, int64_t r0, int64_t rows, int64_t c0,
                         int64_t cols, const float* rowmax, float* out, int64_t ld_out, ctl_stream_t stream) {
  CTL_CHECK_ARG(!(flags & (CTL_DIST_COSINE | CTL_DIST_SQRT)), "re-ranking starts from squared euclidean distances");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = dist_matrix_rows(planes, n, d, flags, r0, rows, c0, cols, out, ld_out, st);
  if (rc || !rowmax) return rc;
  return launch_normalise(out, rows, cols, ld_out, rowmax + r0, st);
}

int ctl_rerank_rank_rows(float* dist, int64_t r0, int64_t rows, int64_t n, int64_t ld, int32_t kr, int32_t* rank,
                         float* rowmax, int32_t* status, ctl_stream_t stream) {
  CTL_CHECK_ARG(dist && rank && rowmax && status, "null pointer");
  CTL_CHECK_ARG(n >= 2 && n < (1ll << 31) && r0 >= 0 && rows >= 1 && r0 + rows <= n && ld >= n,
                "bad row block r0=%lld rows=%lld n=%lld ld=%lld", (long long)r0, (long long)rows, (long long)n,
                (long long)ld);
  CTL_CHECK_ARG(kr >= 1 && kr <= KR_MAX, "kr=%d must be in [1, %d]", kr, KR_MAX);
  int rc = ctl_device_check();
  if (rc) return rc;
  return launch_rank(dist, rows, n, ld, kr, rank + r0 * kr, rowmax + r0, status, (cudaStream_t)stream);
}

int ctl_rerank_expand_rows(const float* nd, int64_t r0, int64_t rows, int64_t n, int64_t ld, const int32_t* rank,
                           int32_t k1, int32_t k2, int32_t* v_idx, float* v_val, int32_t* v_cnt, ctl_stream_t stream) {
  CTL_CHECK_ARG(nd && rank && v_idx && v_val && v_cnt, "null pointer");
  CTL_CHECK_ARG(n >= 2 && n < (1ll << 31) && r0 >= 0 && rows >= 1 && r0 + rows <= n && ld >= n,
                "bad row block r0=%lld rows=%lld n=%lld ld=%lld", (long long)r0, (long long)rows, (long long)n,
                (long long)ld);
  RerankPlan pl;
  CTL_CHECK_ARG(plan_rerank(1, n - 1, k1, k2, &pl) == 0, "unsupported k1=%d k2=%d", k1, k2);
  int rc = ctl_device_check();
  if (rc) return rc;
  return launch_expand(nd, r0, rows, n, ld, rank, k1, pl, v_idx, v_val, v_cnt, (cudaStream_t)stream);
}

int ctl_rerank_jaccard_rows(int64_t nq, int64_t ng, int64_t q0, int64_t rows, const int32_t* idx, const float* val,
                            const int32_t* cnt, int32_t cap, const int32_t* col_ptr, const int32_t* inv_row,
                            const float* inv_val, const float* nd, int64_t ld_nd, float lambda_value, float* out,
                            int64_t ld_out, ctl_stream_t stream) {
  CTL_CHECK_ARG(idx && val && cnt && col_ptr && inv_row && inv_val && nd && out, "null pointer");
  CTL_CHECK_ARG(nq >= 1 && ng >= 1 && nq + ng < (1ll << 31) && q0 >= 0 && rows >= 1 && q0 + rows <= nq && ld_nd >= ng &&
                    ld_out >= ng && cap >= 1,
                "bad shape");
  int rc = ctl_device_check();
  if (rc) return rc;
  return launch_jaccard(q0, rows, ng, idx, val, cnt, cap, col_ptr, inv_row, inv_val, nd, 0, ld_nd, lambda_value, out,
                        ld_out, (cudaStream_t)stream);
}

int ctl_rerank_topk_rows(float* dist, int64_t r0, int64_t rows, int64_t n, int64_t ld, int32_t k, int64_t* out_idx,
                         float* out_dist, ctl_stream_t stream) {
  CTL_CHECK_ARG(dist && out_idx && out_dist, "null pointer");
  CTL_CHECK_ARG(n >= 1 && n < (1ll << 31) && r0 >= 0 && rows >= 1 && ld >= n, "bad shape r0=%lld rows=%lld n=%lld",
                (long long)r0, (long long)rows, (long long)n);
  CTL_CHECK_ARG(k >= 1 && k <= KR_MAX && k <= n, "k=%d must be in [1, min(%d, n=%lld)]", k, KR_MAX, (long long)n);
  int rc = ctl_device_check();
  if (rc) return rc;
  return launch_topk(dist, rows, n, ld, k, reinterpret_cast<long long*>(out_idx) + r0 * k, out_dist + r0 * k,
                     (cudaStream_t)stream);
}

int ctl_rerank_topk(const void* planes, int64_t nq, int64_t ng, int32_t d, int32_t flags, int32_t k1, int32_t k2,
                    float lambda_value, int32_t k, int64_t block_rows, int64_t* out_idx, float* out_dist,
                    const int32_t* q_pid, const int32_t* q_cam, const int32_t* g_pid, const uint64_t* g_cammask,
                    int32_t max_pos, uint64_t* pos_keys, int32_t* pos_count, int32_t* buckets, int32_t* overflow,
                    int32_t* status, void* workspace, size_t workspace_bytes, ctl_stream_t stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  CTL_CHECK_ARG(planes && out_idx && out_dist && status && workspace, "null pointer");
  CTL_CHECK_ARG(!(flags & (CTL_DIST_COSINE | CTL_DIST_SQRT)), "re-ranking starts from squared euclidean distances");
  const bool eval = q_pid != nullptr;
  CTL_CHECK_ARG(!eval || (q_cam && g_pid && g_cammask && pos_keys && pos_count && buckets && overflow && max_pos >= 1),
                "evaluation needs every identity array and output (max_pos >= 1)");
  RerankPlan pl;
  int rc = plan_blocked(nq, ng, d, k1, k2, k, block_rows, &pl);
  if (rc == CTL_ERR_INVALID_ARGUMENT && plan_rerank(nq, ng, k1, k2, &pl) == 0) {
    set_error("blocked re-ranking needs d a positive multiple of 8, 1 <= k <= min(%d, ng) and block_rows >= 1 "
              "(d=%d k=%d ng=%lld block_rows=%lld)", KR_MAX, d, k, (long long)ng, (long long)block_rows);
    return rc;
  }
  if (rc) {
    int32_t a, b, c, e;
    return ctl_rerank_plan(nq, ng, k1, k2, &a, &b, &c, &e);  // the same status, with its message
  }
  BlockedBuffers bf;
  const size_t need = blocked_layout(nq, ng, k2, block_rows, pl, workspace, workspace_bytes, &bf);
  if (need > workspace_bytes) {
    set_error("workspace too small: need %zu bytes, have %zu", need, workspace_bytes);
    return CTL_ERR_WORKSPACE;
  }
  if ((rc = ctl_device_check())) return rc;
  const int64_t n = nq + ng, R = std::min<int64_t>(block_rows, n);
  CTL_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
  if (eval) {
    CTL_CUDA(cudaMemsetAsync(pos_count, 0, (size_t)nq * sizeof(int32_t), st));
    CTL_CUDA(cudaMemsetAsync(buckets, 0, (size_t)nq * (max_pos + 1) * sizeof(int32_t), st));
    CTL_CUDA(cudaMemsetAsync(overflow, 0, sizeof(int32_t), st));
  }
  // sweep A: the row maxima and the rank table, one [R, N] block at a time
  for (int64_t r0 = 0; r0 < n; r0 += R) {
    const int64_t rows = std::min(R, n - r0);
    if ((rc = dist_matrix_rows(planes, n, d, flags, r0, rows, 0, n, bf.blk, n, st))) return rc;
    if ((rc = launch_rank(bf.blk, rows, n, n, pl.kr, bf.rank + r0 * pl.kr, bf.rowmax + r0, status, st))) return rc;
  }
  // sweep B: the same blocks again, normalised by the stored maxima; the expansion reads the rank table of all rows
  for (int64_t r0 = 0; r0 < n; r0 += R) {
    const int64_t rows = std::min(R, n - r0);
    if ((rc = dist_matrix_rows(planes, n, d, flags, r0, rows, 0, n, bf.blk, n, st))) return rc;
    if ((rc = launch_normalise(bf.blk, rows, n, n, bf.rowmax + r0, st))) return rc;
    if ((rc = launch_expand(bf.blk, r0, rows, n, n, bf.rank, k1, pl, bf.v_idx, bf.v_val, bf.v_cnt, st))) return rc;
  }
  if (k2 > 1 && (rc = launch_qe(bf.rank, n, k2, pl, bf.v_idx, bf.v_val, bf.v_cnt, bf.q_idx, bf.q_val, bf.q_cnt, st)))
    return rc;
  const int cap = k2 > 1 ? pl.q_cap : pl.v_cap;
  if ((rc = launch_invert(nq, ng, bf.q_idx, bf.q_val, bf.q_cnt, cap, bf.col_ptr, bf.cursor, bf.inv_row, bf.inv_val, st)))
    return rc;
  // sweep C: query blocks against the gallery only -> final distances -> top-k (and the evaluation passes)
  const int64_t Rq = std::min<int64_t>(block_rows, nq);
  const unsigned long long* gm = reinterpret_cast<const unsigned long long*>(g_cammask);
  for (int64_t q0 = 0; q0 < nq; q0 += Rq) {
    const int64_t rows = std::min(Rq, nq - q0);
    if ((rc = dist_matrix_rows(planes, n, d, flags, q0, rows, nq, ng, bf.blk, ng, st))) return rc;
    if ((rc = launch_normalise(bf.blk, rows, ng, ng, bf.rowmax + q0, st))) return rc;
    if ((rc = launch_jaccard(q0, rows, ng, bf.q_idx, bf.q_val, bf.q_cnt, cap, bf.col_ptr, bf.inv_row, bf.inv_val, bf.blk,
                             0, ng, lambda_value, bf.fin, ng, st)))
      return rc;
    if ((rc = launch_topk(bf.fin, rows, ng, ng, k, reinterpret_cast<long long*>(out_idx) + q0 * k, out_dist + q0 * k, st)))
      return rc;
    if (!eval) continue;
    unsigned long long* pk = reinterpret_cast<unsigned long long*>(pos_keys) + q0 * max_pos;
    eval_matrix_collect_kernel<<<(unsigned)rows, EM_THREADS, 0, st>>>(bf.fin, (int)ng, ng, q_pid + q0, q_cam + q0, g_pid,
                                                                      gm, max_pos, pk, pos_count + q0, overflow);
    CTL_LAUNCH_CHECK();
    if ((rc = ctl_sort_key_rows(reinterpret_cast<uint64_t*>(pk), pos_count + q0, rows, max_pos, stream_))) return rc;
    const size_t smem = max_pos + 1 <= EM_HIST_MAX ? (size_t)(max_pos + 1) * sizeof(int) : 0;
    eval_matrix_count_kernel<<<(unsigned)rows, EM_THREADS, smem, st>>>(bf.fin, (int)ng, ng, q_pid + q0, q_cam + q0, g_pid,
                                                                       gm, max_pos, pk, pos_count + q0,
                                                                       buckets + q0 * (max_pos + 1));
    CTL_LAUNCH_CHECK();
  }
  return 0;
}

}  // extern "C"
