// CTL training-step losses, forward AND backward in one enqueue (no host sync, one 8-float
// result buffer): image-level batch-hard triplet, K centroid-triplet rounds, center loss,
// BatchNorm1d -> bias-free linear -> label-smoothed cross-entropy.
//
// Replaces train_ctl_model.py:54-152 (+ the backward autograd derives from it),
// losses/triplet_loss.py:27-41,68-173,194-205, losses/center_loss.py:26-45,
// modelling/bases.py:359-384 (create_masks_train) of the reference.  SURVEY.md A.1/A.2 give
// the closed forms implemented here.
//
// Data layout (all fp32, row-major): E_all = [ F (B rows) ; cent_0 (P rows) ; ... ; cent_{K-1} ]
// so that ONE Gram matrix G = E_all E_all^T serves the image-level problem (rows < B) and
// every round r (rows {cK+r} U {B + rP + c}); ONE sparse symmetric coefficient matrix Cm
// carries every selected (anchor, positive/negative) pair, and the whole triplet backward is
// dE = rowsum(Cm) * E - Cm E: a second GEMM.  All reductions have a fixed order
// (deterministic, no floating-point atomics).  These problems are tiny (<= 1 GFLOP) and
// latency-bound; they run as fp32 CUDA-core kernels because loss math must stay fp32.
#include <math_constants.h>

#include "common.h"

namespace ctl {

// ---------------------------------------------------------------------------------------
// strided fp32 GEMM: C[m,n] = alpha * sum_k A(m,k) B(k,n) + beta * C[m,n]
// A(m,k) = A[m*sam + k*sak],  B(k,n) = B[k*sbk + n*sbn];  k summed in increasing order.
// ---------------------------------------------------------------------------------------
static constexpr int TM = 64, TN = 64, TK = 16;

__global__ void __launch_bounds__(256) sgemm_kernel(int M, int N, int K, const float* __restrict__ A, long long sam,
                                                    long long sak, const float* __restrict__ Bm, long long sbk,
                                                    long long sbn, float* __restrict__ C, long long ldc, float alpha,
                                                    float beta) {
  __shared__ float As[TK][TM + 4];
  __shared__ float Bs[TK][TN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  const int ty = tid / 16, tx = tid % 16;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += TK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = tid + i * 256;
      int m, k;
      if (sak == 1) { k = e % TK; m = e / TK; } else { m = e % TM; k = e / TM; }
      const int gm = m0 + m, gk = k0 + k;
      As[k][m] = (gm < M && gk < K) ? A[gm * sam + gk * sak] : 0.f;
      int n, kb;
      if (sbn == 1) { n = e % TN; kb = e / TN; } else { kb = e % TK; n = e / TK; }
      const int gn = n0 + n, gkb = k0 + kb;
      Bs[kb][n] = (gn < N && gkb < K) ? Bm[gkb * sbk + gn * sbn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = __fmaf_rn(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gm = m0 + ty * 4 + i, gn = n0 + tx * 4 + j;
      if (gm < M && gn < N) {
        float v = alpha * acc[i][j];
        if (beta != 0.f) v = __fmaf_rn(beta, C[gm * ldc + gn], v);
        C[gm * ldc + gn] = v;
      }
    }
}

static int sgemm(cudaStream_t st, int M, int N, int K, const float* A, long long sam, long long sak, const float* B,
                 long long sbk, long long sbn, float* C, long long ldc, float alpha, float beta) {
  dim3 grid((N + TN - 1) / TN, (M + TM - 1) / TM);
  sgemm_kernel<<<grid, 256, 0, st>>>(M, N, K, A, sam, sak, B, sbk, sbn, C, ldc, alpha, beta);
  CTL_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------
// block reductions (fixed order)
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ float block_sum(float v, float* sm) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane == 0) sm[w] = v;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += sm[i];
  return t;
}

// ---------------------------------------------------------------------------------------
// step metadata derived from is_real on the device (no host sync)
// ---------------------------------------------------------------------------------------
struct StepMeta {
  int n_real;          // B'
  int n_valid_rounds;  // rounds with more than one valid class
  int round_valid[64];
  int round_classes[64];  // P'_r
  int bad_batch;  // != 0: the batch violates the contract (1 label out of [0, C); 2 label not constant in a K-block;
                  // 3 the same label in two blocks) -> every reported loss is NaN, centers are never indexed out of range
};

// slot t < B            : image-level anchor, row t
// slot B + r*2P + c     : round r query anchor of class c  (row cK + r)
// slot B + r*2P + P + c : round r centroid anchor of class c (row B + rP + c)
__global__ void step_setup_kernel(const unsigned char* __restrict__ is_real, const int* __restrict__ labels, int C, int P,
                                  int K, StepMeta* meta, int* __restrict__ n_rc /*[K,P]*/,
                                  int* __restrict__ labels_safe /*[B]*/) {
  __shared__ int s_real, s_rounds, s_bad;
  if (threadIdx.x == 0) { s_real = 0; s_rounds = 0; s_bad = 0; }
  __syncthreads();
  // Batch contract (datasets/bases.py:346-406): the mining kernels derive the class of a row from its POSITION
  // (row / K), so the labels must be constant inside each block of K rows, distinct across blocks, and in [0, C).
  // The reference's label-driven mining would silently compute something else on such a batch; here it is an error.
  for (int i = threadIdx.x; i < P * K; i += blockDim.x) {
    const int y = labels[i];
    int bad = 0;
    if (y < 0 || y >= C) bad = 1;
    else if (y != labels[(i / K) * K]) bad = 2;
    else if (i % K == 0)
      for (int c = 0; c < i / K; ++c)
        if (labels[c * K] == y) bad = 3;
    if (bad) atomicMax(&s_bad, bad);
    labels_safe[i] = (y < 0 || y >= C) ? 0 : y;
  }
  int real = 0;
  for (int i = threadIdx.x; i < P * K; i += blockDim.x) real += is_real[i] ? 1 : 0;
  atomicAdd(&s_real, real);
  for (int r = threadIdx.x; r < K; r += blockDim.x) {
    int classes = 0, with_centroid = 0;
    for (int c = 0; c < P; ++c) {
      const bool q = is_real[c * K + r];
      int n = 0;
      if (q)
        for (int s = 0; s < K; ++s) n += (s != r && is_real[c * K + s]) ? 1 : 0;
      n_rc[r * P + c] = n;
      classes += q ? 1 : 0;
      with_centroid += n > 0 ? 1 : 0;
    }
    // train_ctl_model.py:113: skip the round unless more than one class has a centroid
    const int valid = with_centroid > 1 ? 1 : 0;
    meta->round_valid[r] = valid;
    meta->round_classes[r] = classes;
    if (valid) atomicAdd(&s_rounds, 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    meta->n_real = s_real;
    meta->n_valid_rounds = s_rounds;
    meta->bad_batch = s_bad;
  }
}

// E_all rows B.. : masked mean of the other real members (train_ctl_model.py:89-104); also the
// per-row squared norms of ALL of E_all and the centroid L2 norms.
__global__ void __launch_bounds__(256) build_rows_kernel(const float* __restrict__ F, int B, int D, int P, int K,
                                                         const unsigned char* __restrict__ is_real,
                                                         const int* __restrict__ n_rc, float* __restrict__ E_cent,
                                                         float* __restrict__ sq /*[B + K*P]*/) {
  __shared__ float sm[8];
  const int row = blockIdx.x;  // 0 .. B + K*P
  float ss = 0.f;
  if (row < B) {
    for (int j = threadIdx.x; j < D; j += blockDim.x) {
      const float v = F[(size_t)row * D + j];
      ss = __fmaf_rn(v, v, ss);
    }
  } else {
    const int rc = row - B, r = rc / P, c = rc % P;
    const int n = n_rc[r * P + c];
    const float inv_n = n > 0 ? (float)n : 1.f;
    for (int j = threadIdx.x; j < D; j += blockDim.x) {
      float acc = 0.f;
      if (n > 0)
        for (int s = 0; s < K; ++s)
          if (s != r && is_real[c * K + s]) acc = __fadd_rn(acc, F[(size_t)(c * K + s) * D + j]);
      const float v = __fdiv_rn(acc, inv_n);
      E_cent[(size_t)rc * D + j] = v;
      ss = __fmaf_rn(v, v, ss);
    }
  }
  ss = block_sum(ss, sm);
  if (threadIdx.x == 0) sq[row] = ss;
}

// ---------------------------------------------------------------------------------------
// batch-hard mining: one block per anchor slot
// ---------------------------------------------------------------------------------------
struct MineOut {
  int* a_row;     // [T] anchor row in E_all or -1
  int* p_row;     // [T]
  int* n_row;     // [T]
  float* cap;     // [T] d(loss)/d(d_ap) / d_ap  (0 if the hinge is inactive)
  float* can;     // [T]
  float* hinge;   // [T]
  float* d_ap;    // [T]
  float* d_an;    // [T]
};

__device__ __forceinline__ float pair_dist(const float* __restrict__ G, int ld, const float* __restrict__ sq, int i,
                                           int j, bool* saturated) {
  // losses/triplet_loss.py:36-40: xx + yy - 2 x.y, clamp(min=1e-12), sqrt
  const float s = __fmaf_rn(-2.f, G[(size_t)i * ld + j], __fadd_rn(sq[i], sq[j]));
  *saturated = s < 1e-12f;
  return __fsqrt_rn(fmaxf(s, 1e-12f));
}

// cosine_dist (losses/triplet_loss.py:58-65) from the Gram matrix of the NORMALISED rows: clamp(|1 - cos|, 1e-12);
// *sgn = d(distance)/d(1 - cos) (0 where the clamp saturates)
__device__ __forceinline__ float pair_dist_cos(const float* __restrict__ G, int ld, int i, int j, float* sgn) {
  const float s = __fsub_rn(1.f, G[(size_t)i * ld + j]);
  const float a = fabsf(s);
  *sgn = a < 1e-12f ? 0.f : (s >= 0.f ? 1.f : -1.f);
  return fmaxf(a, 1e-12f);
}

// generic single-problem variant (standalone TripletLoss): candidates are all N rows.
// `cosine`: distances are cosine distances of pre-normalised rows; `soft`: SoftMarginLoss(d_an - d_ap, 1) =
// log(1 + exp(d_ap - d_an)) instead of the hinge (TripletLoss(margin=None), triplet_loss.py:130-131,157-158).
__global__ void __launch_bounds__(128) mine_single_kernel(const float* __restrict__ G, const float* __restrict__ sq,
                                                          const int* __restrict__ labels,
                                                          const unsigned char* __restrict__ anchor_mask, int N,
                                                          float margin, int soft, int cosine, MineOut o) {
  __shared__ float s_v[128];
  __shared__ int s_i[128];
  const int a = blockIdx.x;
  const int la = labels[a];
  float best_p = -CUDART_INF_F, best_n = CUDART_INF_F;
  int ip = -1, in = -1;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    bool sat;
    float sg;
    const float d = cosine ? pair_dist_cos(G, N, a, j, &sg) : pair_dist(G, N, sq, a, j, &sat);
    if (labels[j] == la) {
      if (d > best_p) { best_p = d; ip = j; }
    } else {
      if (d < best_n) { best_n = d; in = j; }
    }
  }
  // max with lowest index on ties
  s_v[threadIdx.x] = best_p; s_i[threadIdx.x] = ip;
  __syncthreads();
  for (int st = 64; st > 0; st >>= 1) {
    if (threadIdx.x < st) {
      const float v2 = s_v[threadIdx.x + st]; const int i2 = s_i[threadIdx.x + st];
      if (i2 >= 0 && (s_i[threadIdx.x] < 0 || v2 > s_v[threadIdx.x] || (v2 == s_v[threadIdx.x] && i2 < s_i[threadIdx.x]))) {
        s_v[threadIdx.x] = v2; s_i[threadIdx.x] = i2;
      }
    }
    __syncthreads();
  }
  const float dap = s_v[0]; const int pidx = s_i[0];
  __syncthreads();
  s_v[threadIdx.x] = best_n; s_i[threadIdx.x] = in;
  __syncthreads();
  for (int st = 64; st > 0; st >>= 1) {
    if (threadIdx.x < st) {
      const float v2 = s_v[threadIdx.x + st]; const int i2 = s_i[threadIdx.x + st];
      if (i2 >= 0 && (s_i[threadIdx.x] < 0 || v2 < s_v[threadIdx.x] || (v2 == s_v[threadIdx.x] && i2 < s_i[threadIdx.x]))) {
        s_v[threadIdx.x] = v2; s_i[threadIdx.x] = i2;
      }
    }
    __syncthreads();
  }
  const float dan = s_v[0]; const int nidx = s_i[0];
  if (threadIdx.x == 0) {
    const bool active = anchor_mask == nullptr || anchor_mask[a];
    const float x = dap - dan;
    // hinge: max(0, x + margin); soft margin: log(1 + exp(x)), slope sigmoid(x)
    const float h = soft ? (fmaxf(x, 0.f) + log1pf(expf(-fabsf(x)))) : fmaxf(x + margin, 0.f);
    // a hinge of exactly 0 passes the gradient, like torch's clamp_min / MarginRankingLoss
    const float slope = soft ? 1.f / (1.f + expf(-x)) : ((x + margin >= 0.f) ? 1.f : 0.f);
    o.a_row[a] = active ? a : -1;
    o.p_row[a] = pidx;
    o.n_row[a] = nidx;
    o.d_ap[a] = dap;
    o.d_an[a] = dan;
    o.hinge[a] = (active && nidx >= 0) ? h : 0.f;
    const bool on = active && nidx >= 0 && slope > 0.f;
    if (cosine) {
      // coefficients of d(loss)/d(cos): the combine step is dXn = -Cm Xn (no 1/d factor, no diagonal term)
      float gp = 0.f, gn = 0.f;
      pair_dist_cos(G, N, a, pidx, &gp);
      if (nidx >= 0) pair_dist_cos(G, N, a, nidx, &gn);
      o.cap[a] = on ? slope * gp : 0.f;
      o.can[a] = on ? slope * gn : 0.f;
    } else {
      bool sp, sn;
      pair_dist(G, N, sq, a, pidx, &sp);
      if (nidx >= 0) pair_dist(G, N, sq, a, nidx, &sn); else sn = true;
      o.cap[a] = (on && !sp) ? slope / dap : 0.f;   // scaled by the problem weight later
      o.can[a] = (on && !sn) ? slope / dan : 0.f;
    }
  }
}

// rows / max(|row|, 1e-12) (cosine_similarity, triplet_loss.py:44-55) and the norms
__global__ void __launch_bounds__(256) normalize_rows_kernel(const float* __restrict__ X, int D, float* __restrict__ Xn,
                                                             float* __restrict__ norm) {
  __shared__ float sm[8];
  const int i = blockIdx.x;
  float ss = 0.f;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const float v = X[(size_t)i * D + j];
    ss = __fmaf_rn(v, v, ss);
  }
  ss = block_sum(ss, sm);
  const float nr = fmaxf(__fsqrt_rn(ss), 1e-12f);
  for (int j = threadIdx.x; j < D; j += blockDim.x) Xn[(size_t)i * D + j] = __fdiv_rn(X[(size_t)i * D + j], nr);
  if (threadIdx.x == 0) norm[i] = nr;
}
// backward of the row normalisation: dX = (dXn - Xn (Xn . dXn)) / |x|, with dXn = dEm (= -Cm Xn);
// rows whose norm was clamped are constant multiples of x (x / 1e-12): dX = dXn / 1e-12
__global__ void __launch_bounds__(256) cosine_combine_kernel(const float* __restrict__ Xn, const float* __restrict__ X, int D,
                                                             const float* __restrict__ dXn, const float* __restrict__ norm,
                                                             float* __restrict__ dX) {
  __shared__ float sm[8];
  const int i = blockIdx.x;
  float dot = 0.f;
  for (int j = threadIdx.x; j < D; j += blockDim.x) dot = __fmaf_rn(Xn[(size_t)i * D + j], dXn[(size_t)i * D + j], dot);
  dot = block_sum(dot, sm);
  const float nr = norm[i];
  const bool clamped = nr <= 1e-12f;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const float g = dXn[(size_t)i * D + j];
    dX[(size_t)i * D + j] = clamped ? g / nr : (g - Xn[(size_t)i * D + j] * dot) / nr;
  }
}

// fused CTL step: slot layout documented at step_setup_kernel.  One block per slot.
__global__ void __launch_bounds__(128) mine_step_kernel(const float* __restrict__ G, int NT,
                                                        const float* __restrict__ sq, int B, int P, int K,
                                                        const unsigned char* __restrict__ is_real,
                                                        const StepMeta* __restrict__ meta, float margin, MineOut o) {
  __shared__ float s_v[128];
  __shared__ int s_i[128];
  const int t = blockIdx.x;
  int a_row, my_class, prob;  // prob 0 = image level, r+1 = round r
  bool active;
  if (t < B) {
    a_row = t; my_class = t / K; prob = 0; active = is_real[t];
  } else {
    const int u = t - B, r = u / (2 * P), w = u % (2 * P), c = w % P;
    prob = r + 1; my_class = c;
    a_row = (w < P) ? (c * K + r) : (B + r * P + c);
    active = meta->round_valid[r] && is_real[c * K + r];
  }
  float best_p = -CUDART_INF_F, best_n = CUDART_INF_F;
  int ip = -1, in = -1;
  if (active) {
    const int n_cand = prob == 0 ? B : 2 * P;
    for (int jj = threadIdx.x; jj < n_cand; jj += blockDim.x) {
      int j_row, j_class;
      bool j_ok = true;
      if (prob == 0) {
        j_row = jj; j_class = jj / K;  // mock rows ARE candidates (A.1)
      } else {
        const int r = prob - 1, c = jj % P;
        j_class = c;
        j_row = (jj < P) ? (c * K + r) : (B + r * P + c);
        j_ok = is_real[c * K + r];
      }
      if (!j_ok) continue;
      bool sat;
      const float d = pair_dist(G, NT, sq, a_row, j_row, &sat);
      if (j_class == my_class) {
        if (d > best_p) { best_p = d; ip = j_row; }
      } else {
        if (d < best_n) { best_n = d; in = j_row; }
      }
    }
  }
  s_v[threadIdx.x] = best_p; s_i[threadIdx.x] = ip;
  __syncthreads();
  for (int st = 64; st > 0; st >>= 1) {
    if (threadIdx.x < st) {
      const float v2 = s_v[threadIdx.x + st]; const int i2 = s_i[threadIdx.x + st];
      if (i2 >= 0 && (s_i[threadIdx.x] < 0 || v2 > s_v[threadIdx.x] || (v2 == s_v[threadIdx.x] && i2 < s_i[threadIdx.x]))) {
        s_v[threadIdx.x] = v2; s_i[threadIdx.x] = i2;
      }
    }
    __syncthreads();
  }
  const float dap = s_v[0]; const int pidx = s_i[0];
  __syncthreads();
  s_v[threadIdx.x] = best_n; s_i[threadIdx.x] = in;
  __syncthreads();
  for (int st = 64; st > 0; st >>= 1) {
    if (threadIdx.x < st) {
      const float v2 = s_v[threadIdx.x + st]; const int i2 = s_i[threadIdx.x + st];
      if (i2 >= 0 && (s_i[threadIdx.x] < 0 || v2 < s_v[threadIdx.x] || (v2 == s_v[threadIdx.x] && i2 < s_i[threadIdx.x]))) {
        s_v[threadIdx.x] = v2; s_i[threadIdx.x] = i2;
      }
    }
    __syncthreads();
  }
  const float dan = s_v[0]; const int nidx = s_i[0];
  if (threadIdx.x == 0) {
    const bool ok = active && pidx >= 0 && nidx >= 0;
    const float h = ok ? dap - dan + margin : 0.f;
    o.a_row[t] = ok ? a_row : -1;
    o.p_row[t] = pidx;
    o.n_row[t] = nidx;
    o.d_ap[t] = ok ? dap : 0.f;
    o.d_an[t] = ok ? dan : 0.f;
    o.hinge[t] = ok ? fmaxf(h, 0.f) : 0.f;
    bool sp = true, sn = true;
    if (ok) { pair_dist(G, NT, sq, a_row, pidx, &sp); pair_dist(G, NT, sq, a_row, nidx, &sn); }
    const bool on = ok && h >= 0.f;  // a hinge of exactly 0 passes the gradient (torch's clamp_min)
    o.cap[t] = (on && !sp) ? 1.f / dap : 0.f;
    o.can[t] = (on && !sn) ? 1.f / dan : 0.f;
  }
}

// ---------------------------------------------------------------------------------------
// loss reduction + per-slot gradient weights (single block, fixed order)
// out[0..7] = total, xent, triplet, center, ctl, dist_ap, dist_an, l2_centroid
// ---------------------------------------------------------------------------------------
__global__ void step_reduce_kernel(int B, int P, int K, const StepMeta* __restrict__ meta, MineOut o,
                                   const float* __restrict__ sq, const unsigned char* __restrict__ is_real,
                                   float w_triplet, float w_ctl, float* __restrict__ slot_w /*[T]*/,
                                   float* __restrict__ out) {
  // executed by one thread: T <= a few thousand, deterministic order
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int n_real = meta->n_real;
  float lq = 0.f;
  for (int t = 0; t < B; ++t) lq += o.hinge[t];
  lq = n_real > 0 ? lq / (float)n_real : 0.f;
  for (int t = 0; t < B; ++t) slot_w[t] = n_real > 0 ? w_triplet / (float)n_real : 0.f;
  float lc = 0.f, sap = 0.f, san = 0.f, sl2 = 0.f;
  const int nvr = meta->n_valid_rounds;
  for (int r = 0; r < K; ++r) {
    const int base = B + r * 2 * P;
    if (!meta->round_valid[r]) {
      for (int w = 0; w < 2 * P; ++w) slot_w[base + w] = 0.f;
      continue;
    }
    const int n_anchor = 2 * meta->round_classes[r];
    float h = 0.f, ap = 0.f, an = 0.f, l2 = 0.f;
    for (int w = 0; w < 2 * P; ++w) { h += o.hinge[base + w]; ap += o.d_ap[base + w]; an += o.d_an[base + w]; }
    for (int c = 0; c < P; ++c)
      if (is_real[c * K + r]) l2 += __fsqrt_rn(sq[B + r * P + c]);
    lc += h / (float)n_anchor;
    sap += ap / (float)n_anchor;
    san += an / (float)n_anchor;
    sl2 += l2 / (float)meta->round_classes[r];
    for (int w = 0; w < 2 * P; ++w) slot_w[base + w] = w_ctl / ((float)nvr * (float)n_anchor);
  }
  out[2] = lq * w_triplet;
  out[4] = nvr > 0 ? (lc / (float)nvr) * w_ctl : 0.f;
  out[5] = nvr > 0 ? sap / (float)nvr : 0.f;
  out[6] = nvr > 0 ? san / (float)nvr : 0.f;
  out[7] = nvr > 0 ? sl2 / (float)nvr : 0.f;
}

// Cm[i][j] = sum over anchor slots of row i and of row j (each row owns <= 2 slots)
__device__ __forceinline__ float slot_pair(const MineOut& o, const float* slot_w, int t, int other) {
  if (t < 0 || o.a_row[t] < 0) return 0.f;
  float v = 0.f;
  if (o.p_row[t] == other) v += slot_w[t] * o.cap[t];
  if (o.n_row[t] == other) v -= slot_w[t] * o.can[t];
  return v;
}
__device__ __forceinline__ void row_slots_step(int row, int B, int P, int K, int* s0, int* s1) {
  if (row < B) {
    const int c = row / K, s = row % K;
    *s0 = row;
    *s1 = B + s * 2 * P + c;
  } else {
    const int rc = row - B, r = rc / P, c = rc % P;
    *s0 = B + r * 2 * P + P + c;
    *s1 = -1;
  }
}
__global__ void build_coef_kernel(int NT, int B, int P, int K, int single, MineOut o, const float* __restrict__ slot_w,
                                  float* __restrict__ Cm, float* __restrict__ rowsum) {
  __shared__ float sm[8];
  const int i = blockIdx.x;
  int i0, i1;
  if (single) { i0 = i; i1 = -1; } else row_slots_step(i, B, P, K, &i0, &i1);
  float rs = 0.f;
  for (int j = threadIdx.x; j < NT; j += blockDim.x) {
    int j0, j1;
    if (single) { j0 = j; j1 = -1; } else row_slots_step(j, B, P, K, &j0, &j1);
    const float v = slot_pair(o, slot_w, i0, j) + slot_pair(o, slot_w, i1, j) + slot_pair(o, slot_w, j0, i) +
                    slot_pair(o, slot_w, j1, i);
    Cm[(size_t)i * NT + j] = v;
    rs += v;
  }
  rs = block_sum(rs, sm);
  if (threadIdx.x == 0) rowsum[i] = rs;
}

// ---------------------------------------------------------------------------------------
// center loss (losses/center_loss.py:26-45) on the gathered center rows
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) center_rows_kernel(const float* __restrict__ F, int D,
                                                          const int* __restrict__ labels,
                                                          const unsigned char* __restrict__ is_real,
                                                          const float* __restrict__ centers,
                                                          float* __restrict__ row_val /*[B]*/,
                                                          unsigned char* __restrict__ row_sat) {
  __shared__ float sm[8];
  const int b = blockIdx.x;
  const bool real = is_real == nullptr || is_real[b];
  float xx = 0.f, cc = 0.f, xc = 0.f;
  if (real) {
    const float* x = F + (size_t)b * D;
    const float* c = centers + (size_t)labels[b] * D;
    for (int j = threadIdx.x; j < D; j += blockDim.x) {
      const float xv = x[j], cv = c[j];
      xx = __fmaf_rn(xv, xv, xx);
      cc = __fmaf_rn(cv, cv, cc);
      xc = __fmaf_rn(xv, cv, xc);
    }
  }
  xx = block_sum(xx, sm);
  cc = block_sum(cc, sm);
  xc = block_sum(xc, sm);
  if (threadIdx.x == 0) {
    const float s = __fmaf_rn(-2.f, xc, __fadd_rn(xx, cc));
    row_val[b] = real ? fminf(fmaxf(s, 1e-12f), 1e12f) : 0.f;
    row_sat[b] = (!real || s < 1e-12f || s > 1e12f) ? 1 : 0;
  }
}

// d(centers)[y] = -2 w / B' * sum_{b: label b == y, real, unsaturated} (F_b - c_y), rows of a
// class visited in batch order.  One block per DISTINCT label occurrence (first row of it).
__global__ void __launch_bounds__(256) center_grad_kernel(const float* __restrict__ F, int B, int D,
                                                          const int* __restrict__ labels,
                                                          const unsigned char* __restrict__ is_real,
                                                          const unsigned char* __restrict__ row_sat,
                                                          const float* __restrict__ centers, const int* n_real_ptr,
                                                          int n_real_host, float w, float* __restrict__ d_centers) {
  const int b0 = blockIdx.x;
  const int y = labels[b0];
  for (int b = 0; b < b0; ++b)
    if (labels[b] == y) return;  // not the first occurrence of this label
  const int n_real = n_real_ptr ? *n_real_ptr : n_real_host;
  const float g = n_real > 0 ? -2.f * w / (float)n_real : 0.f;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const float cv = centers[(size_t)y * D + j];
    float acc = 0.f;
    for (int b = b0; b < B; ++b)
      if (labels[b] == y && (is_real == nullptr || is_real[b]) && !row_sat[b])
        acc = __fadd_rn(acc, __fsub_rn(F[(size_t)b * D + j], cv));
    d_centers[(size_t)y * D + j] = g * acc;
  }
}

// ---------------------------------------------------------------------------------------
// head: BatchNorm1d (batch statistics over the real rows) -> logits -> label-smoothed CE
// ---------------------------------------------------------------------------------------
// per feature j: mean / biased var over real rows; writes xhat (0 for mock rows), updates the
// running statistics like nn.BatchNorm1d (momentum, unbiased running var).
__global__ void __launch_bounds__(256) bn_forward_kernel(const float* __restrict__ F, int B, int D,
                                                         const unsigned char* __restrict__ is_real,
                                                         const float* __restrict__ gamma,
                                                         const float* __restrict__ beta, float eps, float momentum,
                                                         int training, float* __restrict__ run_mean,
                                                         float* __restrict__ run_var, float* __restrict__ xhat,
                                                         float* __restrict__ y, float* __restrict__ inv_std) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= D) return;
  float mean, var;
  int n = 0;
  if (training) {
    float s = 0.f;
    for (int b = 0; b < B; ++b)
      if (is_real == nullptr || is_real[b]) { s = __fadd_rn(s, F[(size_t)b * D + j]); ++n; }
    mean = n > 0 ? s / (float)n : 0.f;
    float v = 0.f;
    for (int b = 0; b < B; ++b)
      if (is_real == nullptr || is_real[b]) { const float dlt = F[(size_t)b * D + j] - mean; v = __fmaf_rn(dlt, dlt, v); }
    var = n > 0 ? v / (float)n : 0.f;
    if (run_mean) {
      run_mean[j] = (1.f - momentum) * run_mean[j] + momentum * mean;
      const float unb = n > 1 ? v / (float)(n - 1) : var;
      run_var[j] = (1.f - momentum) * run_var[j] + momentum * unb;
    }
  } else {
    mean = run_mean[j];
    var = run_var[j];
  }
  const float istd = 1.f / __fsqrt_rn(var + eps);
  inv_std[j] = istd;
  const float g = gamma[j], bt = beta[j];
  for (int b = 0; b < B; ++b) {
    const bool real = is_real == nullptr || is_real[b];
    const float xh = real ? (F[(size_t)b * D + j] - mean) * istd : 0.f;
    xhat[(size_t)b * D + j] = xh;
    y[(size_t)b * D + j] = real ? __fmaf_rn(xh, g, bt) : 0.f;
  }
}

// one block per row: log-softmax, loss row, d(logits) = w/B' (softmax - t) in place
__global__ void __launch_bounds__(256) xent_rows_kernel(float* __restrict__ logits, int C, const int* __restrict__ labels,
                                                        const unsigned char* __restrict__ is_real,
                                                        const int* n_real_ptr, int n_real_host, float epsilon, float w,
                                                        float* __restrict__ row_loss) {
  __shared__ float sm[8];
  __shared__ float s_max;
  const int b = blockIdx.x;
  float* z = logits + (size_t)b * C;
  const bool real = is_real == nullptr || is_real[b];
  if (!real) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) z[c] = 0.f;
    if (threadIdx.x == 0) row_loss[b] = 0.f;
    return;
  }
  float mx = -CUDART_INF_F;
  for (int c = threadIdx.x; c < C; c += blockDim.x) mx = fmaxf(mx, z[c]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = sm[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) m = fmaxf(m, sm[i]);
    s_max = m;
  }
  __syncthreads();
  mx = s_max;
  float se = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) se += expf(z[c] - mx);
  se = block_sum(se, sm);
  const float lse = mx + logf(se);
  const int y = labels[b];
  const int n_real = n_real_ptr ? *n_real_ptr : n_real_host;
  const float scale = n_real > 0 ? w / (float)n_real : 0.f;
  const float t_off = epsilon / (float)C, t_on = (1.f - epsilon) + t_off;
  float l = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float logp = z[c] - lse;
    const float t = (c == y) ? t_on : t_off;
    l = __fmaf_rn(-t, logp, l);
    z[c] = scale * (expf(logp) - t);
  }
  l = block_sum(l, sm);
  if (threadIdx.x == 0) row_loss[b] = l;
}

// BN backward per feature (training statistics): dgamma_j and d(F) contribution
__global__ void __launch_bounds__(256) bn_backward_kernel(const float* __restrict__ dy, const float* __restrict__ xhat,
                                                          int B, int D, const unsigned char* __restrict__ is_real,
                                                          const float* __restrict__ gamma,
                                                          const float* __restrict__ inv_std, int training,
                                                          float* __restrict__ dgamma, float* __restrict__ dF_head) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= D) return;
  float s1 = 0.f, s2 = 0.f;
  int n = 0;
  for (int b = 0; b < B; ++b)
    if (is_real == nullptr || is_real[b]) {
      const float g = dy[(size_t)b * D + j];
      s1 = __fadd_rn(s1, g);
      s2 = __fmaf_rn(g, xhat[(size_t)b * D + j], s2);
      ++n;
    }
  dgamma[j] = s2;
  const float g = gamma[j], is = inv_std[j];
  const float m1 = n > 0 ? s1 / (float)n : 0.f, m2 = n > 0 ? s2 / (float)n : 0.f;
  for (int b = 0; b < B; ++b) {
    const bool real = is_real == nullptr || is_real[b];
    float v = 0.f;
    if (real) {
      const float d = dy[(size_t)b * D + j];
      v = training ? g * is * (d - m1 - xhat[(size_t)b * D + j] * m2) : g * is * d;
    }
    dF_head[(size_t)b * D + j] = v;
  }
}

// final scalar assembly (center + xent) and the feature-gradient combine
__global__ void step_scalars_kernel(int B, int C, const StepMeta* __restrict__ meta, const float* __restrict__ center_rows,
                                    const float* __restrict__ xent_rows, float w_center, float w_xent,
                                    float* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int n = meta->n_real;
  float cs = 0.f, xs = 0.f;
  for (int b = 0; b < B; ++b) { cs += center_rows[b]; xs += xent_rows[b]; }
  // each of the B'(C-1) masked zeros is clamped to 1e-12 (center_loss.py:43-44)
  const float center = n > 0 ? w_center * (cs + (float)n * (float)(C - 1) * 1e-12f) / (float)n : 0.f;
  const float xent = n > 0 ? w_xent * xs / (float)n : 0.f;
  out[1] = xent;
  out[3] = center;
  out[0] = out[4] + center + xent + out[2];  // train_ctl_model.py:150-152 order
  if (meta->bad_batch) {  // contract violation: poison every reported value (the shim turns this into ValueError)
    for (int i = 0; i < 8; ++i) out[i] = __int_as_float(0x7fc00000 | meta->bad_batch);
  }
}

__global__ void __launch_bounds__(256) combine_grad_kernel(const float* __restrict__ F, int B, int D, int P, int K,
                                                           const unsigned char* __restrict__ is_real,
                                                           const int* __restrict__ n_rc, const float* __restrict__ E_cent,
                                                           const float* __restrict__ dE /* = -Cm E_all */,
                                                           const float* __restrict__ rowsum,
                                                           const float* __restrict__ dF_head,
                                                           const int* __restrict__ labels,
                                                           const float* __restrict__ centers,
                                                           const unsigned char* __restrict__ row_sat,
                                                           const StepMeta* __restrict__ meta, float w_center,
                                                           float* __restrict__ dF) {
  const int i = blockIdx.x, c = i / K, s = i % K;
  const bool real = is_real[i];
  const int n_real = meta->n_real;
  const float gc = (real && !row_sat[i] && n_real > 0) ? 2.f * w_center / (float)n_real : 0.f;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const float f = F[(size_t)i * D + j];
    float g = __fmaf_rn(rowsum[i], f, dE[(size_t)i * D + j]);
    if (real)
      for (int r = 0; r < K; ++r) {
        const int n = n_rc[r * P + c];
        if (r != s && n > 0 && is_real[c * K + r]) {
          const int row = B + r * P + c;
          const float gcent = __fmaf_rn(rowsum[row], E_cent[(size_t)(row - B) * D + j], dE[(size_t)row * D + j]);
          g = __fadd_rn(g, __fdiv_rn(gcent, (float)n));
        }
      }
    g = __fadd_rn(g, dF_head[(size_t)i * D + j]);
    if (gc != 0.f) g = __fmaf_rn(gc, f - centers[(size_t)labels[i] * D + j], g);
    dF[(size_t)i * D + j] = g;
  }
}

// standalone triplet: dE_i = rowsum_i * E_i - (Cm E)_i, loss = sum(hinge)/n_active
__global__ void __launch_bounds__(256) single_combine_kernel(const float* __restrict__ E, int D,
                                                             const float* __restrict__ dEm,
                                                             const float* __restrict__ rowsum, float* __restrict__ dE) {
  const int i = blockIdx.x;
  for (int j = threadIdx.x; j < D; j += blockDim.x)
    dE[(size_t)i * D + j] = __fmaf_rn(rowsum[i], E[(size_t)i * D + j], dEm[(size_t)i * D + j]);
}
__global__ void single_reduce_kernel(int N, MineOut o, float weight, float* __restrict__ slot_w, float* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int n = 0;
  float h = 0.f;
  for (int t = 0; t < N; ++t)
    if (o.a_row[t] >= 0) { ++n; h += o.hinge[t]; }
  out[0] = n > 0 ? weight * h / (float)n : 0.f;
  for (int t = 0; t < N; ++t) slot_w[t] = n > 0 ? weight / (float)n : 0.f;
}
__global__ void sqnorm_rows_kernel(const float* __restrict__ X, int D, float* __restrict__ sq) {
  __shared__ float sm[8];
  float ss = 0.f;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const float v = X[(size_t)blockIdx.x * D + j];
    ss = __fmaf_rn(v, v, ss);
  }
  ss = block_sum(ss, sm);
  if (threadIdx.x == 0) sq[blockIdx.x] = ss;
}
__global__ void sum_rows_kernel(const float* __restrict__ v, int n, float scale, float add, float* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float s = 0.f;
  for (int i = 0; i < n; ++i) s += v[i];
  out[0] = (s + add) * scale;
}

__global__ void center_dx_kernel(const float* __restrict__ x, int d, const int* __restrict__ labels,
                                 const float* __restrict__ centers, const unsigned char* __restrict__ sat, int b,
                                 float* __restrict__ dx) {
  const int i = blockIdx.x;
  const float g = sat[i] ? 0.f : 2.f / (float)b;
  for (int j = threadIdx.x; j < d; j += blockDim.x)
    dx[(size_t)i * d + j] = g * (x[(size_t)i * d + j] - centers[(size_t)labels[i] * d + j]);
}

static MineOut take_mine(Workspace& ws, int T) {
  MineOut o;
  o.a_row = ws.take<int>(T);
  o.p_row = ws.take<int>(T);
  o.n_row = ws.take<int>(T);
  o.cap = ws.take<float>(T);
  o.can = ws.take<float>(T);
  o.hinge = ws.take<float>(T);
  o.d_ap = ws.take<float>(T);
  o.d_an = ws.take<float>(T);
  return o;
}

struct StepBuffers {
  StepMeta* meta;
  int* n_rc;
  float *E_all, *sq, *G, *Cm, *rowsum, *dE, *slot_w;
  MineOut mine;
  float *center_rows, *xent_rows, *xhat, *y, *inv_std, *logits, *dy, *dF_head;
  unsigned char* row_sat;
  int* labels_safe;
  bool ok;
};

static StepBuffers carve_step(Workspace& ws, const ctl_loss_config& c) {
  StepBuffers b;
  const int NT = c.B + c.K * c.P, T = c.B + 2 * c.P * c.K;
  b.meta = ws.take<StepMeta>(1);
  b.n_rc = ws.take<int>((size_t)c.K * c.P);
  b.E_all = ws.take<float>((size_t)NT * c.D);
  b.sq = ws.take<float>(NT);
  b.G = ws.take<float>((size_t)NT * NT);
  b.Cm = ws.take<float>((size_t)NT * NT);
  b.rowsum = ws.take<float>(NT);
  b.dE = ws.take<float>((size_t)NT * c.D);
  b.slot_w = ws.take<float>(T);
  b.mine = take_mine(ws, T);
  b.center_rows = ws.take<float>(c.B);
  b.xent_rows = ws.take<float>(c.B);
  b.xhat = ws.take<float>((size_t)c.B * c.D);
  b.y = ws.take<float>((size_t)c.B * c.D);
  b.inv_std = ws.take<float>(c.D);
  b.logits = ws.take<float>((size_t)c.B * c.C);
  b.dy = ws.take<float>((size_t)c.B * c.D);
  b.dF_head = ws.take<float>((size_t)c.B * c.D);
  b.row_sat = ws.take<unsigned char>(c.B);
  b.labels_safe = ws.take<int>(c.B);
  b.ok = b.labels_safe != nullptr && b.meta != nullptr;
  return b;
}

static int check_cfg(const ctl_loss_config* c) {
  CTL_CHECK_ARG(c != nullptr, "null config");
  CTL_CHECK_ARG(c->P >= 1 && c->K >= 1 && c->K <= 64 && c->B == c->P * c->K,
                "batch contract: B = P*K pid-major, K <= 64 (B=%d P=%d K=%d)", c->B, c->P, c->K);
  CTL_CHECK_ARG(c->D >= 1 && c->C >= 1, "bad dims D=%d C=%d", c->D, c->C);
  return 0;
}

}  // namespace ctl

using namespace ctl;

extern "C" {

size_t ctl_loss_workspace_bytes(const ctl_loss_config* cfg) {
  if (check_cfg(cfg)) return 0;
  Workspace ws(nullptr, 0);
  carve_step(ws, *cfg);
  return ws.off;
}

int ctl_loss_step(const ctl_loss_config* cfg, const float* feats, const int32_t* labels, const uint8_t* is_real,
                  const float* centers, const float* bn_weight, const float* bn_bias, float* bn_running_mean,
                  float* bn_running_var, const float* fc_weight, float* out_losses, float* d_feats, float* d_centers,
                  float* d_bn_weight, float* d_fc_weight, void* workspace, size_t workspace_bytes,
                  ctl_stream_t stream_) {
  int rc = check_cfg(cfg);
  if (rc) return rc;
  CTL_CHECK_ARG(feats && labels && is_real && centers && bn_weight && bn_bias && fc_weight && out_losses && d_feats &&
                    d_centers && d_bn_weight && d_fc_weight && workspace,
                "null pointer");
  if ((rc = ctl_device_check())) return rc;
  cudaStream_t st = (cudaStream_t)stream_;
  const ctl_loss_config& c = *cfg;
  const int B = c.B, D = c.D, P = c.P, K = c.K, C = c.C;
  const int NT = B + K * P, T = B + 2 * P * K;
  Workspace ws(workspace, workspace_bytes);
  StepBuffers b = carve_step(ws, c);
  if (!b.ok) {
    set_error("workspace too small: need %zu bytes, have %zu", ws.off, workspace_bytes);
    return CTL_ERR_WORKSPACE;
  }
  // ---- metadata, centroid rows, norms --------------------------------------------------
  step_setup_kernel<<<1, 128, 0, st>>>(is_real, labels, C, P, K, b.meta, b.n_rc, b.labels_safe);
  labels = b.labels_safe;  // range-checked copy: no kernel below can index centers / logits out of bounds
  CTL_LAUNCH_CHECK();
  CTL_CUDA(cudaMemcpyAsync(b.E_all, feats, (size_t)B * D * sizeof(float), cudaMemcpyDeviceToDevice, st));
  build_rows_kernel<<<NT, 256, 0, st>>>(feats, B, D, P, K, is_real, b.n_rc, b.E_all + (size_t)B * D, b.sq);
  CTL_LAUNCH_CHECK();
  // ---- Gram, mining, loss reduction ----------------------------------------------------
  if ((rc = sgemm(st, NT, NT, D, b.E_all, D, 1, b.E_all, 1, D, b.G, NT, 1.f, 0.f))) return rc;
  mine_step_kernel<<<T, 128, 0, st>>>(b.G, NT, b.sq, B, P, K, is_real, b.meta, c.margin, b.mine);
  CTL_LAUNCH_CHECK();
  step_reduce_kernel<<<1, 32, 0, st>>>(B, P, K, b.meta, b.mine, b.sq, is_real, c.triplet_weight, c.ctl_weight, b.slot_w,
                                      out_losses);
  CTL_LAUNCH_CHECK();
  // ---- triplet backward: dE = rowsum*E - Cm E -------------------------------------------
  build_coef_kernel<<<NT, 128, 0, st>>>(NT, B, P, K, 0, b.mine, b.slot_w, b.Cm, b.rowsum);
  CTL_LAUNCH_CHECK();
  if ((rc = sgemm(st, NT, D, NT, b.Cm, NT, 1, b.E_all, D, 1, b.dE, D, -1.f, 0.f))) return rc;
  // ---- center loss ---------------------------------------------------------------------
  center_rows_kernel<<<B, 256, 0, st>>>(feats, D, labels, is_real, centers, b.center_rows, b.row_sat);
  CTL_LAUNCH_CHECK();
  CTL_CUDA(cudaMemsetAsync(d_centers, 0, (size_t)C * D * sizeof(float), st));
  center_grad_kernel<<<B, 256, 0, st>>>(feats, B, D, labels, is_real, b.row_sat, centers, &b.meta->n_real, 0,
                                        c.center_weight, d_centers);
  CTL_LAUNCH_CHECK();
  // ---- head: BN1d -> fc -> label-smoothed CE, and its backward ---------------------------
  bn_forward_kernel<<<(D + 255) / 256, 256, 0, st>>>(feats, B, D, is_real, bn_weight, bn_bias, c.bn_eps, c.bn_momentum,
                                                   1, bn_running_mean, bn_running_var, b.xhat, b.y, b.inv_std);
  CTL_LAUNCH_CHECK();
  if ((rc = sgemm(st, B, C, D, b.y, D, 1, fc_weight, 1, D, b.logits, C, 1.f, 0.f))) return rc;  // y W^T
  xent_rows_kernel<<<B, 256, 0, st>>>(b.logits, C, labels, is_real, &b.meta->n_real, 0, c.label_smooth, c.xent_weight,
                                      b.xent_rows);
  CTL_LAUNCH_CHECK();
  // logits now hold d(loss)/d(logits)
  if ((rc = sgemm(st, C, D, B, b.logits, 1, C, b.y, D, 1, d_fc_weight, D, 1.f, 0.f))) return rc;  // dZ^T y
  if ((rc = sgemm(st, B, D, C, b.logits, C, 1, fc_weight, D, 1, b.dy, D, 1.f, 0.f))) return rc;   // dZ W
  bn_backward_kernel<<<(D + 255) / 256, 256, 0, st>>>(b.dy, b.xhat, B, D, is_real, bn_weight, b.inv_std, 1, d_bn_weight,
                                                    b.dF_head);
  CTL_LAUNCH_CHECK();
  // ---- scalars + feature gradient -------------------------------------------------------
  step_scalars_kernel<<<1, 32, 0, st>>>(B, C, b.meta, b.center_rows, b.xent_rows, c.center_weight, c.xent_weight, out_losses);
  CTL_LAUNCH_CHECK();
  combine_grad_kernel<<<B, 256, 0, st>>>(feats, B, D, P, K, is_real, b.n_rc, b.E_all + (size_t)B * D, b.dE, b.rowsum,
                                         b.dF_head, labels, centers, b.row_sat, b.meta, c.center_weight, d_feats);
  CTL_LAUNCH_CHECK();
  return 0;
}

// ---- standalone drop-ins ------------------------------------------------------------------
size_t ctl_triplet_workspace_bytes(int32_t n, int32_t d) {
  Workspace ws(nullptr, 0);
  ws.take<float>(n);
  ws.take<float>((size_t)n * n);
  ws.take<float>((size_t)n * n);
  ws.take<float>(n);
  ws.take<float>((size_t)n * d);
  ws.take<float>(n);
  take_mine(ws, n);
  ws.take<float>((size_t)n * d);  // normalised rows (cosine)
  ws.take<float>(n);              // row norms (cosine)
  return ws.off;
}

int ctl_triplet_step(const float* feats, int32_t n, int32_t d, const int32_t* labels, const uint8_t* anchor_mask,
                     float margin, float* out_loss, float* out_dist_ap, float* out_dist_an, float* d_feats,
                     void* workspace, size_t workspace_bytes, ctl_stream_t stream_) {
  return ctl_triplet_step_ex(feats, n, d, labels, anchor_mask, margin, 0, 0, out_loss, out_dist_ap, out_dist_an, d_feats,
                             workspace, workspace_bytes, stream_);
}

int ctl_triplet_step_ex(const float* feats, int32_t n, int32_t d, const int32_t* labels, const uint8_t* anchor_mask,
                        float margin, int32_t soft_margin, int32_t cosine, float* out_loss, float* out_dist_ap,
                        float* out_dist_an, float* d_feats, void* workspace, size_t workspace_bytes, ctl_stream_t stream_) {
  CTL_CHECK_ARG(feats && labels && out_loss && out_dist_ap && out_dist_an && d_feats && workspace, "null pointer");
  CTL_CHECK_ARG(n >= 2 && d >= 1, "bad shape n=%d d=%d", n, d);
  int rc = ctl_device_check();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream_;
  Workspace ws(workspace, workspace_bytes);
  float* sq = ws.take<float>(n);
  float* G = ws.take<float>((size_t)n * n);
  float* Cm = ws.take<float>((size_t)n * n);
  float* rowsum = ws.take<float>(n);
  float* dEm = ws.take<float>((size_t)n * d);
  float* slot_w = ws.take<float>(n);
  MineOut o = take_mine(ws, n);
  float* Xn = ws.take<float>((size_t)n * d);
  float* norm = ws.take<float>(n);
  if (!o.d_an || !norm) {
    set_error("workspace too small: need %zu bytes, have %zu", ws.off, workspace_bytes);
    return CTL_ERR_WORKSPACE;
  }
  const float* E = feats;  // the rows the Gram matrix is taken of
  if (cosine) {
    normalize_rows_kernel<<<n, 256, 0, st>>>(feats, d, Xn, norm);
    E = Xn;
  } else {
    sqnorm_rows_kernel<<<n, 256, 0, st>>>(feats, d, sq);
  }
  CTL_LAUNCH_CHECK();
  if ((rc = sgemm(st, n, n, d, E, d, 1, E, 1, d, G, n, 1.f, 0.f))) return rc;
  mine_single_kernel<<<n, 128, 0, st>>>(G, sq, labels, anchor_mask, n, margin, soft_margin ? 1 : 0, cosine ? 1 : 0, o);
  CTL_LAUNCH_CHECK();
  single_reduce_kernel<<<1, 32, 0, st>>>(n, o, 1.f, slot_w, out_loss);
  CTL_LAUNCH_CHECK();
  build_coef_kernel<<<n, 128, 0, st>>>(n, 0, 0, 1, 1, o, slot_w, Cm, rowsum);
  CTL_LAUNCH_CHECK();
  if ((rc = sgemm(st, n, d, n, Cm, n, 1, E, d, 1, dEm, d, -1.f, 0.f))) return rc;  // -Cm E
  if (cosine)
    cosine_combine_kernel<<<n, 256, 0, st>>>(Xn, feats, d, dEm, norm, d_feats);
  else
    single_combine_kernel<<<n, 256, 0, st>>>(feats, d, dEm, rowsum, d_feats);
  CTL_LAUNCH_CHECK();
  CTL_CUDA(cudaMemcpyAsync(out_dist_ap, o.d_ap, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  CTL_CUDA(cudaMemcpyAsync(out_dist_an, o.d_an, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

}  // extern "C"

namespace ctl {
// range check of a label vector: safe[i] = label in [0, C) ? label : 0; *bad != 0 if any label was out of range
__global__ void sanitize_labels_kernel(const int* __restrict__ labels, int n, int C, int* __restrict__ safe, int* __restrict__ bad) {
  __shared__ int s_bad;
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int y = labels[i];
    const bool oob = y < 0 || y >= C;
    if (oob) s_bad = 1;
    safe[i] = oob ? 0 : y;
  }
  __syncthreads();
  if (threadIdx.x == 0) *bad = s_bad;
}
__global__ void poison_if_kernel(const int* __restrict__ bad, float* __restrict__ out) {
  if (*bad) *out = __int_as_float(0x7fc00001);  // NaN with payload 1: label out of range
}
}  // namespace ctl

extern "C" {

int ctl_center_loss_step(const float* x, int32_t b, int32_t d, const int32_t* labels, const float* centers, int32_t c,
                         float* out_loss, float* d_x, float* d_centers, void* workspace, size_t workspace_bytes,
                         ctl_stream_t stream_) {
  CTL_CHECK_ARG(x && labels && centers && out_loss && d_x && d_centers && workspace, "null pointer");
  CTL_CHECK_ARG(b >= 1 && d >= 1 && c >= 1, "bad shape");
  int rc = ctl_device_check();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream_;
  Workspace ws(workspace, workspace_bytes);
  float* rows = ws.take<float>(b);
  unsigned char* sat = ws.take<unsigned char>(b);
  int* safe = ws.take<int>((size_t)b + 1);  // [b] range-checked labels + 1 flag
  if (!safe) {
    set_error("workspace too small: need %zu bytes, have %zu", ws.off, workspace_bytes);
    return CTL_ERR_WORKSPACE;
  }
  // labels index `centers`: an out-of-range label (num_classes mismatch) must not become an out-of-bounds access;
  // it is reported as a NaN loss (payload 1) that the Python shim turns into ValueError
  sanitize_labels_kernel<<<1, 256, 0, st>>>(labels, b, c, safe, safe + b);
  CTL_LAUNCH_CHECK();
  labels = safe;
  center_rows_kernel<<<b, 256, 0, st>>>(x, d, labels, nullptr, centers, rows, sat);
  CTL_LAUNCH_CHECK();
  sum_rows_kernel<<<1, 32, 0, st>>>(rows, b, 1.f / (float)b, (float)b * (float)(c - 1) * 1e-12f, out_loss);
  CTL_LAUNCH_CHECK();
  CTL_CUDA(cudaMemsetAsync(d_centers, 0, (size_t)c * d * sizeof(float), st));
  center_grad_kernel<<<b, 256, 0, st>>>(x, b, d, labels, nullptr, sat, centers, nullptr, b, 1.f, d_centers);
  CTL_LAUNCH_CHECK();
  center_dx_kernel<<<b, 256, 0, st>>>(x, d, labels, centers, sat, b, d_x);
  CTL_LAUNCH_CHECK();
  poison_if_kernel<<<1, 1, 0, st>>>(safe + b, out_loss);
  CTL_LAUNCH_CHECK();
  return 0;
}

int ctl_xent_smooth_step(const float* logits, int32_t b, int32_t c, const int32_t* targets, float epsilon,
                         float* out_loss, float* d_logits, void* workspace, size_t workspace_bytes,
                         ctl_stream_t stream_) {
  CTL_CHECK_ARG(logits && targets && out_loss && d_logits && workspace, "null pointer");
  CTL_CHECK_ARG(b >= 1 && c >= 1, "bad shape");
  int rc = ctl_device_check();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream_;
  Workspace ws(workspace, workspace_bytes);
  float* rows = ws.take<float>(b);
  if (!rows) {
    set_error("workspace too small: need %zu bytes, have %zu", ws.off, workspace_bytes);
    return CTL_ERR_WORKSPACE;
  }
  CTL_CUDA(cudaMemcpyAsync(d_logits, logits, (size_t)b * c * sizeof(float), cudaMemcpyDeviceToDevice, st));
  xent_rows_kernel<<<b, 256, 0, st>>>(d_logits, c, targets, nullptr, nullptr, b, epsilon, 1.f, rows);
  CTL_LAUNCH_CHECK();
  sum_rows_kernel<<<1, 32, 0, st>>>(rows, b, 1.f / (float)b, 0.f, out_loss);
  CTL_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------
// base-model step (train_base_model.py:38-96): query triplet over all B rows with the anchors
// masked to is_real, center loss and BN1d -> fc -> label-smoothed CE over ALL B rows (mock rows
// included).  The kernels above do the work; only the scalar assembly and the final row-wise
// combine of the three feature-gradient terms are specific to this step.
// ---------------------------------------------------------------------------------------
namespace ctl {

// out[0..5] = total, xent, triplet (already written by single_reduce_kernel), center, dist_ap, dist_an
__global__ void base_scalars_kernel(int B, int C, MineOut o, const float* __restrict__ center_rows,
                                    const float* __restrict__ xent_rows, float w_center, float w_xent,
                                    const int* __restrict__ bad, float* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float cs = 0.f, xs = 0.f, sap = 0.f, san = 0.f;
  int n_anchor = 0;
  for (int b = 0; b < B; ++b) {
    cs += center_rows[b];
    xs += xent_rows[b];
    if (o.a_row[b] >= 0) { sap += o.d_ap[b]; san += o.d_an[b]; ++n_anchor; }
  }
  // every one of the B(C-1) masked zeros is clamped to 1e-12 (center_loss.py:43-44)
  const float center = w_center * (cs + (float)B * (float)(C - 1) * 1e-12f) / (float)B;
  const float xent = w_xent * xs / (float)B;
  out[1] = xent;
  out[3] = center;
  out[0] = center + xent + out[2];  // train_base_model.py:75 order
  // train_base_model.py:91-94: means over the masked (real) anchors
  out[4] = n_anchor > 0 ? sap / (float)n_anchor : 0.f;
  out[5] = n_anchor > 0 ? san / (float)n_anchor : 0.f;
  if (*bad)  // a label outside [0, C): poison every reported value (payload 1; the shim raises ValueError)
    for (int i = 0; i < 6; ++i) out[i] = __int_as_float(0x7fc00001);
}

// dF = triplet term + BN/head term + center term.  The triplet term is rowsum_i F_i - (Cm F)_i (euclidean) or, for
// cosine, already in dF (cosine_combine_kernel wrote the gradient through the row normalisation there).
__global__ void __launch_bounds__(256) base_combine_kernel(const float* __restrict__ F, int B, int D, int cosine,
                                                           const float* __restrict__ dEm, const float* __restrict__ rowsum,
                                                           const float* __restrict__ dF_head,
                                                           const int* __restrict__ labels,
                                                           const float* __restrict__ centers,
                                                           const unsigned char* __restrict__ row_sat, float w_center,
                                                           float* __restrict__ dF) {
  const int i = blockIdx.x;
  const float gc = row_sat[i] ? 0.f : 2.f * w_center / (float)B;
  const float* c = centers + (size_t)labels[i] * D;
  for (int j = threadIdx.x; j < D; j += blockDim.x) {
    const size_t k = (size_t)i * D + j;
    const float f = F[k];
    float g = cosine ? dF[k] : __fmaf_rn(rowsum[i], f, dEm[k]);
    g = __fadd_rn(g, dF_head[k]);
    if (gc != 0.f) g = __fmaf_rn(gc, f - c[j], g);
    dF[k] = g;
  }
}

struct BaseBuffers {
  int* labels_safe;  // [B + 1]: range-checked labels, then the out-of-range flag
  float *sq, *Xn, *norm, *G, *Cm, *rowsum, *dEm, *slot_w;
  MineOut mine;
  float *center_rows, *xent_rows, *xhat, *y, *inv_std, *logits, *dy, *dF_head;
  unsigned char* row_sat;
  bool ok;
};

static BaseBuffers carve_base(Workspace& ws, const ctl_base_loss_config& c) {
  BaseBuffers b;
  const int B = c.B, D = c.D;
  b.labels_safe = ws.take<int>((size_t)B + 1);
  b.sq = ws.take<float>(B);
  b.Xn = c.cosine ? ws.take<float>((size_t)B * D) : nullptr;
  b.norm = c.cosine ? ws.take<float>(B) : nullptr;
  b.G = ws.take<float>((size_t)B * B);
  b.Cm = ws.take<float>((size_t)B * B);
  b.rowsum = ws.take<float>(B);
  b.dEm = ws.take<float>((size_t)B * D);
  b.slot_w = ws.take<float>(B);
  b.mine = take_mine(ws, B);
  b.center_rows = ws.take<float>(B);
  b.xent_rows = ws.take<float>(B);
  b.xhat = ws.take<float>((size_t)B * D);
  b.y = ws.take<float>((size_t)B * D);
  b.inv_std = ws.take<float>(D);
  b.logits = ws.take<float>((size_t)B * c.C);
  b.dy = ws.take<float>((size_t)B * D);
  b.dF_head = ws.take<float>((size_t)B * D);
  b.row_sat = ws.take<unsigned char>(B);
  b.ok = b.labels_safe != nullptr && b.row_sat != nullptr;
  return b;
}

static int check_base_cfg(const ctl_base_loss_config* c) {
  CTL_CHECK_ARG(c != nullptr, "null config");
  CTL_CHECK_ARG(c->B >= 2 && c->D >= 1 && c->C >= 1, "bad dims B=%d D=%d C=%d", c->B, c->D, c->C);
  return 0;
}

}  // namespace ctl

extern "C" {

size_t ctl_base_loss_workspace_bytes(const ctl_base_loss_config* cfg) {
  if (check_base_cfg(cfg)) return 0;
  Workspace ws(nullptr, 0);
  carve_base(ws, *cfg);
  return ws.off;
}

int ctl_base_loss_step(const ctl_base_loss_config* cfg, const float* feats, const int32_t* labels,
                       const uint8_t* is_real, const float* centers, const float* bn_weight, const float* bn_bias,
                       float* bn_running_mean, float* bn_running_var, const float* fc_weight, float* out_losses,
                       float* d_feats, float* d_centers, float* d_bn_weight, float* d_fc_weight, void* workspace,
                       size_t workspace_bytes, ctl_stream_t stream_) {
  int rc = check_base_cfg(cfg);
  if (rc) return rc;
  CTL_CHECK_ARG(feats && labels && is_real && centers && bn_weight && bn_bias && fc_weight && out_losses && d_feats &&
                    d_centers && d_bn_weight && d_fc_weight && workspace,
                "null pointer");
  CTL_CHECK_ARG((bn_running_mean == nullptr) == (bn_running_var == nullptr), "running mean and var: both or neither");
  if ((rc = ctl_device_check())) return rc;
  cudaStream_t st = (cudaStream_t)stream_;
  const ctl_base_loss_config& c = *cfg;
  const int B = c.B, D = c.D, C = c.C;
  const int cosine = c.cosine ? 1 : 0;
  Workspace ws(workspace, workspace_bytes);
  BaseBuffers b = carve_base(ws, c);
  if (!b.ok) {
    set_error("workspace too small: need %zu bytes, have %zu", ws.off, workspace_bytes);
    return CTL_ERR_WORKSPACE;
  }
  // labels index `centers` and the logits: an out-of-range label becomes 0 here and poisons every output below
  sanitize_labels_kernel<<<1, 256, 0, st>>>(labels, B, C, b.labels_safe, b.labels_safe + B);
  CTL_LAUNCH_CHECK();
  labels = b.labels_safe;
  // ---- query triplet (train_base_model.py:60-65): Gram over all B rows, anchors masked to is_real ----------
  const float* E = feats;
  if (cosine) {
    normalize_rows_kernel<<<B, 256, 0, st>>>(feats, D, b.Xn, b.norm);
    E = b.Xn;
  } else {
    sqnorm_rows_kernel<<<B, 256, 0, st>>>(feats, D, b.sq);
  }
  CTL_LAUNCH_CHECK();
  if ((rc = sgemm(st, B, B, D, E, D, 1, E, 1, D, b.G, B, 1.f, 0.f))) return rc;
  mine_single_kernel<<<B, 128, 0, st>>>(b.G, b.sq, labels, is_real, B, c.margin, c.soft_margin ? 1 : 0, cosine, b.mine);
  CTL_LAUNCH_CHECK();
  single_reduce_kernel<<<1, 32, 0, st>>>(B, b.mine, c.triplet_weight, b.slot_w, out_losses + 2);
  CTL_LAUNCH_CHECK();
  build_coef_kernel<<<B, 128, 0, st>>>(B, 0, 0, 1, 1, b.mine, b.slot_w, b.Cm, b.rowsum);
  CTL_LAUNCH_CHECK();
  if ((rc = sgemm(st, B, D, B, b.Cm, B, 1, E, D, 1, b.dEm, D, -1.f, 0.f))) return rc;  // -Cm E
  if (cosine) {
    cosine_combine_kernel<<<B, 256, 0, st>>>(b.Xn, feats, D, b.dEm, b.norm, d_feats);
    CTL_LAUNCH_CHECK();
  }
  // ---- center loss over all B rows (train_base_model.py:67-69) ------------------------------------------
  center_rows_kernel<<<B, 256, 0, st>>>(feats, D, labels, nullptr, centers, b.center_rows, b.row_sat);
  CTL_LAUNCH_CHECK();
  CTL_CUDA(cudaMemsetAsync(d_centers, 0, (size_t)C * D * sizeof(float), st));
  center_grad_kernel<<<B, 256, 0, st>>>(feats, B, D, labels, nullptr, b.row_sat, centers, nullptr, B, c.center_weight,
                                        d_centers);
  CTL_LAUNCH_CHECK();
  // ---- head over all B rows (train_base_model.py:70-73): BN1d -> fc -> label-smoothed CE, and its backward --
  bn_forward_kernel<<<(D + 255) / 256, 256, 0, st>>>(feats, B, D, nullptr, bn_weight, bn_bias, c.bn_eps, c.bn_momentum,
                                                   1, bn_running_mean, bn_running_var, b.xhat, b.y, b.inv_std);
  CTL_LAUNCH_CHECK();
  if ((rc = sgemm(st, B, C, D, b.y, D, 1, fc_weight, 1, D, b.logits, C, 1.f, 0.f))) return rc;  // y W^T
  xent_rows_kernel<<<B, 256, 0, st>>>(b.logits, C, labels, nullptr, nullptr, B, c.label_smooth, c.xent_weight,
                                      b.xent_rows);
  CTL_LAUNCH_CHECK();
  // logits now hold d(loss)/d(logits)
  if ((rc = sgemm(st, C, D, B, b.logits, 1, C, b.y, D, 1, d_fc_weight, D, 1.f, 0.f))) return rc;  // dZ^T y
  if ((rc = sgemm(st, B, D, C, b.logits, C, 1, fc_weight, D, 1, b.dy, D, 1.f, 0.f))) return rc;   // dZ W
  bn_backward_kernel<<<(D + 255) / 256, 256, 0, st>>>(b.dy, b.xhat, B, D, nullptr, bn_weight, b.inv_std, 1, d_bn_weight,
                                                    b.dF_head);
  CTL_LAUNCH_CHECK();
  // ---- scalars + feature gradient ---------------------------------------------------------------------------
  base_scalars_kernel<<<1, 32, 0, st>>>(B, C, b.mine, b.center_rows, b.xent_rows, c.center_weight, c.xent_weight,
                                        b.labels_safe + B, out_losses);
  CTL_LAUNCH_CHECK();
  base_combine_kernel<<<B, 256, 0, st>>>(feats, B, D, cosine, b.dEm, b.rowsum, b.dF_head, labels, centers, b.row_sat,
                                         c.center_weight, d_feats);
  CTL_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"

