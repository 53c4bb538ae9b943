// Training-side kernels of the trunk (reference: autograd through modelling/backbones/resnet.py:67-87,122-133
// in train mode -- torch.nn.Conv2d weight gradients, BatchNorm2d batch statistics and their backward).
//
// 1. conv2d weight gradient as a wgmma GEMM over the pixel dimension:
//      dW[co][tap][ci] = sum_pixels dy[pixel][co] * x[pixel + tap][ci]
//    Both operands are the SAME TMA boxes the forward uses ([128 pixels][64 channels], 128-byte rows,
//    SWIZZLE_128B) -- read by the tensor core as MN-major (transposed) operands:
//    rows are the K (pixel) dimension, the 64 channels of a row the M / N dimension.  The reduction is long
//    (N*Ho*Wo pixels) and the output small, so the pixel range is split across CTAs; fp32 partial tiles are
//    reduced in a fixed order by a second kernel (deterministic, no atomics).
#include <cuda_fp16.h>
#include <stdint.h>

#include <algorithm>

#include "common.h"
#include "wgmma.cuh"

namespace ctl {

struct ConvTapW {
  int map;  // which activation tensor map (stride-2 parity view)
  int dh, dw;
};

// producer warpgroup (one TMA thread) + two consumer warpgroups: warpgroup g owns output channels
// [64 g, 64 g + 64) of the 128-channel cout tile (= dy box g) and the whole N = cin-per-item width
static constexpr int WG_THREADS = 384;
static constexpr int WG_BOX_BYTES = 128 * 64 * 2;  // one [128 px][64 ch] box
static constexpr uint32_t WG_PRODUCER_REGS = 40, WG_CONSUMER_REGS = 232;
static constexpr int WG_CHAIN_TILES = 8;  // pixel tiles per wgmma accumulation chain: 64 k16 steps (see the consumer)
// N (cin per work item) = 64 or 128: the wider the item, the more MMA work one dy tile feeds (less TMA fill per
// flop), the shallower the ring that fits in shared memory
template <int BNW>
struct WgCfg {
  static constexpr int XBOXES = BNW / 64;
  static constexpr int STAGES = BNW == 128 ? 3 : 4;
  static constexpr int STAGE_BYTES = (2 + XBOXES) * WG_BOX_BYTES;  // dy: 2 boxes (128 cout) + x boxes
  static constexpr size_t SMEM = 1024 + STAGES * STAGE_BYTES + 256;
  static_assert(SMEM <= 227 * 1024, "conv_wgrad_kernel shared memory");
};

struct WgradParams {
  CUtensorMap x_map[4];
  CUtensorMap dy_map;
  ConvTapW taps[9];
  int n_taps, cin, cout;
  int TW, TH, tiles_w, tiles_h, m_tiles;
  int bnw;         // cin per work item: 64 or 128
  int cin_chunks;  // cin / bnw
  int cout_tiles;  // ceil(cout / 128)
  int n_items;     // cout_tiles * n_taps * cin_chunks
  int splits;      // pixel-range splits
  int cout_pad;    // cout_tiles * 128
  float* part;     // [splits][cout_pad][n_taps * cin]
};

template <int BNW>
__global__ void __launch_bounds__(WG_THREADS, 1) conv_wgrad_kernel(const __grid_constant__ WgradParams p) {
  constexpr int WG_STAGES = WgCfg<BNW>::STAGES, WG_STAGE_BYTES = WgCfg<BNW>::STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + WG_STAGES * WG_STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (WG_STAGES + s); };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < WG_STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
    tma_prefetch_desc(&p.dy_map);
    for (int i = 0; i < 4; ++i) tma_prefetch_desc(&p.x_map[i]);
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  const int n_units = p.n_items * p.splits;
  const int tiles_per_img = p.tiles_w * p.tiles_h;
  // unit -> (work item, pixel-tile range)
  auto unit_range = [&](int u, int& item, int& t0, int& t1) {
    item = u / p.splits;
    const int s = u - item * p.splits;
    t0 = (int)((long long)p.m_tiles * s / p.splits);
    t1 = (int)((long long)p.m_tiles * (s + 1) / p.splits);
  };
  auto item_coords = [&](int item, int& ct, int& tap, int& chunk) {
    ct = item / (p.n_taps * p.cin_chunks);
    const int r = item - ct * (p.n_taps * p.cin_chunks);
    tap = r / p.cin_chunks;
    chunk = r - tap * p.cin_chunks;
  };

  if (warp < 4) {
    setmaxnreg_dec<WG_PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
        int item, t0, t1, ct, tapi, chunk;
        unit_range(u, item, t0, t1);
        item_coords(item, ct, tapi, chunk);
        const ConvTapW tap = p.taps[tapi];
        int img = t0 / tiles_per_img;
        int tr = t0 - img * tiles_per_img;
        int th = tr / p.tiles_w, tw = tr - th * p.tiles_w;
        for (int t = t0; t < t1; ++t) {
          const int h0 = th * p.TH, w0 = tw * p.TW;
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t dst = smem_base + stage * WG_STAGE_BYTES;
          mbar_arrive_expect_tx(full_bar(stage), WG_STAGE_BYTES);
          tma_load_4d(dst, &p.dy_map, full_bar(stage), ct * 128, w0, h0, img);
          tma_load_4d(dst + WG_BOX_BYTES, &p.dy_map, full_bar(stage), ct * 128 + 64, w0, h0, img);  // OOB channels -> 0
          for (int j = 0; j < BNW / 64; ++j)
            tma_load_4d(dst + (2 + j) * WG_BOX_BYTES, &p.x_map[tap.map], full_bar(stage), chunk * BNW + 64 * j,
                        w0 + tap.dw, h0 + tap.dh, img);
          if (++stage == WG_STAGES) {
            stage = 0;
            phase ^= 1u;
          }
          if (++tw == p.tiles_w) {
            tw = 0;
            if (++th == p.tiles_h) {
              th = 0;
              ++img;
            }
          }
        }
      }
    }
  } else {
    // ===== consumers: D[64 cout][BNW cin] += dy^T x over the unit's pixels (both operands MN-major: rows of a box
    // are the K = pixel dimension), then the fp32 partial tile goes straight from the registers to `part` =====
    setmaxnreg_inc<WG_CONSUMER_REGS>();
    const int wg = (threadIdx.x >> 7) - 1;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const int row0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // cout inside the 128-channel tile
    const int ktot = p.n_taps * p.cin;
    // wgmma's fp32 accumulation does not round like IEEE addition: on same-sign terms its error grows with the chain
    // length C (about C * 2^-24 * sum |terms|, measured on an H100), not with sqrt(C).  So a unit runs as chains of
    // WG_CHAIN_TILES pixel tiles (8 k16 steps each), and each finished chain is added to `sum` with ordinary FADDs.
    float acc[BNW / 2], sum[BNW / 2];
    auto fold = [&](bool first) {  // sum (+)= acc once the chain's wgmma groups have completed
#pragma unroll
      for (int i = 0; i < BNW / 2; ++i) {
        asm volatile("" : "+f"(acc[i])::"memory");  // keep the reads after wgmma_wait
        sum[i] = first ? acc[i] : sum[i] + acc[i];
      }
    };
    int stage = 0;
    uint32_t phase = 0;
    for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
      int item, t0, t1, ct, tapi, chunk;
      unit_range(u, item, t0, t1);
      item_coords(item, ct, tapi, chunk);
      const int split = u - item * p.splits;
      int held = -1;
      for (int t = t0; t < t1; ++t) {
        const int c = (t - t0) % WG_CHAIN_TILES;  // tile index inside the current chain
        mbar_wait(full_bar(stage), phase);
        const uint32_t a0 = smem_base + stage * WG_STAGE_BYTES + wg * WG_BOX_BYTES, b0 = smem_base + stage * WG_STAGE_BYTES + 2 * WG_BOX_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 8; ++k) {  // 16 pixels (rows) per MMA
          const uint64_t da = make_sw128_mnmajor_desc(a0 + k * 2048, WG_BOX_BYTES);
          const uint64_t db = make_sw128_mnmajor_desc(b0 + k * 2048, WG_BOX_BYTES);
          wgmma_f16<BNW, 1, 1>(acc, da, db, (c > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (held >= 0 && wg_leader) mbar_arrive(empty_bar(held));
        held = stage;
        if (++stage == WG_STAGES) {
          stage = 0;
          phase ^= 1u;
        }
        if (c == WG_CHAIN_TILES - 1 && t + 1 < t1) {
          wgmma_wait<0>();
          fold(t - t0 < WG_CHAIN_TILES);
        }
      }
      wgmma_wait<0>();
      if (held >= 0 && wg_leader) mbar_arrive(empty_bar(held));
      fold(t1 - t0 <= WG_CHAIN_TILES);
      float* dst = p.part + ((size_t)split * p.cout_pad + ct * 128 + row0) * ktot + tapi * p.cin + chunk * BNW + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BNW / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          *reinterpret_cast<float2*>(dst + (size_t)(8 * h) * ktot + 8 * j) = make_float2(sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1]);
    }
  }
}

// dW[row][col] = sum over splits (fixed order) of the fp32 partial tiles; rows >= cout are padding
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float* __restrict__ part, int splits, int cout_pad,
                                                           int cout, int ktot, float* __restrict__ dw) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t n4 = (size_t)cout * ktot / 4;
  const size_t stride4 = (size_t)cout_pad * ktot / 4;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    float4 acc = reinterpret_cast<const float4*>(part)[i];
    for (int s = 1; s < splits; ++s) {
      const float4 v = reinterpret_cast<const float4*>(part)[i + s * stride4];
      acc.x += v.x;
      acc.y += v.y;
      acc.z += v.z;
      acc.w += v.w;
    }
    reinterpret_cast<float4*>(dw)[i] = acc;
  }
}

// same reduction, result multiplied by `scale` and written in the reference's parameter layout [Cout][Cin][k][k]
// (torch.nn.Conv2d.weight) instead of the operand layout [Cout][k][k][Cin].  Replaces a permute + mul pass per layer.
// A block owns 256 consecutive (cout, cin) pairs: reads are coalesced over cin for every tap, the k*k results of the
// block are transposed through shared memory and leave as ONE contiguous run of 256 * k*k floats.
template <int KK>
__global__ void __launch_bounds__(256) wgrad_reduce_nchw_kernel(const float* __restrict__ part, int splits, int cout_pad,
                                                                int cout, int cin, float scale, float* __restrict__ dw) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float tile[KK > 1 ? 256 * KK : 1];
  const size_t n = (size_t)cout * cin;
  const size_t split_stride = (size_t)cout_pad * KK * cin;
  for (size_t base = (size_t)blockIdx.x * 256; base < n; base += (size_t)gridDim.x * 256) {
    const size_t i = base + threadIdx.x;
    if (i < n) {
      const size_t co = i / cin, ci = i - co * cin;
#pragma unroll
      for (int rs = 0; rs < KK; ++rs) {
        const size_t src = (co * KK + rs) * cin + ci;
        float acc = part[src];
        for (int s = 1; s < splits; ++s) acc += part[src + s * split_stride];
        if (KK == 1) dw[i] = acc * scale;
        else tile[threadIdx.x * KK + rs] = acc * scale;
      }
    }
    if (KK > 1) {
      __syncthreads();
      const size_t cnt = min((size_t)256, n - base) * KK;
      for (size_t j = threadIdx.x; j < cnt; j += 256) dw[base * KK + j] = tile[j];
      __syncthreads();
    }
  }
}

// Operand packs of ALL convolutions of a training step in one launch (replaces permute / contiguous / half / flip chains
// per layer): src fp32 [Cout][Cin][k][k] (torch.nn.Conv2d.weight) ->
//   fwd  fp16 [Cout][k][k][Cin]            the forward operand of ctl_conv2d_nhwc_f16
//   dgr  fp16 [Cin][k][k][Cout], taps flipped: the operand of the data-gradient convolution (the transposed conv)
struct PackEntry {
  const float* src;
  __half* fwd;
  __half* dgr;
  int cout, cin, k, pad_;
  long long chunk_begin;
};

__global__ void __launch_bounds__(256) train_pack_kernel(const PackEntry* __restrict__ table, int n_tensors, long long n_chunks) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
    int lo = 0, hi = n_tensors - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (table[mid].chunk_begin <= chunk) lo = mid; else hi = mid - 1;
    }
    const PackEntry e = table[lo];
    const int kk = e.k * e.k;
    const long long numel = (long long)e.cout * e.cin * kk;
    const long long base = (chunk - e.chunk_begin) * CTL_PACK_CHUNK;
    const long long end = min(numel, base + CTL_PACK_CHUNK);
    for (long long i = base + threadIdx.x; i < end; i += blockDim.x) {
      const int rs = (int)(i % kk);
      const long long t = i / kk;
      const int ci = (int)(t % e.cin), co = (int)(t / e.cin);
      const __half v = __float2half_rn(e.src[i]);
      e.fwd[((long long)co * kk + rs) * e.cin + ci] = v;
      if (e.dgr) e.dgr[((long long)ci * kk + (kk - 1 - rs)) * e.cout + co] = v;
    }
  }
}

static int wgrad_plan(int n, int h, int w, int cin, int cout, int ksize, int stride, WgradParams* p) {
  const int pad = ksize == 3 ? 1 : 0;
  const int Ho = (h + 2 * pad - ksize) / stride + 1, Wo = (w + 2 * pad - ksize) / stride + 1;
  pick_tile(Ho, Wo, &p->TH, &p->TW);
  p->tiles_h = (Ho + p->TH - 1) / p->TH;
  p->tiles_w = (Wo + p->TW - 1) / p->TW;
  p->m_tiles = n * p->tiles_h * p->tiles_w;
  p->n_taps = ksize * ksize;
  p->cin = cin;
  p->cout = cout;
  p->bnw = cin % 128 == 0 ? 128 : 64;
  p->cin_chunks = cin / p->bnw;
  p->cout_tiles = (cout + 127) / 128;
  p->cout_pad = p->cout_tiles * 128;
  p->n_items = p->cout_tiles * p->n_taps * p->cin_chunks;
  const int want = (2 * sm_count() + p->n_items - 1) / p->n_items;
  p->splits = std::max(1, std::min(want, p->m_tiles));
  return Ho * 65536 + Wo;
}

// the bytes ctl_conv2d_wgrad_workspace_bytes reports and the launch requires: the partial tiles plus 256 bytes of slack
static size_t wgrad_workspace_need(const WgradParams& p) {
  return (size_t)p.splits * p.cout_pad * p.n_taps * p.cin * sizeof(float) + 256;
}


// =======================================================================================
// 2. BatchNorm2d with batch statistics over NHWC fp16 ([rows = N*H*W][C]) -- forward and backward.
//    A thread owns 8 consecutive channels (one 16-byte load per row); a block walks a contiguous slab of rows,
//    its threads tiled (channel group, row lane); per-block partial sums go to a workspace and are combined in a
//    fixed order in double precision (deterministic, no atomics).
// =======================================================================================
static constexpr int BN_THREADS = 256;
static constexpr int BN_MAX_BLOCKS = 528;  // 132 SMs x 4

struct BnGeom {
  int groups;         // C / 8
  int lanes;          // row lanes per block = BN_THREADS / groups (>= 1)
  int blocks;         // row slabs
  long long rows_per_block;
};

static BnGeom bn_geom(long long rows, int C) {
  BnGeom g;
  g.groups = C / 8;
  g.lanes = std::max(1, BN_THREADS / g.groups);
  const long long iters = (rows + g.lanes - 1) / g.lanes;
  // enough row slabs to fill the machine, but not so many that the finalize pass (blocks x C partials) dominates
  const long long cap = std::max<long long>(2 * sm_count(), std::min<long long>(BN_MAX_BLOCKS, 1048576 / C));
  g.blocks = (int)std::min<long long>(cap, std::max<long long>(1, iters / 4));
  g.rows_per_block = (rows + g.blocks - 1) / g.blocks;
  return g;
}

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __half22float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
// a 16-byte load by value: unpack8 of a dereferenced global pointer reads the four __half2 one by one
__device__ __forceinline__ uint4 ldg16(const __half* p) { return *reinterpret_cast<const uint4*>(p); }

__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 v;
  __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  return v;
}

// Block-level reduction of per-thread 8-channel partials over the row lanes -> part[block][which][C].
// blockDim.x = groups * lanes when groups <= 256; for C > 2048 a thread loops over several groups (gstride).
template <int NQ>
__device__ __forceinline__ void bn_block_store(float (&acc)[NQ][8], int group, int lane_row, int lanes, int C,
                                               float* __restrict__ part_block, float* sred) {
  // sred: [lanes][NQ][C] floats would be too big for large C; reduce lane by lane through registers of lane 0
  // using shared memory slabs of [NQ][C] (lanes is small when C is large and vice versa: lanes * C = 2048)
  for (int q = 0; q < NQ; ++q)
#pragma unroll
    for (int i = 0; i < 8; ++i) sred[((size_t)lane_row * NQ + q) * C + group * 8 + i] = acc[q][i];
  __syncthreads();
  if (lane_row == 0) {
    for (int q = 0; q < NQ; ++q)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float t = 0.f;
        for (int l = 0; l < lanes; ++l) t += sred[((size_t)l * NQ + q) * C + group * 8 + i];
        part_block[(size_t)q * C + group * 8 + i] = t;
      }
  }
}

// pass A of the forward: per-block sum and sum of squares of y - p, p = the channel's value in one row (`pivot`).
// Summing y and y^2 directly and forming E[y^2] - mean^2 cancels catastrophically when |mean| >> std (fp32 partials of
// y^2 lose the variance); shifted by a sample of the channel the sums stay of the order of the variance.  The fp32
// partial error is still amplified by 1 + (p - mean)^2 / var: about 1-10 for a sample of a bell-shaped channel, but a pivot
// row that is a far outlier of its channel brings the cancellation back (unlike the Welford InstanceNorm statistics
// below, which are robust; here they would need the (count, mean, M2) triples carried through bn_block_store and the
// double-precision finalize).
__global__ void __launch_bounds__(BN_THREADS) bn_stats_kernel(const __half* __restrict__ y, long long rows, int C, int pitch,
                                                              long long rows_per_block, int lanes,
                                                              const __half* __restrict__ pivot, float* __restrict__ part) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float sred[];
  const int groups = C / 8;
  const int group = threadIdx.x % groups, lane_row = threadIdx.x / groups;
  float acc[2][8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[0][i] = acc[1][i] = 0.f;
  if (lane_row < lanes) {
    float piv[8];
    unpack8(*reinterpret_cast<const uint4*>(pivot + group * 8), piv);
    const long long r0 = (long long)blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
    long long r = r0 + lane_row;
    for (; r + 3LL * lanes < r1; r += 4LL * lanes) {  // four independent 16-byte loads in flight per thread
      uint4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const uint4*>(y + (r + (long long)u * lanes) * pitch + group * 8);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float f[8];
        unpack8(v[u], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = f[i] - piv[i];
          acc[0][i] += d;
          acc[1][i] = fmaf(d, d, acc[1][i]);
        }
      }
    }
    for (; r < r1; r += lanes) {
      float f[8];
      unpack8(*reinterpret_cast<const uint4*>(y + r * pitch + group * 8), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d = f[i] - piv[i];
        acc[0][i] += d;
        acc[1][i] = fmaf(d, d, acc[1][i]);
      }
    }
  }
  if (lane_row < lanes) bn_block_store<2>(acc, group, lane_row, lanes, C, part + (size_t)blockIdx.x * 2 * C, sred);
}

// finalize of the forward: batch mean / biased variance -> invstd, scale = gamma*invstd, shift = beta - mean*scale;
// running statistics updated like torch (momentum, unbiased variance).
// Sum of the per-block partials of 32 channels: 32 warps split the block index (stride 32), partial sums are combined in
// a fixed order (deterministic).  Returns the two totals of channel `c` to the threads with part == 0.
__device__ __forceinline__ void bn_sum_partials(const float* __restrict__ part, int blocks, int C, int c, int part_id,
                                                double (*sh)[2][32], double& s0, double& s1) {  // sh[32][2][32]
  // the partials are loaded in groups of 4 INDEPENDENT loads (5 memory round trips instead of a chain of up to 19
  // dependent ones -- the finalize kernels are pure latency, 127 launches per training step) and summed in a fixed
  // order (deterministic).  Loading all 19 at once takes 64 registers x 1024 threads = the whole register file of an
  // SM, and the kernel then showed sporadic 20-80 ms stalls -- keep the footprint low.
  constexpr int MAXQ = (BN_MAX_BLOCKS + 31) / 32, GRP = 4;
  double a = 0.0, b = 0.0;
#pragma unroll 1
  for (int q0 = 0; q0 < MAXQ; q0 += GRP) {
    float va[GRP], vb[GRP];
#pragma unroll
    for (int j = 0; j < GRP; ++j) {
      const int blk = part_id + 32 * (q0 + j);
      const bool ok = c < C && blk < blocks;
      va[j] = ok ? part[(size_t)blk * 2 * C + c] : 0.f;
      vb[j] = ok ? part[(size_t)blk * 2 * C + C + c] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < GRP; ++j) {
      if (c < C && part_id + 32 * (q0 + j) < blocks) {
        a += (double)va[j];
        b += (double)vb[j];
      }
    }
  }
  sh[part_id][0][threadIdx.x & 31] = a;
  sh[part_id][1][threadIdx.x & 31] = b;
  __syncthreads();
  s0 = s1 = 0.0;
  if (part_id == 0)
    for (int q = 0; q < 32; ++q) {
      s0 += sh[q][0][threadIdx.x & 31];
      s1 += sh[q][1][threadIdx.x & 31];
    }
}

// finalize of the forward: batch mean / biased variance -> invstd, scale = gamma*invstd, shift = beta - mean*scale;
// running statistics updated like torch (momentum, unbiased variance).  The partials are sums of y - pivot
// (bn_stats_kernel); the pivot row is read here again.  grid = C / 32 blocks of 1024 threads.
__global__ void __launch_bounds__(1024) bn_finalize_kernel(const float* __restrict__ part, int blocks, int C, double count,
                                                          const __half* __restrict__ pivot,
                                                          const float* __restrict__ gamma, const float* __restrict__ beta,
                                                          float eps, float momentum, float* __restrict__ running_mean,
                                                          float* __restrict__ running_var, float* __restrict__ mean,
                                                          float* __restrict__ invstd, float* __restrict__ scale,
                                                          float* __restrict__ shift) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double sh[32][2][32];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31), part_id = threadIdx.x >> 5;
  double s, ss;
  bn_sum_partials(part, blocks, C, c, part_id, sh, s, ss);
  if (part_id != 0 || c >= C) return;
  const double d = s / count;  // mean - pivot
  const double m = (double)__half2float(pivot[c]) + d;
  double var = ss / count - d * d;
  if (var < 0.0) var = 0.0;
  const float is = (float)(1.0 / sqrt(var + (double)eps));
  mean[c] = (float)m;
  invstd[c] = is;
  const float sc = gamma[c] * is;
  scale[c] = sc;
  shift[c] = beta[c] - (float)m * sc;
  if (running_mean) {
    const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)m;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
  }
}

// z = [relu](y * scale + shift [+ residual]) -> fp16.  A thread keeps the coefficients of its 8 channels in registers
// and walks rows (blockDim = groups * lanes, like the statistics kernels).
__global__ void __launch_bounds__(BN_THREADS) bn_apply_kernel(const __half* __restrict__ y, long long rows, int C, int pitch, int lanes,
                                                              const float* __restrict__ scale, const float* __restrict__ shift,
                                                              const __half* __restrict__ residual, int relu,
                                                              __half* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int groups = C / 8;
  const int group = threadIdx.x % groups, lane_row = threadIdx.x / groups;
  float sc[8], sh[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    sc[k] = scale[group * 8 + k];
    sh[k] = shift[group * 8 + k];
  }
  const long long step = (long long)gridDim.x * lanes;
  for (long long r = (long long)blockIdx.x * lanes + lane_row; r < rows; r += 2 * step) {
    const bool two = r + step < rows;
    const size_t off0 = (size_t)r * pitch + group * 8, off1 = two ? off0 + (size_t)step * pitch : off0;
    const uint4 v0 = *reinterpret_cast<const uint4*>(y + off0);
    const uint4 v1 = *reinterpret_cast<const uint4*>(y + off1);
    uint4 r0 = make_uint4(0, 0, 0, 0), r1 = r0;
    if (residual) {
      r0 = *reinterpret_cast<const uint4*>(residual + off0);
      r1 = *reinterpret_cast<const uint4*>(residual + off1);
    }
    float f[8], g2[8], rr[8];
    unpack8(v0, f);
    unpack8(v1, g2);
    unpack8(r0, rr);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      f[k] = fmaf(f[k], sc[k], sh[k]) + rr[k];
      if (relu) f[k] = fmaxf(f[k], 0.f);
    }
    *reinterpret_cast<uint4*>(out + off0) = pack8(f);
    if (two) {
      unpack8(r1, rr);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        g2[k] = fmaf(g2[k], sc[k], sh[k]) + rr[k];
        if (relu) g2[k] = fmaxf(g2[k], 0.f);
      }
      *reinterpret_cast<uint4*>(out + off1) = pack8(g2);
    }
  }
}

// pass A of the backward: g = dz * (z > 0) (written to g_out when a ReLU mask is given), per-block sum g and
// sum g * xhat with xhat = (y - mean) * invstd
__global__ void __launch_bounds__(BN_THREADS) bn_bwd_reduce_kernel(const __half* __restrict__ dz, const __half* __restrict__ z,
                                                                   const __half* __restrict__ y, long long rows, int C, int pitch,
                                                                   long long rows_per_block, int lanes,
                                                                   const float* __restrict__ mean,
                                                                   const float* __restrict__ invstd,
                                                                   __half* __restrict__ g_out, float* __restrict__ part) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float sred[];
  const int groups = C / 8;
  const int group = threadIdx.x % groups, lane_row = threadIdx.x / groups;
  float acc[2][8], mu[8], is[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    acc[0][i] = acc[1][i] = 0.f;
    mu[i] = mean[group * 8 + i];
    is[i] = invstd[group * 8 + i];
  }
  if (lane_row < lanes) {
    const long long r0 = (long long)blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
    // (one row per iteration: a two-row version was measured in round 2 -- 78 registers, 3 instead of 4 blocks per SM,
    // 2.85 -> 3.04 ms per step; capped at 64 registers it spilled.  The kernel is latency-bound on its small layers.)
    for (long long r = r0 + lane_row; r < r1; r += lanes) {
      const size_t off = (size_t)r * pitch + group * 8;
      float g[8], yv[8];
      unpack8(*reinterpret_cast<const uint4*>(dz + off), g);
      unpack8(*reinterpret_cast<const uint4*>(y + off), yv);
      if (z) {
        float zv[8];
        unpack8(*reinterpret_cast<const uint4*>(z + off), zv);
#pragma unroll
        for (int i = 0; i < 8; ++i) g[i] = zv[i] > 0.f ? g[i] : 0.f;
        *reinterpret_cast<uint4*>(g_out + off) = pack8(g);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        acc[0][i] += g[i];
        acc[1][i] = fmaf(g[i], (yv[i] - mu[i]) * is[i], acc[1][i]);
      }
    }
    bn_block_store<2>(acc, group, lane_row, lanes, C, part + (size_t)blockIdx.x * 2 * C, sred);
  }
}

// finalize of the backward: dgamma, dbeta (multiplied by `grad_unscale`), and the per-channel coefficients of
// dy = A * g + B * y + Cc  (= gamma*invstd * (g - dbeta/M - xhat * dgamma/M))
__global__ void __launch_bounds__(1024) bn_bwd_finalize_kernel(const float* __restrict__ part, int blocks, int C, double count,
                                                              const float* __restrict__ gamma, const float* __restrict__ mean,
                                                              const float* __restrict__ invstd, float grad_unscale,
                                                              float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                              float* __restrict__ coef) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double sh[32][2][32];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31), part_id = threadIdx.x >> 5;
  double sg, sgx;
  bn_sum_partials(part, blocks, C, c, part_id, sh, sg, sgx);
  if (part_id != 0 || c >= C) return;
  dbeta[c] = (float)sg * grad_unscale;
  dgamma[c] = (float)sgx * grad_unscale;
  const double k1 = (double)gamma[c] * invstd[c];
  const double k2 = sg / count;
  const double k3 = sgx / count * invstd[c];
  coef[c] = (float)k1;
  coef[C + c] = (float)(-k1 * k3);
  coef[2 * C + c] = (float)(k1 * ((double)mean[c] * k3 - k2));
}

__global__ void __launch_bounds__(BN_THREADS) bn_bwd_apply_kernel(const __half* __restrict__ g, const __half* __restrict__ y,
                                                                  long long rows, int C, int pitch, int lanes,
                                                                  const float* __restrict__ coef, __half* __restrict__ dy) {
  pdl_launch_dependents();
  pdl_wait();
  const int groups = C / 8;
  const int group = threadIdx.x % groups, lane_row = threadIdx.x / groups;
  float ca[8], cb[8], cc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    ca[k] = coef[group * 8 + k];
    cb[k] = coef[C + group * 8 + k];
    cc[k] = coef[2 * C + group * 8 + k];
  }
  const long long step = (long long)gridDim.x * lanes;
  for (long long r = (long long)blockIdx.x * lanes + lane_row; r < rows; r += 2 * step) {
    const bool two = r + step < rows;
    const size_t off0 = (size_t)r * pitch + group * 8, off1 = two ? off0 + (size_t)step * pitch : off0;
    const uint4 a0 = *reinterpret_cast<const uint4*>(g + off0), b0 = *reinterpret_cast<const uint4*>(y + off0);
    const uint4 a1 = *reinterpret_cast<const uint4*>(g + off1), b1 = *reinterpret_cast<const uint4*>(y + off1);
    float gv[8], yv[8], o[8];
    unpack8(a0, gv);
    unpack8(b0, yv);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = fmaf(ca[k], gv[k], fmaf(cb[k], yv[k], cc[k]));
    *reinterpret_cast<uint4*>(dy + off0) = pack8(o);
    if (two) {
      unpack8(a1, gv);
      unpack8(b1, yv);
#pragma unroll
      for (int k = 0; k < 8; ++k) o[k] = fmaf(ca[k], gv[k], fmaf(cb[k], yv[k], cc[k]));
      *reinterpret_cast<uint4*>(dy + off1) = pack8(o);
    }
  }
}

// =======================================================================================
// 2b. InstanceNorm2d(affine) + ReLU on the first `half` channels of an IBN layer (resnet_ibn_a.py:18-32), train mode:
//     statistics per (image, channel) over the H*W positions -- always instance statistics, no running buffers.
//     One block per (image, 8-channel group); the block reduction order is fixed (deterministic).
// =======================================================================================
__device__ __forceinline__ void in_block_reduce(float (&acc)[2][8], float* sred /* [256][16] */, float (&tot)[2][8]) {
#pragma unroll
  for (int q = 0; q < 2; ++q)
#pragma unroll
    for (int i = 0; i < 8; ++i) sred[threadIdx.x * 16 + q * 8 + i] = acc[q][i];
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if ((int)threadIdx.x < off)
#pragma unroll
      for (int j = 0; j < 16; ++j) sred[threadIdx.x * 16 + j] += sred[(threadIdx.x + off) * 16 + j];
    __syncthreads();
  }
#pragma unroll
  for (int q = 0; q < 2; ++q)
#pragma unroll
    for (int i = 0; i < 8; ++i) tot[q][i] = sred[q * 8 + i];
  __syncthreads();
}

// Chan's pairwise update: (na, ma, m2a) becomes the count, mean and M2 of both parts
__device__ __forceinline__ void in_chan_merge(float& na, float nb, float (&ma)[8], float (&m2a)[8], const float (&mb)[8],
                                              const float (&m2b)[8]) {
  const float nab = na + nb, wb = nb * __frcp_rn(nab);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float d = mb[i] - ma[i];
    ma[i] = fmaf(d, wb, ma[i]);
    m2a[i] += m2b[i] + d * d * na * wb;
  }
  na = nab;
}

// Block reduction of per-thread (count, mean, M2 = sum of squared deviations) of 8 channels by Chan's pairwise update,
// in a fixed tree order (deterministic): thread t takes in t + off for off = 128, 64, .., 1, the three cross-warp levels
// through shared memory (value-major, so a warp's accesses hit 32 banks) and the five in-warp levels in warp 0 through
// shuffles.  Returns the block's mean and M2 to every thread.
__device__ __forceinline__ void in_block_welford(float cnt, float (&mean)[8], float (&m2)[8], float* sred /* [16][256] */,
                                                 float* scnt /* [256] */) {
  const int t = threadIdx.x;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sred[i * 256 + t] = mean[i];
    sred[(8 + i) * 256 + t] = m2[i];
  }
  scnt[t] = cnt;
  __syncthreads();
  for (int off = 128; off >= 32; off >>= 1) {
    if (t < off && scnt[t + off] > 0.f) {
      float mb[8], m2b[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        mean[i] = sred[i * 256 + t];
        m2[i] = sred[(8 + i) * 256 + t];
        mb[i] = sred[i * 256 + t + off];
        m2b[i] = sred[(8 + i) * 256 + t + off];
      }
      float na = scnt[t];
      in_chan_merge(na, scnt[t + off], mean, m2, mb, m2b);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        sred[i * 256 + t] = mean[i];
        sred[(8 + i) * 256 + t] = m2[i];
      }
      scnt[t] = na;
    }
    __syncthreads();
  }
  if (t < 32) {
    float na = scnt[t];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      mean[i] = sred[i * 256 + t];
      m2[i] = sred[(8 + i) * 256 + t];
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float nb = __shfl_down_sync(0xffffffffu, na, off);
      float mb[8], m2b[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        mb[i] = __shfl_down_sync(0xffffffffu, mean[i], off);
        m2b[i] = __shfl_down_sync(0xffffffffu, m2[i], off);
      }
      if (t < off && nb > 0.f) in_chan_merge(na, nb, mean, m2, mb, m2b);
    }
    if (t == 0)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        sred[i] = mean[i];
        sred[8 + i] = m2[i];
      }
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    mean[i] = sred[i];
    m2[i] = sred[8 + i];
  }
  __syncthreads();
}

// statistics in ONE pass over the instance with Welford's update per thread and Chan's combination across threads (the
// update PyTorch's own normalisation kernels use), not E[y^2] - mean^2, which cancels catastrophically in fp32 when
// |mean| >> std.  The eval trunk runs it in place (out == y, each thread rewrites only the rows it read) without saving
// the statistics (save_mean == save_invstd == nullptr).
__global__ void __launch_bounds__(256) in_train_forward_kernel(const __half* y, int HW, int pitch, int half,
                                                               const float* __restrict__ gamma, const float* __restrict__ beta,
                                                               float eps, float* __restrict__ save_mean,
                                                               float* __restrict__ save_invstd, __half* out) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sred[256 * 16];
  __shared__ float scnt[256];
  const int g = blockIdx.x, n = blockIdx.y;
  const size_t base = (size_t)n * HW * pitch + g * 8;
  float cnt = 0.f, m[8], m2[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) m[i] = m2[i] = 0.f;
  for (int r = threadIdx.x; r < HW; r += blockDim.x) {
    float f[8];
    unpack8(ldg16(y + base + (size_t)r * pitch), f);
    cnt += 1.f;
    const float inv = __frcp_rn(cnt);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float d = f[i] - m[i];
      m[i] = fmaf(d, inv, m[i]);
      m2[i] = fmaf(d, f[i] - m[i], m2[i]);
    }
  }
  in_block_welford(cnt, m, m2, sred, scnt);
  float sc[8], sh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float var = m2[i] / HW;
    const float is = rsqrtf(var + eps);
    sc[i] = gamma[g * 8 + i] * is;
    sh[i] = beta[g * 8 + i] - m[i] * sc[i];
    if (threadIdx.x == 0 && save_mean) {
      save_mean[(size_t)n * half + g * 8 + i] = m[i];
      save_invstd[(size_t)n * half + g * 8 + i] = is;
    }
  }
  for (int r = threadIdx.x; r < HW; r += blockDim.x) {
    float f[8];
    unpack8(ldg16(y + base + (size_t)r * pitch), f);
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = fmaxf(fmaf(f[i], sc[i], sh[i]), 0.f);
    *reinterpret_cast<uint4*>(out + base + (size_t)r * pitch) = pack8(f);
  }
}

// g = dz * (z > 0) (written back over dz), per-instance sums -> dy; per-(image, channel) dgamma / dbeta partials
__global__ void __launch_bounds__(256) in_train_backward_kernel(__half* __restrict__ dz, const __half* __restrict__ z,
                                                                const __half* __restrict__ y, int HW, int pitch, int half,
                                                                const float* __restrict__ gamma,
                                                                const float* __restrict__ save_mean,
                                                                const float* __restrict__ save_invstd, float grad_unscale,
                                                                float* __restrict__ dgamma_part, float* __restrict__ dbeta_part,
                                                                __half* __restrict__ dy) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sred[256 * 16];
  const int g = blockIdx.x, n = blockIdx.y;
  const size_t base = (size_t)n * HW * pitch + g * 8;
  float mu[8], is[8], acc[2][8], tot[2][8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    acc[0][i] = acc[1][i] = 0.f;
    mu[i] = save_mean[(size_t)n * half + g * 8 + i];
    is[i] = save_invstd[(size_t)n * half + g * 8 + i];
  }
  for (int r = threadIdx.x; r < HW; r += blockDim.x) {
    const size_t off = base + (size_t)r * pitch;
    float gv[8], zv[8], yv[8];
    unpack8(*reinterpret_cast<const uint4*>(dz + off), gv);
    unpack8(*reinterpret_cast<const uint4*>(z + off), zv);
    unpack8(*reinterpret_cast<const uint4*>(y + off), yv);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      gv[i] = zv[i] > 0.f ? gv[i] : 0.f;
      acc[0][i] += gv[i];
      acc[1][i] = fmaf(gv[i], (yv[i] - mu[i]) * is[i], acc[1][i]);
    }
    *reinterpret_cast<uint4*>(dz + off) = pack8(gv);
  }
  in_block_reduce(acc, sred, tot);
  float ca[8], cb[8], cc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float k1 = gamma[g * 8 + i] * is[i];
    const float k2 = tot[0][i] / HW;
    const float k3 = tot[1][i] / HW * is[i];
    ca[i] = k1;
    cb[i] = -k1 * k3;
    cc[i] = k1 * (mu[i] * k3 - k2);
    if (threadIdx.x == 0) {
      dbeta_part[(size_t)n * half + g * 8 + i] = tot[0][i] * grad_unscale;
      dgamma_part[(size_t)n * half + g * 8 + i] = tot[1][i] * grad_unscale;
    }
  }
  for (int r = threadIdx.x; r < HW; r += blockDim.x) {
    const size_t off = base + (size_t)r * pitch;
    float gv[8], yv[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(dz + off), gv);  // this thread's own writes of the first loop
    unpack8(*reinterpret_cast<const uint4*>(y + off), yv);
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = fmaf(ca[i], gv[i], fmaf(cb[i], yv[i], cc[i]));
    *reinterpret_cast<uint4*>(dy + off) = pack8(o);
  }
}

// =======================================================================================
// 3. small backward helpers: global-average-pool, max-pool 3x3/2, zero-insertion upsampling (stride-2 dgrad)
// =======================================================================================
__global__ void __launch_bounds__(256) gap_backward_kernel(const float* __restrict__ dfeat, int N, int HW, int C, float scale,
                                                           __half* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int groups = C / 8;
  const long long total = (long long)N * HW * groups;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    const int n = (int)(i / ((long long)HW * groups));
    float f[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = dfeat[(size_t)n * C + g * 8 + k] * scale;
    *reinterpret_cast<uint4*>(out + i * 8) = pack8(f);
  }
}

// dx[p] = sum over the (<= 4) windows that contain p of dy[window] * [p is the window's first maximum in scan order]
// (torch max_pool2d keeps the first maximum: the forward updates only on `val > max`)
__global__ void __launch_bounds__(256) maxpool_backward_kernel(const __half* __restrict__ x, const __half* __restrict__ dy,
                                                               int N, int H, int W, int C, int Ho, int Wo,
                                                               __half* __restrict__ dx) {
  pdl_launch_dependents();
  pdl_wait();
  const int groups = C / 8;
  const long long total = (long long)N * H * W * groups;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    long long t = i / groups;
    const int pw = (int)(t % W);
    t /= W;
    const int ph = (int)(t % H);
    const int n = (int)(t / H);
    const __half* xn = x + (size_t)n * H * W * C + g * 8;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int oy = (ph + 1) / 2 - ((ph & 1) ? 1 : 0); oy <= (ph + 1) / 2; ++oy) {
      if (oy < 0 || oy >= Ho || 2 * oy - 1 > ph || 2 * oy + 1 < ph) continue;
      for (int ox = (pw + 1) / 2 - ((pw & 1) ? 1 : 0); ox <= (pw + 1) / 2; ++ox) {
        if (ox < 0 || ox >= Wo || 2 * ox - 1 > pw || 2 * ox + 1 < pw) continue;
        // first maximum of window (oy, ox), per channel
        float best[8];
        int arg[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          best[k] = -INFINITY;
          arg[k] = -1;
        }
        for (int r = 0; r < 3; ++r) {
          const int yy = 2 * oy - 1 + r;
          if (yy < 0 || yy >= H) continue;
          for (int s = 0; s < 3; ++s) {
            const int xx = 2 * ox - 1 + s;
            if (xx < 0 || xx >= W) continue;
            float v[8];
            unpack8(*reinterpret_cast<const uint4*>(xn + ((size_t)yy * W + xx) * C), v);
#pragma unroll
            for (int k = 0; k < 8; ++k)
              if (v[k] > best[k] || arg[k] < 0) {
                best[k] = v[k];
                arg[k] = yy * W + xx;
              }
          }
        }
        float d[8];
        unpack8(*reinterpret_cast<const uint4*>(dy + (((size_t)n * Ho + oy) * Wo + ox) * C + g * 8), d);
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (arg[k] == ph * W + pw) acc[k] += d[k];
      }
    }
    *reinterpret_cast<uint4*>(dx + i * 8) = pack8(acc);
  }
}

// Training forward of the pool: also records, per output element, which of the 9 window taps (r*3 + s) held the
// first maximum (one byte per channel) so that the backward is a 4-window gather instead of 36 loads per pixel.
__global__ void __launch_bounds__(256) maxpool_arg_kernel(const __half* __restrict__ x, int N, int H, int W, int C, int Ho,
                                                          int Wo, __half* __restrict__ out, uint2* __restrict__ arg) {
  pdl_launch_dependents();
  pdl_wait();
  const int groups = C / 8;
  const long long total = (long long)N * Ho * Wo * groups;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    long long t = i / groups;
    const int ox = (int)(t % Wo);
    t /= Wo;
    const int oy = (int)(t % Ho);
    const int n = (int)(t / Ho);
    float best[8];
    unsigned a[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      best[k] = -INFINITY;
      a[k] = 255u;
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int yy = 2 * oy - 1 + r;
      if (yy < 0 || yy >= H) continue;
#pragma unroll
      for (int s2 = 0; s2 < 3; ++s2) {
        const int xx = 2 * ox - 1 + s2;
        if (xx < 0 || xx >= W) continue;
        float v[8];
        unpack8(*reinterpret_cast<const uint4*>(x + (((size_t)n * H + yy) * W + xx) * C + g * 8), v);
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (v[k] > best[k] || a[k] == 255u) {
            best[k] = v[k];
            a[k] = r * 3 + s2;
          }
      }
    }
    *reinterpret_cast<uint4*>(out + i * 8) = pack8(best);
    arg[i] = make_uint2(a[0] | (a[1] << 8) | (a[2] << 16) | (a[3] << 24), a[4] | (a[5] << 8) | (a[6] << 16) | (a[7] << 24));
  }
}

__global__ void __launch_bounds__(256) maxpool_backward_arg_kernel(const uint2* __restrict__ arg, const __half* __restrict__ dy,
                                                                   int N, int H, int W, int C, int Ho, int Wo,
                                                                   __half* __restrict__ dx) {
  pdl_launch_dependents();
  pdl_wait();
  const int groups = C / 8;
  const long long total = (long long)N * H * W * groups;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    long long t = i / groups;
    const int pw = (int)(t % W);
    t /= W;
    const int ph = (int)(t % H);
    const int n = (int)(t / H);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    const int oy0 = ph / 2, ox0 = pw / 2;  // windows (oy0 [, oy0 + 1 when ph is odd]) x (ox0 [, ox0 + 1])
#pragma unroll
    for (int dyi = 0; dyi < 2; ++dyi) {
      const int oy = oy0 + dyi;
      if ((dyi == 1 && !(ph & 1)) || oy >= Ho) continue;
      const int r = ph - (2 * oy - 1);
#pragma unroll
      for (int dxi = 0; dxi < 2; ++dxi) {
        const int ox = ox0 + dxi;
        if ((dxi == 1 && !(pw & 1)) || ox >= Wo) continue;
        const unsigned tap = (unsigned)(r * 3 + pw - (2 * ox - 1));
        const size_t o = (((size_t)n * Ho + oy) * Wo + ox) * groups + g;
        const uint2 a = arg[o];
        float d[8];
        unpack8(*reinterpret_cast<const uint4*>(dy + o * 8), d);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const unsigned ak = ((k < 4 ? a.x : a.y) >> (8 * (k & 3))) & 255u;
          if (ak == tap) acc[k] += d[k];
        }
      }
    }
    *reinterpret_cast<uint4*>(dx + i * 8) = pack8(acc);
  }
}

// out[n][2i][2j] = x[n][i][j] (+ add), every other position = add (or 0): the transposed view of a stride-2 subsampling
__global__ void __launch_bounds__(256) upsample2_zero_kernel(const __half* __restrict__ x, int N, int H, int W, int C,
                                                             const __half* __restrict__ add, __half* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int groups = C / 8;
  const int H2 = 2 * H, W2 = 2 * W;
  const long long total = (long long)N * H2 * W2 * groups;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    long long t = i / groups;
    const int xx = (int)(t % W2);
    t /= W2;
    const int yy = (int)(t % H2);
    const int n = (int)(t / H2);
    float f[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = 0.f;
    if (((xx | yy) & 1) == 0)
      unpack8(*reinterpret_cast<const uint4*>(x + (((size_t)n * H + yy / 2) * W + xx / 2) * C + g * 8), f);
    if (add) {
      float a[8];
      unpack8(*reinterpret_cast<const uint4*>(add + i * 8), a);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] += a[k];
    }
    *reinterpret_cast<uint4*>(out + i * 8) = pack8(f);
  }
}

// im2col of the stem for its weight gradient: out[pixel][k], k = (c*7 + r)*8 + s (s = 7 and k >= 168 zero): the K
// ordering of ctl_stem_conv7x7_tc's weight operand, fp16.
// One block per (image, output row): the 7 x 3 input rows that feed this output row are staged ONCE in shared memory
// (coalesced loads, zero outside the image, 3 zero columns of left border), then every thread assembles 16-byte chunks
// from 7 consecutive shared-memory words.  Round 1 read the 7 taps of every chunk straight from global memory (42
// scattered 4-byte loads per thread: 0.84 ms at bs 256, an LSU-bound kernel that only writes 805 MB).
static constexpr int IM2COL_MAXW = 512;  // widest input row staged: 21 x 521 floats stay under the 48 KB default

__global__ void __launch_bounds__(256) stem_im2col_kernel(const float* __restrict__ x, int N, int H, int W, int Ho, int Wo,
                                                          __half* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float srow[];  // [21][pitch], pitch = (W + 8) | 1: srow[cr][3 + xx] = x[c][2 oy - 3 + r][xx]
  const int pitch = (W + 8) | 1;  // odd pitch: the 24 chunks of one pixel hit distinct banks
  const int n = blockIdx.x / Ho, oy = blockIdx.x - n * Ho;
  for (int i = threadIdx.x; i < 21 * pitch; i += blockDim.x) {
    const int cr = i / pitch, col = i - cr * pitch;
    const int c = cr / 7, r = cr - c * 7;
    const int yy = 2 * oy - 3 + r, xx = col - 3;
    float v = 0.f;
    if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = x[(((size_t)n * 3 + c) * H + yy) * W + xx];
    srow[i] = v;
  }
  __syncthreads();
  __half* orow = out + ((size_t)n * Ho + oy) * Wo * 192;
  for (int i = threadIdx.x; i < Wo * 24; i += blockDim.x) {
    const int ox = i / 24, chunk = i - ox * 24;
    float f[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = 0.f;
    if (chunk < 21) {
      const float* src = srow + chunk * pitch + 2 * ox;  // column 2 ox - 3 + s  ->  index 3 + 2 ox - 3 + s
#pragma unroll
      for (int sft = 0; sft < 7; ++sft) f[sft] = src[sft];
    }
    *reinterpret_cast<uint4*>(orow + (size_t)i * 8) = pack8(f);
  }
}

static int row_grid(long long rows, int lanes) {
  return (int)std::min<long long>((rows + 2 * lanes - 1) / (2 * lanes), (long long)sm_count() * 8);
}
static int ew_grid(long long total) {
  return (int)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
}

}  // namespace ctl

using namespace ctl;

extern "C" {

size_t ctl_conv2d_wgrad_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t ksize,
                                        int32_t stride) {
  if (n < 1 || h < 1 || w < 1 || cin % 64 != 0 || cout % 64 != 0 || (ksize != 1 && ksize != 3) ||
      (stride != 1 && stride != 2) || (stride == 2 && (h % 2 != 0 || w % 2 != 0)))
    return 0;
  WgradParams p = {};
  wgrad_plan(n, h, w, cin, cout, ksize, stride, &p);
  return wgrad_workspace_need(p);
}

int ctl_conv2d_wgrad_nhwc_f16(const void* x, int32_t n, int32_t h, int32_t w, int32_t cin, const void* dy, int32_t cout,
                              int32_t ksize, int32_t stride, void* workspace, size_t workspace_bytes, float* dw,
                              ctl_stream_t stream) {
  return ctl_conv2d_wgrad_nhwc_f16_ex(x, n, h, w, cin, dy, cout, ksize, stride, workspace, workspace_bytes, dw, 1.f, 0, stream);
}

int ctl_train_pack_weights(const void* table_device, int32_t n_tensors, int64_t n_chunks, ctl_stream_t stream) {
  CTL_CHECK_ARG(table_device && n_tensors >= 1 && n_chunks >= 1, "bad arguments");
  static_assert(sizeof(PackEntry) == 48, "ctl_pack_entry layout");
  int rc = ctl_device_check();
  if (rc) return rc;
  const int grid = (int)std::min<long long>(n_chunks, (long long)sm_count() * 8);
  CTL_CUDA(launch_k(train_pack_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, static_cast<const PackEntry*>(table_device),
                    (int)n_tensors, (long long)n_chunks));
  return 0;
}

int ctl_conv2d_wgrad_nhwc_f16_ex(const void* x, int32_t n, int32_t h, int32_t w, int32_t cin, const void* dy, int32_t cout,
                                 int32_t ksize, int32_t stride, void* workspace, size_t workspace_bytes, float* dw,
                                 float out_scale, int32_t param_layout, ctl_stream_t stream) {
  CTL_CHECK_ARG(x && dy && dw && workspace, "null pointer");
  CTL_CHECK_ARG(n >= 1 && h >= 1 && w >= 1, "bad activation shape");
  CTL_CHECK_ARG(cin % 64 == 0 && cout % 64 == 0, "Cin=%d and Cout=%d must be multiples of 64", cin, cout);
  CTL_CHECK_ARG((ksize == 1 || ksize == 3) && (stride == 1 || stride == 2), "only 1x1 / 3x3, stride 1 / 2");
  CTL_CHECK_ARG(stride == 1 || (h % 2 == 0 && w % 2 == 0), "stride 2 needs even H, W (got %dx%d)", h, w);
  int rc = ctl_device_check();
  if (rc) return rc;
  WgradParams p = {};
  const int hw = wgrad_plan(n, h, w, cin, cout, ksize, stride, &p);
  const int Ho = hw >> 16, Wo = hw & 65535;
  const size_t need = wgrad_workspace_need(p);
  CTL_CHECK_ARG(workspace_bytes >= need, "workspace too small: %zu < %zu", workspace_bytes, need);
  CTL_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 15u) == 0 && (reinterpret_cast<uintptr_t>(dw) & 15u) == 0,
                "workspace and dw must be 16-byte aligned");
  p.part = static_cast<float*>(workspace);
  const int pad = ksize == 3 ? 1 : 0;
  const __half* xb = static_cast<const __half*>(x);
  const uint32_t abox[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, 1};
  if (stride == 1) {
    const uint64_t dims[4] = {(uint64_t)cin, (uint64_t)w, (uint64_t)h, (uint64_t)n};
    const uint64_t strd[4] = {2, (uint64_t)cin * 2, (uint64_t)w * cin * 2, (uint64_t)h * w * cin * 2};
    for (int i = 0; i < 4; ++i)
      if ((rc = encode_tensor_map(&p.x_map[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, xb, dims, strd, abox,
                                  CU_TENSOR_MAP_SWIZZLE_128B)))
        return rc;
    for (int r = 0; r < ksize; ++r)
      for (int s = 0; s < ksize; ++s) p.taps[r * ksize + s] = ConvTapW{0, r - pad, s - pad};
  } else {
    // parity views (as the forward): view (ph, pw) holds input pixels (2i + ph, 2j + pw)
    const uint64_t dims[4] = {(uint64_t)cin, (uint64_t)(w / 2), (uint64_t)(h / 2), (uint64_t)n};
    const uint64_t strd[4] = {2, (uint64_t)cin * 4, (uint64_t)w * cin * 4, (uint64_t)h * w * cin * 2};
    for (int ph = 0; ph < 2; ++ph)
      for (int pw = 0; pw < 2; ++pw)
        if ((rc = encode_tensor_map(&p.x_map[ph * 2 + pw], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4,
                                    xb + ((size_t)ph * w + pw) * cin, dims, strd, abox, CU_TENSOR_MAP_SWIZZLE_128B)))
          return rc;
    for (int r = 0; r < ksize; ++r)
      for (int s = 0; s < ksize; ++s) {
        const int ar = r - pad, as = s - pad;
        const int ph = ((ar % 2) + 2) % 2, pw = ((as % 2) + 2) % 2;
        p.taps[r * ksize + s] = ConvTapW{ph * 2 + pw, (ar - ph) / 2, (as - pw) / 2};
      }
  }
  {
    const uint64_t odims[4] = {(uint64_t)cout, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)n};
    const uint64_t ostr[4] = {2, (uint64_t)cout * 2, (uint64_t)Wo * cout * 2, (uint64_t)Ho * Wo * cout * 2};
    if ((rc = encode_tensor_map(&p.dy_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, dy, odims, ostr, abox,
                                CU_TENSOR_MAP_SWIZZLE_128B)))
      return rc;
  }
  static bool attr_set = false;
  if (!attr_set) {
    CTL_CUDA(cudaFuncSetAttribute(conv_wgrad_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WgCfg<64>::SMEM));
    CTL_CUDA(cudaFuncSetAttribute(conv_wgrad_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WgCfg<128>::SMEM));
    attr_set = true;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = std::min(p.n_items * p.splits, sm_count());
  if (p.bnw == 128)
    CTL_CUDA(launch_k(conv_wgrad_kernel<128>, dim3(grid), dim3(WG_THREADS), WgCfg<128>::SMEM, st, p));
  else
    CTL_CUDA(launch_k(conv_wgrad_kernel<64>, dim3(grid), dim3(WG_THREADS), WgCfg<64>::SMEM, st, p));
  if (param_layout != 0 || out_scale != 1.f) {
    const size_t np = (size_t)cout * cin;
    const int rgrid = (int)std::min<size_t>((np + 255) / 256, (size_t)sm_count() * 8);
    if (param_layout != 0 && p.n_taps == 9) {
      CTL_CUDA(launch_k(wgrad_reduce_nchw_kernel<9>, dim3(rgrid), dim3(256), 0, st, (const float*)p.part, p.splits, p.cout_pad,
                        (int)cout, (int)cin, out_scale, dw));
    } else {  // 1x1, or operand layout scaled: [Cout][k*k*Cin] is the parameter layout of a 1x1 with Cin' = k*k*Cin
      const size_t np1 = (size_t)cout * p.n_taps * cin;
      const int g1 = (int)std::min<size_t>((np1 + 255) / 256, (size_t)sm_count() * 8);
      CTL_CUDA(launch_k(wgrad_reduce_nchw_kernel<1>, dim3(g1), dim3(256), 0, st, (const float*)p.part, p.splits, p.cout_pad,
                        (int)cout, p.n_taps * (int)cin, out_scale, dw));
    }
    return 0;
  }
  const size_t n4 = (size_t)cout * p.n_taps * cin / 4;
  const int rgrid = (int)std::min<size_t>((n4 + 255) / 256, (size_t)sm_count() * 8);
  CTL_CUDA(launch_k(wgrad_reduce_kernel, dim3(rgrid), dim3(256), 0, st, (const float*)p.part, p.splits, p.cout_pad, (int)cout,
                    p.n_taps * (int)cin, dw));
  return 0;
}


size_t ctl_bn_workspace_bytes(int64_t rows, int32_t c) {
  if (rows < 1 || c < 32 || c > 2048 || (c & (c - 1)) != 0) return 0;
  const BnGeom g = bn_geom(rows, c);
  return ((size_t)g.blocks * 2 * c + 4 * (size_t)c) * sizeof(float) + 256;
}

static int bn_check(const char* what, int64_t rows, int32_t c, const void* ws, size_t ws_bytes) {
  CTL_CHECK_ARG(rows >= 1 && c >= 32 && c <= 2048 && (c & (c - 1)) == 0, "%s: C=%d must be a power of two in [32, 2048]", what, c);
  CTL_CHECK_ARG(ws && ws_bytes >= ctl_bn_workspace_bytes(rows, c) - 256, "%s: workspace too small", what);
  CTL_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15u) == 0, "%s: workspace must be 16-byte aligned", what);
  return ctl_device_check();
}

int ctl_bn_train_forward_nhwc_f16(const void* y, int64_t rows, int32_t c, int32_t pitch, const float* gamma, const float* beta, float eps,
                                  float momentum, float* running_mean, float* running_var, const void* residual,
                                  int32_t relu, void* workspace, size_t workspace_bytes, float* save_mean,
                                  float* save_invstd, void* out, ctl_stream_t stream) {
  CTL_CHECK_ARG(y && gamma && beta && save_mean && save_invstd && out, "null pointer");
  CTL_CHECK_ARG((running_mean == nullptr) == (running_var == nullptr), "running_mean / running_var: both or neither");
  CTL_CHECK_ARG(pitch >= c && pitch % 8 == 0, "pitch=%d must be a multiple of 8 and >= C=%d", pitch, c);
  CTL_CHECK_ARG((reinterpret_cast<uintptr_t>(y) & 15u) == 0 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0 &&
                    (reinterpret_cast<uintptr_t>(residual) & 15u) == 0,
                "tensors (channel-slice base pointers) must be 16-byte aligned");
  int rc = bn_check("bn forward", rows, c, workspace, workspace_bytes);
  if (rc) return rc;
  const BnGeom g = bn_geom(rows, c);
  float* part = static_cast<float*>(workspace);
  float* scale = part + (size_t)g.blocks * 2 * c;
  float* shift = scale + c;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t sm = (size_t)g.lanes * 2 * c * sizeof(float);
  // the pivot is the slice's last row.  Any row serves equally well numerically; the row changes the last bits of the
  // statistics and, through the ReLU masks, of every training gradient -- see the margin note on
  // tests/test_reference_autocast_gpu.py::test_training_step_at_bench_shape_vs_reference_cuda_autocast
  const __half* pivot = static_cast<const __half*>(y) + (size_t)(rows - 1) * pitch;
  CTL_CUDA(launch_k(bn_stats_kernel, dim3(g.blocks), dim3(BN_THREADS), sm, st, static_cast<const __half*>(y), (long long)rows,
                    (int)c, (int)pitch, g.rows_per_block, g.lanes, pivot, part));
  CTL_CUDA(launch_k(bn_finalize_kernel, dim3((c + 31) / 32), dim3(1024), 0, st, (const float*)part, g.blocks, (int)c,
                    (double)rows, pivot, gamma, beta, eps, momentum, running_mean, running_var, save_mean, save_invstd, scale, shift));
  CTL_CUDA(launch_k(bn_apply_kernel, dim3(row_grid(rows, g.lanes)), dim3(BN_THREADS), 0, st, static_cast<const __half*>(y),
                    (long long)rows, (int)c, (int)pitch, g.lanes, (const float*)scale, (const float*)shift, static_cast<const __half*>(residual),
                    (int)relu, static_cast<__half*>(out)));
  return 0;
}

int ctl_bn_train_backward_nhwc_f16(const void* dz, const void* z, const void* y, int64_t rows, int32_t c, int32_t pitch,
                                   const float* gamma,
                                   const float* save_mean, const float* save_invstd, float grad_unscale, void* workspace,
                                   size_t workspace_bytes, void* g_out, float* dgamma, float* dbeta, void* dy,
                                   ctl_stream_t stream) {
  CTL_CHECK_ARG(dz && y && gamma && save_mean && save_invstd && dgamma && dbeta && dy, "null pointer");
  CTL_CHECK_ARG(z == nullptr || g_out != nullptr, "a ReLU mask (z) needs g_out (it may alias dz)");
  CTL_CHECK_ARG(pitch >= c && pitch % 8 == 0, "pitch=%d must be a multiple of 8 and >= C=%d", pitch, c);
  int rc = bn_check("bn backward", rows, c, workspace, workspace_bytes);
  if (rc) return rc;
  const BnGeom g = bn_geom(rows, c);
  float* part = static_cast<float*>(workspace);
  float* coef = part + (size_t)g.blocks * 2 * c;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t sm = (size_t)g.lanes * 2 * c * sizeof(float);
  CTL_CUDA(launch_k(bn_bwd_reduce_kernel, dim3(g.blocks), dim3(BN_THREADS), sm, st, static_cast<const __half*>(dz),
                    static_cast<const __half*>(z), static_cast<const __half*>(y), (long long)rows, (int)c, (int)pitch, g.rows_per_block,
                    g.lanes, save_mean, save_invstd, static_cast<__half*>(g_out), part));
  CTL_CUDA(launch_k(bn_bwd_finalize_kernel, dim3((c + 31) / 32), dim3(1024), 0, st, (const float*)part, g.blocks, (int)c,
                    (double)rows, gamma, save_mean, save_invstd, grad_unscale, dgamma, dbeta, coef));
  const __half* gsrc = z ? static_cast<const __half*>(g_out) : static_cast<const __half*>(dz);
  CTL_CUDA(launch_k(bn_bwd_apply_kernel, dim3(row_grid(rows, g.lanes)), dim3(BN_THREADS), 0, st, gsrc, static_cast<const __half*>(y),
                    (long long)rows, (int)c, (int)pitch, g.lanes, (const float*)coef, static_cast<__half*>(dy)));
  return 0;
}

int ctl_instnorm_train_forward_nhwc_f16(const void* y, int32_t n, int32_t hw, int32_t pitch, int32_t half, const float* gamma,
                                        const float* beta, float eps, float* save_mean, float* save_invstd, void* out,
                                        ctl_stream_t stream) {
  CTL_CHECK_ARG(y && gamma && beta && out, "null pointer");
  CTL_CHECK_ARG(!save_mean == !save_invstd, "save_mean and save_invstd are both given or both null");
  CTL_CHECK_ARG(n >= 1 && hw >= 1 && half >= 8 && half % 8 == 0 && pitch >= half && pitch % 8 == 0, "bad shape");
  int rc = ctl_device_check();
  if (rc) return rc;
  CTL_CUDA(launch_k(in_train_forward_kernel, dim3(half / 8, n), dim3(256), 0, (cudaStream_t)stream,
                    static_cast<const __half*>(y), (int)hw, (int)pitch, (int)half, gamma, beta, eps, save_mean, save_invstd,
                    static_cast<__half*>(out)));
  return 0;
}

int ctl_instnorm_relu_nhwc_f16(void* x, int32_t n, int32_t hw, int32_t c, int32_t half, const float* gamma,
                               const float* beta, float eps, ctl_stream_t stream) {
  return ctl_instnorm_train_forward_nhwc_f16(x, n, hw, c, half, gamma, beta, eps, nullptr, nullptr, x, stream);
}

int ctl_instnorm_train_backward_nhwc_f16(void* dz, const void* z, const void* y, int32_t n, int32_t hw, int32_t pitch,
                                         int32_t half, const float* gamma, const float* save_mean, const float* save_invstd,
                                         float grad_unscale, float* dgamma_part, float* dbeta_part, void* dy,
                                         ctl_stream_t stream) {
  CTL_CHECK_ARG(dz && z && y && gamma && save_mean && save_invstd && dgamma_part && dbeta_part && dy, "null pointer");
  CTL_CHECK_ARG(n >= 1 && hw >= 1 && half >= 8 && half % 8 == 0 && pitch >= half && pitch % 8 == 0, "bad shape");
  int rc = ctl_device_check();
  if (rc) return rc;
  CTL_CUDA(launch_k(in_train_backward_kernel, dim3(half / 8, n), dim3(256), 0, (cudaStream_t)stream, static_cast<__half*>(dz),
                    static_cast<const __half*>(z), static_cast<const __half*>(y), (int)hw, (int)pitch, (int)half, gamma,
                    save_mean, save_invstd, grad_unscale, dgamma_part, dbeta_part, static_cast<__half*>(dy)));
  return 0;
}

int ctl_gap_backward_nhwc_f16(const float* dfeat, int32_t n, int32_t hw, int32_t c, float scale, void* out,
                              ctl_stream_t stream) {
  CTL_CHECK_ARG(dfeat && out && n >= 1 && hw >= 1 && c % 8 == 0, "bad arguments");
  int rc = ctl_device_check();
  if (rc) return rc;
  CTL_CUDA(launch_k(gap_backward_kernel, dim3(ew_grid((long long)n * hw * (c / 8))), dim3(256), 0, (cudaStream_t)stream, dfeat,
                    (int)n, (int)hw, (int)c, scale, static_cast<__half*>(out)));
  return 0;
}

int ctl_maxpool3x3s2_backward_nhwc_f16(const void* x, const void* dy, int32_t n, int32_t h, int32_t w, int32_t c, void* dx,
                                       ctl_stream_t stream) {
  CTL_CHECK_ARG(x && dy && dx && n >= 1 && h >= 1 && w >= 1 && c % 8 == 0, "bad arguments");
  int rc = ctl_device_check();
  if (rc) return rc;
  const int Ho = (h + 2 - 3) / 2 + 1, Wo = (w + 2 - 3) / 2 + 1;
  CTL_CUDA(launch_k(maxpool_backward_kernel, dim3(ew_grid((long long)n * h * w * (c / 8))), dim3(256), 0, (cudaStream_t)stream,
                    static_cast<const __half*>(x), static_cast<const __half*>(dy), (int)n, (int)h, (int)w, (int)c, Ho, Wo,
                    static_cast<__half*>(dx)));
  return 0;
}

int ctl_maxpool3x3s2_argmax_nhwc_f16(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, void* out, void* arg_u8,
                                     ctl_stream_t stream) {
  CTL_CHECK_ARG(x && out && arg_u8 && n >= 1 && h >= 1 && w >= 1 && c % 8 == 0, "bad arguments");
  int rc = ctl_device_check();
  if (rc) return rc;
  const int Ho = (h + 2 - 3) / 2 + 1, Wo = (w + 2 - 3) / 2 + 1;
  CTL_CUDA(launch_k(maxpool_arg_kernel, dim3(ew_grid((long long)n * Ho * Wo * (c / 8))), dim3(256), 0, (cudaStream_t)stream,
                    static_cast<const __half*>(x), (int)n, (int)h, (int)w, (int)c, Ho, Wo, static_cast<__half*>(out),
                    static_cast<uint2*>(arg_u8)));
  return 0;
}

int ctl_maxpool3x3s2_backward_argmax_nhwc_f16(const void* arg_u8, const void* dy, int32_t n, int32_t h, int32_t w, int32_t c,
                                              void* dx, ctl_stream_t stream) {
  CTL_CHECK_ARG(arg_u8 && dy && dx && n >= 1 && h >= 1 && w >= 1 && c % 8 == 0, "bad arguments");
  int rc = ctl_device_check();
  if (rc) return rc;
  const int Ho = (h + 2 - 3) / 2 + 1, Wo = (w + 2 - 3) / 2 + 1;
  CTL_CUDA(launch_k(maxpool_backward_arg_kernel, dim3(ew_grid((long long)n * h * w * (c / 8))), dim3(256), 0,
                    (cudaStream_t)stream, static_cast<const uint2*>(arg_u8), static_cast<const __half*>(dy), (int)n, (int)h,
                    (int)w, (int)c, Ho, Wo, static_cast<__half*>(dx)));
  return 0;
}

int ctl_upsample2_zero_nhwc_f16(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, const void* add, void* out,
                                ctl_stream_t stream) {
  CTL_CHECK_ARG(x && out && n >= 1 && h >= 1 && w >= 1 && c % 8 == 0, "bad arguments");
  int rc = ctl_device_check();
  if (rc) return rc;
  CTL_CUDA(launch_k(upsample2_zero_kernel, dim3(ew_grid((long long)n * 4 * h * w * (c / 8))), dim3(256), 0, (cudaStream_t)stream,
                    static_cast<const __half*>(x), (int)n, (int)h, (int)w, (int)c, static_cast<const __half*>(add),
                    static_cast<__half*>(out)));
  return 0;
}

int ctl_stem_im2col_f16(const float* x_nchw, int32_t n, int32_t h, int32_t w, void* out, ctl_stream_t stream) {
  CTL_CHECK_ARG(x_nchw && out && n >= 1 && h >= 7 && w >= 7, "bad arguments");
  int rc = ctl_device_check();
  if (rc) return rc;
  CTL_CHECK_ARG(w <= IM2COL_MAXW, "stem im2col stages whole input rows: W=%d exceeds %d", w, IM2COL_MAXW);
  const int Ho = (h + 6 - 7) / 2 + 1, Wo = (w + 6 - 7) / 2 + 1;
  const size_t smem = (size_t)21 * ((w + 8) | 1) * sizeof(float);
  CTL_CUDA(launch_k(stem_im2col_kernel, dim3((unsigned)(n * Ho)), dim3(256), smem, (cudaStream_t)stream, x_nchw, (int)n, (int)h,
                    (int)w, Ho, Wo, static_cast<__half*>(out)));
  return 0;
}

}  // extern "C"
