// Trunk (ResNet50 / ResNet50-IBN-A) inference forward: fused conv + folded-BN (+ residual)
// (+ ReLU) as implicit GEMM on Hopper tensor cores (wgmma), fed by TMA.
//
// Replaces modelling/backbones/resnet.py:51-133, resnet_ibn_a.py:18-141,
// modelling/baseline.py:91-96 and the eval embedding path modelling/bases.py:169-177 /
// inference/inference_utils.py:104-113.
//
// Layout.  Activations NHWC fp16; weights [Cout][kh][kw][Cin] fp16 with the eval-mode
// BatchNorm scale folded in, bias fp32.  GEMM view: D[M = N*Ho*Wo, Cout] = A[M, K] W^T with
// K = kh*kw*Cin.  There is no im2col buffer: an M-tile is a TH x TW block of output pixels
// of one image (TH*TW = 128) and, for every filter tap (r, s) and 64-channel slab, ONE 4-D TMA
// box {64 ch, TW, TH, 1} at (c0, w0 + s - pad, h0 + r - pad, n) lands in shared memory as a
// 128-row x 128-byte K-major operand tile (SWIZZLE_128B); out-of-bounds coordinates are
// zero-filled by the TMA unit, which IS the convolution's zero padding.  Stride-2 convolutions
// read four parity views {h%2, w%2} of the input (strided tensor maps), so every box is still a
// dense stride-1 box.  Accumulators live in the registers of the two consumer warpgroups
// (64 pixels each), whose epilogue applies bias / residual / ReLU and writes fp16 NHWC.
//
// Roofline: tensor pipe for the 3x3 and wide 1x1 convolutions, HBM for the narrow 1x1s
// (arithmetic intensity 2*Cin*Cout/(2*(Cin+Cout)) flop/B < 221); algorithmic bytes per conv =
// 2*(M*Cin [if read once] + M*Cout [+ M*Cout residual]) + 2*K*Cout.
#include <stdlib.h>

#include <algorithm>

#include "common.h"
#include "wgmma.cuh"

namespace ctl {

static constexpr int CBM = 128;  // output pixels per tile
static constexpr int CBK = 64;   // channels per k-block (128 bytes)
// producer warpgroup (one TMA thread) + two consumer warpgroups, each the wgmma issuer and the
// epilogue of 64 of the tile's 128 pixels
static constexpr int CONV_THREADS = 384;
static constexpr int A_TILE_BYTES = CBM * CBK * 2;
static constexpr int A_HALF_BYTES = A_TILE_BYTES / 2;  // the 64 rows of one consumer warpgroup
// register split between the warpgroups (setmaxnreg): 128 x 40 + 256 x 232 <= 64 K registers
static constexpr uint32_t PRODUCER_REGS = 40, CONSUMER_REGS = 232;

struct ConvTap {
  int map;      // which A tensor map (parity view, or the second source of a K-concatenated 1x1)
  int dh, dw;
  int koff;     // offset of this tap's channel slab inside the weight K dimension
  int cblocks;  // 64-channel slabs of this tap (its source's Cin / 64)
};

struct ConvKernelParams {
  CUtensorMap a_map[4];
  CUtensorMap b_map;
  CUtensorMap out_map;  // NHWC output, box {64 ch, TW, TH, 1}
  CUtensorMap res_map;  // residual, same geometry
  ConvTap taps[9];
  int n_taps;
  int k_blocks;  // sum of the taps' cblocks = K / 64
  int n_img, Ho, Wo, Cout;
  int TW, TH, tiles_w, tiles_h;
  int m_tiles, n_tiles;
  const float* bias;        // [Cout]
  int has_residual;
  int relu;                 // apply ReLU to channels >= relu_from
  int relu_from;
  // chained launch (conv_gemm_kernel<BN, N2 > 0>): the next 1x1 convolution of the layer, out2 = act(out W2^T + bias2)
  // with ReLU on channels >= relu_from2, computed from the staged fp16 output tile
  CUtensorMap b2_map;    // W2 [N2][Cout] fp16, box {64, N2}
  CUtensorMap out2_map;  // NHWC [.., N2] output, box {64 ch, TW, TH, 1}
  const float* bias2;    // [N2]
  int relu_from2;
  // tap 9: the shortcut of the K-concatenated 3x3 + 1x1 form (ctl_conv3x3_dual_nhwc_f16).  It sits outside taps[]
  // because a ten-entry array changes the register allocation of conv_gemm_kernel<256> (more spill traffic).
  ConvTap tap9;
};

// Operands wait in two rings with their own depths and producers.  The A ring's 16 KiB slots carry the activation
// k-blocks and the residual slabs (one [128 px][64 ch] slab per slot); the B ring's slots carry the weight k-blocks
// and a chained launch's W2 slabs (N2 x 64 fp16, no larger than a BN = 128 slot).  So a residual slab holds one
// 16 KiB slot instead of a whole activation + weight stage, and activations, which come from HBM whenever the
// previous launch's output outgrew L2, are fetched further ahead than the L2-resident weights.
template <int BN>
struct ConvCfg {
  static constexpr int B_TILE_BYTES = BN * CBK * 2;
  // Depths from a sweep of the eval trunk at the bench shape on H100: at BN = 256, two weight slots leave the MMAs
  // waiting on L2 and cost more than any activation depth gains, so B gets three slots, A five, and the staging
  // slabs give up two of their four to make room; BN = 128 / 64 fill the same budget.
  static constexpr int A_SLOTS = BN == 256 ? 5 : 6;
  static constexpr int B_SLOTS = BN == 256 ? 3 : (BN == 128 ? 5 : 8);
  static constexpr int OUT_SLABS = 2;                  // [128 px][64 ch] fp16 staging slabs for the TMA stores
  static constexpr int BIAS_BYTES = 2048 * 4;          // the layer's whole bias vector (Cout <= 2048), loaded once
  static constexpr size_t SMEM =
      (size_t)(A_SLOTS + OUT_SLABS) * A_TILE_BYTES + (size_t)B_SLOTS * B_TILE_BYTES + BIAS_BYTES + 1024 + 256;
  static_assert(SMEM <= 227 * 1024, "conv_gemm_kernel shared memory");
  static_assert(A_SLOTS >= 2 && B_SLOTS >= 2 && 2 * (A_SLOTS + B_SLOTS) * 8 <= 256, "ring depths / barrier space");
};

// a position in a ring of S slots: the slot, and the parity of the current pass over the ring (the mbarrier phase)
template <int S>
struct RingPos {
  int slot = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void next() {
    if (++slot == S) {
      slot = 0;
      phase ^= 1u;
    }
  }
  __device__ __forceinline__ int prev() const { return slot == 0 ? S - 1 : slot - 1; }
};

// Tile order: n fastest, then pixel tiles row-major inside an image, then images.  An unchained launch of more than
// one n-tile deals the tiles round-robin: CTA c takes tiles c, c + grid, c + 2 grid, ...  So the CTAs running at any
// moment hold every n-tile of a few consecutive m-tiles, and the n_tiles reads of one activation tile fall within one
// tile's runtime: the first brings its lines into L2 and the others hit them.  A contiguous range per CTA instead
// spaces those reads one tile apart per CTA while all other CTAs stream their own activation tiles through L2; where
// those add up to more than L2 (layer4 at the bench shape: 132 x 512 KB), each n-tile re-reads its activation tile
// from HBM.  A launch of one n-tile has no such re-read and keeps a contiguous range per CTA: the order in which it
// reads its input then matches what the launch before it left in L2.  A chained launch (N2 > 0) owns a contiguous
// range of whole m-tiles.  In a contiguous range the coordinates advance by carries; a round-robin step recomputes
// them from the tile index (a few integer divisions per tile).
struct TileIter {
  int nt, tw, th, img;
  __device__ __forceinline__ void init(int tile, const ConvKernelParams& p) {
    const int mt = tile / p.n_tiles;
    nt = tile - mt * p.n_tiles;
    const int per_img = p.tiles_w * p.tiles_h;
    img = mt / per_img;
    const int tr = mt - img * per_img;
    th = tr / p.tiles_w;
    tw = tr - th * p.tiles_w;
  }
  __device__ __forceinline__ void next(const ConvKernelParams& p) {
    if (++nt == p.n_tiles) {
      nt = 0;
      if (++tw == p.tiles_w) {
        tw = 0;
        if (++th == p.tiles_h) {
          th = 0;
          ++img;
        }
      }
    }
  }
  // to `tile`, `step` tiles after the current one
  __device__ __forceinline__ void advance(int tile, int step, const ConvKernelParams& p) {
    if (step == 1)
      next(p);
    else
      init(tile, p);
  }
};

// One 64-channel sub-tile of a consumer warpgroup's accumulator (d = its 32 registers, channels ch0 .. ch0 + 63 of
// the n-tile) -> (+residual) +bias, ReLU from channel relu_from on -> fp16 -> rows of the swizzled [128 px][64 ch]
// staging slab.  `res` (may be null) is a [128 px][64 ch] fp16 residual tile in the same swizzled layout, as the TMA
// unit lands it; it is added before the bias.
__device__ __forceinline__ void store_subtile_f16(const float* d, uint8_t* slab, int row0, const float* bias, int ch_abs0,
                                                  int relu, int relu_from, const uint8_t* res = nullptr) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = 8 * i + 2 * (lane & 3);
    const float2 bb = *reinterpret_cast<const float2*>(bias + c);
    const bool do_relu = relu && ch_abs0 + c >= relu_from;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int px = row0 + (lane >> 2) + 8 * h;
      const int off = px * 128 + ((i ^ (px & 7)) << 4) + (lane & 3) * 4;
      float a0 = d[4 * i + 2 * h], a1 = d[4 * i + 2 * h + 1];
      if (res) {
        const float2 r = __half22float2(*reinterpret_cast<const __half2*>(res + off));
        a0 += r.x;
        a1 += r.y;
      }
      float v0 = a0 + bb.x, v1 = a1 + bb.y;
      if (do_relu) {
        v0 = fmaxf(v0, 0.f);
        v1 = fmaxf(v1, 0.f);
      }
      *reinterpret_cast<__half2*>(slab + off) = __floats2half2_rn(v0, v1);
    }
  }
}

// N2 > 0: chained launch.  Staging slab j of an output tile is exactly the K-major SWIZZLE_128B A operand of
// k-block (nt * BN / 64 + j) of the next 1x1 convolution (K2 = Cout, N2 outputs), so once a slab is complete each
// consumer warpgroup issues that k-block (m64 nN2 k16 x 4, the shape and k order of the stand-alone launch: same bits)
// into a second accumulator that lives across the m-tile's n-tiles; its weight slab W2[:, 64 kb .. 64 kb + 63] rides
// the B ring after the tile's weight k-blocks.  After the last n-tile the second accumulator goes through the
// same epilogue into out2, so the block output is never re-read from HBM.  Each CTA owns whole m-tiles.
template <int BN, int N2 = 0>
__global__ void __launch_bounds__(CONV_THREADS, 1) conv_gemm_kernel(const __grid_constant__ ConvKernelParams p) {
  using Cfg = ConvCfg<BN>;
  constexpr int NSUB = BN / 64;
  static_assert(N2 == 0 || N2 == 64 || N2 == 128, "chained 1x1 width");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t ring_b = smem_base + Cfg::A_SLOTS * A_TILE_BYTES;
  const uint32_t out_stage = ring_b + Cfg::B_SLOTS * Cfg::B_TILE_BYTES;
  const uint32_t bias_sm = out_stage + Cfg::OUT_SLABS * A_TILE_BYTES;
  const uint32_t bar_base = bias_sm + Cfg::BIAS_BYTES;
  auto a_slot = [&](int s) { return smem_base + s * A_TILE_BYTES; };
  auto b_slot = [&](int s) { return ring_b + s * Cfg::B_TILE_BYTES; };
  auto a_full = [&](int s) { return bar_base + 8u * s; };
  auto a_empty = [&](int s) { return bar_base + 8u * (Cfg::A_SLOTS + s); };
  auto b_full = [&](int s) { return bar_base + 8u * (2 * Cfg::A_SLOTS + s); };
  auto b_empty = [&](int s) { return bar_base + 8u * (2 * Cfg::A_SLOTS + Cfg::B_SLOTS + s); };
  uint8_t* gsm = smem_raw + (smem_base - smem_u32(smem_raw));  // generic view of the aligned arena

  const int warp = threadIdx.x >> 5;
  const int num_tiles = p.m_tiles * p.n_tiles;
  const int conv_kblocks = p.k_blocks;
  // this CTA's tiles: t_begin, t_begin + t_step, ... < t_end (see "Tile order"); both producers and both consumer
  // warpgroups walk the same sequence
  int t_begin = (int)blockIdx.x, t_end = num_tiles, t_step = (int)gridDim.x;
  if (N2 > 0 || p.n_tiles == 1) {  // a contiguous, balanced range of whole m-tiles
    const int per = p.m_tiles / (int)gridDim.x, rem = p.m_tiles - per * (int)gridDim.x;
    t_begin = ((int)blockIdx.x * per + min((int)blockIdx.x, rem)) * p.n_tiles;
    t_end = t_begin + (per + ((int)blockIdx.x < rem ? 1 : 0)) * p.n_tiles;
    t_step = 1;
  }

  if (threadIdx.x == 0) {
    for (int s = 0; s < Cfg::A_SLOTS; ++s) {
      mbar_init(a_full(s), 1);
      mbar_init(a_empty(s), 2);  // one arrive per consumer warpgroup
    }
    for (int s = 0; s < Cfg::B_SLOTS; ++s) {
      mbar_init(b_full(s), 1);
      mbar_init(b_empty(s), 2);
    }
    fence_barrier_init();
    for (int i = 0; i < 4; ++i) tma_prefetch_desc(&p.a_map[i]);
    tma_prefetch_desc(&p.b_map);
    tma_prefetch_desc(&p.out_map);
    tma_prefetch_desc(&p.res_map);
    if constexpr (N2 > 0) {
      tma_prefetch_desc(&p.b2_map);
      tma_prefetch_desc(&p.out2_map);
    }
  }
  for (int i = threadIdx.x; i < p.Cout; i += blockDim.x)
    reinterpret_cast<float*>(gsm + (bias_sm - smem_base))[i] = p.bias[i];
  if constexpr (N2 > 0)  // bias2 right after bias (Cout + N2 <= 2048)
    for (int i = threadIdx.x; i < N2; i += blockDim.x)
      reinterpret_cast<float*>(gsm + (bias_sm - smem_base))[p.Cout + i] = p.bias2[i];
  __syncthreads();
  pdl_launch_dependents();  // the next kernel may begin its prologue
  pdl_wait();               // activations of the previous kernel are complete and visible

  if (warp < 4) {
    // ===================== TMA producers: one thread per ring =====================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      // A ring: the tile's activation k-blocks, then its residual slabs, one per 64 output channels, each read by
      // the epilogue of that sub-tile straight from its slot
      RingPos<Cfg::A_SLOTS> ra;
      TileIter it;
      it.init(t_begin, p);
      for (int tile = t_begin; tile < t_end; tile += t_step, it.advance(tile, t_step, p)) {
        const int h0 = it.th * p.TH, w0 = it.tw * p.TW;
        for (int t = 0; t < p.n_taps; ++t) {
          const ConvTap tap = t < 9 ? p.taps[t] : p.tap9;
          for (int cb = 0; cb < tap.cblocks; ++cb) {
            mbar_wait(a_empty(ra.slot), ra.phase ^ 1u);
            mbar_arrive_expect_tx(a_full(ra.slot), A_TILE_BYTES);
            tma_load_4d(a_slot(ra.slot), &p.a_map[tap.map], a_full(ra.slot), cb * CBK, w0 + tap.dw, h0 + tap.dh,
                        it.img);
            ra.next();
          }
        }
        if (p.has_residual) {
          for (int j = 0; j < NSUB; ++j) {
            mbar_wait(a_empty(ra.slot), ra.phase ^ 1u);
            mbar_arrive_expect_tx(a_full(ra.slot), A_TILE_BYTES);
            tma_load_4d(a_slot(ra.slot), &p.res_map, a_full(ra.slot), it.nt * BN + j * 64, w0, h0, it.img);
            ra.next();
          }
        }
      }
    } else if (threadIdx.x == 32) {
      // B ring: the tile's weight k-blocks, then (chained launch) the W2 slab of each sub-tile's GEMM2 k-block
      RingPos<Cfg::B_SLOTS> rb;
      TileIter it;
      it.init(t_begin, p);
      for (int tile = t_begin; tile < t_end; tile += t_step, it.advance(tile, t_step, p)) {
        for (int t = 0; t < p.n_taps; ++t) {
          const ConvTap tap = t < 9 ? p.taps[t] : p.tap9;
          for (int cb = 0; cb < tap.cblocks; ++cb) {
            mbar_wait(b_empty(rb.slot), rb.phase ^ 1u);
            mbar_arrive_expect_tx(b_full(rb.slot), Cfg::B_TILE_BYTES);
            tma_load_2d(b_slot(rb.slot), &p.b_map, b_full(rb.slot), tap.koff + cb * CBK, it.nt * BN);
            rb.next();
          }
        }
        if constexpr (N2 > 0) {
          for (int j = 0; j < NSUB; ++j) {
            mbar_wait(b_empty(rb.slot), rb.phase ^ 1u);
            mbar_arrive_expect_tx(b_full(rb.slot), N2 * CBK * 2);
            tma_load_2d(b_slot(rb.slot), &p.b2_map, b_full(rb.slot), it.nt * BN + j * 64, 0);
            rb.next();
          }
        }
      }
    }
  } else {
    // ===== consumers: warpgroup wg issues the wgmmas of tile rows [64 wg, 64 wg + 64) (M = 64, N = BN) into its
    // registers, then drains them in 64-channel sub-tiles: (+residual from the A ring, +bias, ReLU) -> fp16 ->
    // swizzled staging slab shared by both warpgroups -> one TMA store per sub-tile; OUT_SLABS slabs keep up to
    // OUT_SLABS - 1 stores in flight.
    setmaxnreg_inc<CONSUMER_REGS>();
    const int wg = (threadIdx.x >> 7) - 1;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const bool leader = threadIdx.x == 128;
    const int row0 = 64 * wg + 16 * (warp & 3);  // first accumulator row of this warp
    uint8_t* oslabs = gsm + (out_stage - smem_base);
    const float* bias_s = reinterpret_cast<const float*>(gsm + (bias_sm - smem_base));
    float acc[BN / 2];
    [[maybe_unused]] float acc2[N2 > 0 ? N2 / 2 : 1];  // GEMM2 (chained launch only)
    RingPos<Cfg::A_SLOTS> ra;
    RingPos<Cfg::B_SLOTS> rb;
    uint32_t g = 0;  // running sub-tile counter -> staging slab
    TileIter it;
    it.init(t_begin, p);
    for (int tile = t_begin; tile < t_end; tile += t_step, it.advance(tile, t_step, p)) {
      const int h0 = it.th * p.TH, w0 = it.tw * p.TW;
      for (int kb = 0; kb < conv_kblocks; ++kb) {
        mbar_wait(a_full(ra.slot), ra.phase);
        mbar_wait(b_full(rb.slot), rb.phase);
        const uint64_t da = make_sw128_kmajor_desc(a_slot(ra.slot) + wg * A_HALF_BYTES);
        const uint64_t db = make_sw128_kmajor_desc(b_slot(rb.slot));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < CBK / 16; ++k)
          wgmma_f16<BN>(acc, desc_advance_k(da, k), desc_advance_k(db, k), (kb > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's group is done reading its slots
        if (kb > 0 && wg_leader) {
          mbar_arrive(a_empty(ra.prev()));
          mbar_arrive(b_empty(rb.prev()));
        }
        ra.next();
        rb.next();
      }
      wgmma_wait<0>();
      if (wg_leader) {  // the last k-block's slots
        mbar_arrive(a_empty(ra.prev()));
        mbar_arrive(b_empty(rb.prev()));
      }
#pragma unroll
      for (int j = 0; j < NSUB; ++j, ++g) {
        const uint32_t b = g & (Cfg::OUT_SLABS - 1);
        const uint8_t* res = nullptr;
        if (p.has_residual) {  // this sub-tile's residual slab, next in the A ring
          mbar_wait(a_full(ra.slot), ra.phase);
          res = gsm + ra.slot * A_TILE_BYTES;
        }
        // slab b was handed to a TMA store OUT_SLABS sub-tiles ago: wait until that store has read it
        if (leader) tma_store_wait_read<Cfg::OUT_SLABS - 1>();
        named_bar_sync(1, 256);
        store_subtile_f16(acc + 32 * j, oslabs + b * A_TILE_BYTES, row0, bias_s + it.nt * BN + j * 64,
                          it.nt * BN + j * 64, p.relu, p.relu_from, res);
        fence_proxy_async();     // staging writes (generic proxy) -> visible to the TMA store (async proxy)
        named_bar_sync(1, 256);  // slab complete; both warpgroups are done with the residual slot
        if (p.has_residual) {
          if (wg_leader) mbar_arrive(a_empty(ra.slot));
          ra.next();
        }
        if (leader) {
          tma_store_4d(&p.out_map, out_stage + b * A_TILE_BYTES, it.nt * BN + j * 64, w0, h0, it.img);
          tma_store_commit();
        }
        if constexpr (N2 > 0) {
          // GEMM2 k-block nt * NSUB + j from this warpgroup's 64 rows of slab b.  Each warpgroup reads only the rows it
          // wrote, and the group reading slab b has completed (wgmma_wait<1> one sub-tile later) before it is rewritten.
          mbar_wait(b_full(rb.slot), rb.phase);
          const uint64_t da = make_sw128_kmajor_desc(out_stage + b * A_TILE_BYTES + wg * A_HALF_BYTES);
          const uint64_t db = make_sw128_kmajor_desc(b_slot(rb.slot));
          const bool first = it.nt == 0 && j == 0;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < CBK / 16; ++k)
            wgmma_f16<N2>(acc2, desc_advance_k(da, k), desc_advance_k(db, k), (!first || k > 0) ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();
          if (j > 0 && wg_leader) mbar_arrive(b_empty(rb.prev()));  // the previous W2 slab, one slot back in the B ring
          rb.next();
        }
      }
      if constexpr (N2 > 0) {
        wgmma_wait<0>();
        if (wg_leader) mbar_arrive(b_empty(rb.prev()));  // the last W2 slab
        if (it.nt == p.n_tiles - 1) {  // the m-tile's GEMM2 is complete: its epilogue, into out2
#pragma unroll
          for (int j = 0; j < N2 / 64; ++j, ++g) {
            const uint32_t b = g & (Cfg::OUT_SLABS - 1);
            if (leader) tma_store_wait_read<Cfg::OUT_SLABS - 1>();
            named_bar_sync(1, 256);
            store_subtile_f16(acc2 + 32 * j, oslabs + b * A_TILE_BYTES, row0, bias_s + p.Cout + j * 64, j * 64, 1,
                              p.relu_from2);
            fence_proxy_async();
            named_bar_sync(1, 256);
            if (leader) {
              tma_store_4d(&p.out2_map, out_stage + b * A_TILE_BYTES, j * 64, w0, h0, it.img);
              tma_store_commit();
            }
          }
        }
      }
    }
    if (leader) tma_store_wait<0>();  // shared memory must outlive the last stores
  }
}

// ---------------------------------------------------------------------------------------
// 3x3 / stride 1 / 64 -> 64 channels (layer1.conv2, the most fill-bound layer of the trunk: the
// generic kernel re-reads the activation tile once per filter tap, 216 KiB of shared-memory fill
// for 9.4 MFLOP).  Here the 9 x [64 x 64] weight slabs (72 KiB) stay RESIDENT in shared memory and
// each 16 x 8 output tile loads ONE halo slab -- 18 rows x 16 pixel lines x 128 B, i.e. the 18 x 10
// halo padded to a 2 KiB row pitch -- by a single TMA box; the nine taps are nine SHIFTED VIEWS of
// that slab: descriptor start = slab + (r*16 + s)*128 B, 8-row groups 2 KiB apart (one output row
// each).  The 128-byte-swizzle XOR is a function of the absolute shared-memory address bits [7,10)
// -- exactly what the TMA unit used when it wrote the slab -- so a start address shifted by whole
// 128-byte lines needs NO descriptor base_offset (tests/test_trunk_gpu.py::test_conv_shapes[case3]
// pins this).  36 KiB of fill per tile instead of 216 KiB.  Consumer warpgroup wg computes output
// rows [8 wg, 8 wg + 8) of the tile (M = 64, N = 64).
//
// RES (a BasicBlock's layer1 conv2, identity shortcut): the tile's [128 px][64 ch] residual is one more TMA box of the
// output's geometry, landed in its own 16 KiB slab in the swizzled layout store_subtile_f16 reads.  Shared memory:
// 72 KiB weights + 2 x 36 KiB halos + 4 x 16 KiB output slabs + 16 KiB residual + 512 B bias + barriers and the
// 1 KiB alignment slack = 225.75 KiB of the 227 KiB an SM grants one CTA.  A second producer thread (warp 1) owns the
// residual slab: it loads tile t + 1's residual as soon as the epilogue of tile t has read the slab, while the
// consumers run tile t + 1's MMAs, so the halo ring never waits on it.
// ---------------------------------------------------------------------------------------
static constexpr int C64_HALO_BYTES = 18 * 16 * 128;  // 36 KiB
static constexpr int C64_W_BYTES = 9 * 64 * 128;      // 72 KiB
static constexpr int C64_HALOS = 2;
static constexpr int C64_OUT_SLABS = 4;
template <bool RES>
struct C64Cfg {
  static constexpr int RES_BYTES = RES ? A_TILE_BYTES : 0;
  static constexpr size_t SMEM =
      C64_W_BYTES + C64_HALOS * C64_HALO_BYTES + C64_OUT_SLABS * A_TILE_BYTES + RES_BYTES + 512 + 1024 + 256;
  static_assert(SMEM <= 227 * 1024, "conv3x3_c64_kernel shared memory");
};

struct C64Params {
  CUtensorMap x_map;    // NHWC input, box {64, 16, 18, 1}
  CUtensorMap w_map;    // [64][576] weights, box {64, 64}
  CUtensorMap out_map;  // NHWC output, box {64, 8, 16, 1}
  const float* bias;
  int n_img, H, W, tiles_h, tiles_w, relu;
  CUtensorMap res_map;  // NHWC residual (RES), box {64, 8, 16, 1}
};

template <bool RES>
__global__ void __launch_bounds__(CONV_THREADS, 1) conv3x3_c64_kernel(const __grid_constant__ C64Params p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t w_sm = smem_base;
  const uint32_t halo_sm = w_sm + C64_W_BYTES;
  const uint32_t out_stage = halo_sm + C64_HALOS * C64_HALO_BYTES;
  const uint32_t res_sm = out_stage + C64_OUT_SLABS * A_TILE_BYTES;  // 1024-aligned, like every slab
  const uint32_t bias_sm = res_sm + C64Cfg<RES>::RES_BYTES;
  const uint32_t bar_base = bias_sm + 512;
  const uint32_t w_bar = bar_base;
  auto full_bar = [&](int s) { return bar_base + 8u * (1 + s); };
  auto empty_bar = [&](int s) { return bar_base + 8u * (1 + C64_HALOS + s); };
  const uint32_t res_full = bar_base + 8u * (1 + 2 * C64_HALOS), res_empty = res_full + 8u;
  uint8_t* gsm = smem_raw + (smem_base - smem_u32(smem_raw));
  const int warp = threadIdx.x >> 5;
  const int tiles_per_img = p.tiles_h * p.tiles_w;
  const int num_tiles = p.n_img * tiles_per_img;
  const int per = num_tiles / (int)gridDim.x, rem = num_tiles - per * (int)gridDim.x;
  const int t_begin = (int)blockIdx.x * per + min((int)blockIdx.x, rem);
  const int t_end = t_begin + per + ((int)blockIdx.x < rem ? 1 : 0);
  auto coords = [&](int tile, int& w0, int& h0, int& img) {
    img = tile / tiles_per_img;
    const int tr = tile - img * tiles_per_img;
    h0 = (tr / p.tiles_w) * 16;
    w0 = (tr % p.tiles_w) * 8;
  };
  if (threadIdx.x == 0) {
    mbar_init(w_bar, 1);
    for (int s = 0; s < C64_HALOS; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);
    }
    if constexpr (RES) {
      mbar_init(res_full, 1);
      mbar_init(res_empty, 1);
    }
    fence_barrier_init();
    tma_prefetch_desc(&p.x_map);
    tma_prefetch_desc(&p.w_map);
    tma_prefetch_desc(&p.out_map);
    if constexpr (RES) tma_prefetch_desc(&p.res_map);
  }
  if (threadIdx.x >= 128 && threadIdx.x < 192) reinterpret_cast<float*>(gsm + (bias_sm - smem_base))[threadIdx.x - 128] = p.bias[threadIdx.x - 128];
  __syncthreads();
  pdl_launch_dependents();  // the next kernel may begin its prologue
  pdl_wait();               // activations of the previous kernel are complete and visible

  if (warp < 4) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(w_bar, C64_W_BYTES);
      for (int t = 0; t < 9; ++t) tma_load_2d(w_sm + t * 64 * 128, &p.w_map, w_bar, t * 64, 0);
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = t_begin; tile < t_end; ++tile) {
        int w0, h0, img;
        coords(tile, w0, h0, img);
        mbar_wait(empty_bar(stage), phase ^ 1u);
        mbar_arrive_expect_tx(full_bar(stage), C64_HALO_BYTES);
        tma_load_4d(halo_sm + stage * C64_HALO_BYTES, &p.x_map, full_bar(stage), 0, w0 - 1, h0 - 1, img);
        if (++stage == C64_HALOS) {
          stage = 0;
          phase ^= 1u;
        }
      }
    }
    if constexpr (RES) {
      if (threadIdx.x == 32) {  // the residual slab: one load per tile, once the previous tile's epilogue has read it
        uint32_t phase = 0;
        for (int tile = t_begin; tile < t_end; ++tile) {
          int w0, h0, img;
          coords(tile, w0, h0, img);
          mbar_wait(res_empty, phase ^ 1u);
          mbar_arrive_expect_tx(res_full, A_TILE_BYTES);
          tma_load_4d(res_sm, &p.res_map, res_full, 0, w0, h0, img);
          phase ^= 1u;
        }
      }
    }
  } else {
    setmaxnreg_inc<CONSUMER_REGS>();
    const int wg = (threadIdx.x >> 7) - 1;
    const bool leader = threadIdx.x == 128;
    const int row0 = 64 * wg + 16 * (warp & 3);
    uint8_t* oslabs = gsm + (out_stage - smem_base);
    const float* bias_s = reinterpret_cast<const float*>(gsm + (bias_sm - smem_base));
    mbar_wait(w_bar, 0);
    float acc[32];
    int stage = 0;
    uint32_t phase = 0, g = 0;
    for (int tile = t_begin; tile < t_end; ++tile, ++g) {
      int w0, h0, img;
      coords(tile, w0, h0, img);
      mbar_wait(full_bar(stage), phase);
      const uint32_t slab = halo_sm + stage * C64_HALO_BYTES + wg * 8 * 2048;
      wgmma_fence();
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const int r = t / 3, s = t - 3 * r;
        const uint32_t a0 = slab + (r * 16 + s) * 128;
        const uint64_t da = make_sw128_kmajor_desc(a0, 2048);
        const uint64_t db = make_sw128_kmajor_desc(w_sm + t * 64 * 128);
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_f16<64>(acc, desc_advance_k(da, k), desc_advance_k(db, k), (t | k) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(empty_bar(stage));
      if (++stage == C64_HALOS) {
        stage = 0;
        phase ^= 1u;
      }
      const uint32_t b = g & (C64_OUT_SLABS - 1);
      if (leader) tma_store_wait_read<C64_OUT_SLABS - 1>();
      named_bar_sync(1, 256);
      if constexpr (RES) {
        mbar_wait(res_full, g & 1u);
        store_subtile_f16(acc, oslabs + b * A_TILE_BYTES, row0, bias_s, 0, p.relu, 0, gsm + (res_sm - smem_base));
      } else {
        store_subtile_f16(acc, oslabs + b * A_TILE_BYTES, row0, bias_s, 0, p.relu, 0);
      }
      fence_proxy_async();
      named_bar_sync(1, 256);
      if (leader) {
        if constexpr (RES) mbar_arrive(res_empty);  // both warpgroups have read the residual slab
        tma_store_4d(&p.out_map, out_stage + b * A_TILE_BYTES, 0, w0, h0, img);
        tma_store_commit();
      }
    }
    if (leader) tma_store_wait<0>();
  }
}

// ---------------------------------------------------------------------------------------
// stem on the tensor cores: the 7x7/2 convolution as a GEMM with K = 21 (c, r) groups x 8
// (s = 0..6 plus one zero column) = 168, padded to 192 = three 64-wide K slabs.
// Per tile of 4 x 32 output pixels: the fp32 NCHW input patch (13 x 72 x 3) is converted to
// fp16 in shared memory, every thread then assembles 16-byte K-chunks -- the 8 taps of one
// (c, r) group are 8 CONSECUTIVE patch columns -- straight into the SWIZZLE_128B operand
// layout (generic-proxy stores + fence.proxy.async), one warpgroup issues 2 x 12 wgmma
// (M=64, N=64), adds the folded-BN bias (+ReLU for IBN) and writes one full 128-byte NHWC line
// per pixel.  Weights [64][192] fp16 stay resident in shared memory.
// ---------------------------------------------------------------------------------------
static constexpr int SK = 192;                    // padded K
static constexpr int S_TH = 4, S_TW = 32;         // output tile
static constexpr int S_PH = 2 * S_TH + 5;         // 13 input rows
static constexpr int S_PW = 72;                   // 2*32 + 5 = 69 input columns, padded to 72
static constexpr int STEM_BUILDERS = 256;                   // warpgroups 0-1 assemble operand tiles
static constexpr int STEM_TC_THREADS = STEM_BUILDERS + 128;  // + the MMA / epilogue warpgroup
static constexpr int S_A_BYTES = 3 * A_TILE_BYTES;          // 48 KiB: three [128][64] fp16 slabs
static constexpr int S_B_BYTES = 3 * 64 * 128;              // 24 KiB: three [64][64] fp16 slabs
static constexpr int S_PATCH_BYTES = 3 * S_PH * S_PW * 2;   // 5.6 KiB
static constexpr size_t STEM_TC_SMEM =
    2 * S_A_BYTES + S_B_BYTES + 2 * A_TILE_BYTES /*store staging*/ + 2 * S_PATCH_BYTES + 1024 + 128 + 256;

struct StemParams {
  CUtensorMap w_map;    // [64][192] fp16, box {64, 64}
  CUtensorMap out_map;  // NHWC fp16 output, box {64 ch, 32, 4, 1}
  const float* x;       // NCHW fp32
  const float* bias;
  __half* out;        // NHWC fp16 [n, Ho, Wo, 64]
  int n_img, H, W, Ho, Wo, tiles_h, tiles_w, relu;
};

// Persistent, one CTA per SM, two roles connected by mbarriers:
//   builders (8 warps): prefetched fp32 patch -> fp16 patch in smem -> swizzled operand tile A[buf]
//   MMA warpgroup     : 2 x 12 wgmma (M=64, N=64) per tile -> +bias (+ReLU) -> fp16 -> one TMA store per tile
// A and the patch are double-buffered, so the builders assemble tile i+1 while tile i is multiplied.
__global__ void __launch_bounds__(STEM_TC_THREADS, 1) stem_tc_kernel(const __grid_constant__ StemParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t sA = base, sB = base + 2 * S_A_BYTES, sO = sB + S_B_BYTES;
  constexpr int S_FIXED = 2 * S_A_BYTES + S_B_BYTES + 2 * A_TILE_BYTES;
  __half* patch0 = reinterpret_cast<__half*>(gbase + S_FIXED);
  const uint32_t bars = base + S_FIXED + 2 * S_PATCH_BYTES;
  const uint32_t bar_w = bars;  // weights landed
  auto a_full = [&](int b) { return bars + 8u * (1 + b); };
  auto a_empty = [&](int b) { return bars + 8u * (3 + b); };
  float* bias_s = reinterpret_cast<float*>(gbase + S_FIXED + 2 * S_PATCH_BYTES + 128);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid < 64) bias_s[tid] = p.bias[tid];
  if (tid == 0) {
    mbar_init(bar_w, 1);
    for (int b = 0; b < 2; ++b) {
      mbar_init(a_full(b), STEM_BUILDERS / 32);  // one arrive per builder warp
      mbar_init(a_empty(b), 1);
    }
    fence_barrier_init();
    tma_prefetch_desc(&p.w_map);
    tma_prefetch_desc(&p.out_map);
  }
  if (tid < STEM_BUILDERS) {
    // the three zero chunks (k = 168..191) of every pixel never change: chunks 5,6,7 of slab 2, both buffers
    for (int q = tid; q < 2 * 128 * 3; q += STEM_BUILDERS) {
      const int buf = q / 384, qq = q - buf * 384, px = qq & 127, ch = 5 + (qq >> 7);
      *reinterpret_cast<uint4*>(gbase + buf * S_A_BYTES + 2 * A_TILE_BYTES + px * 128 + ((ch ^ (px & 7)) << 4)) =
          make_uint4(0, 0, 0, 0);
    }
    fence_proxy_async();
  }
  __syncthreads();
  pdl_launch_dependents();  // the next kernel may begin its prologue
  pdl_wait();               // activations of the previous kernel are complete and visible
  const int tiles_per_img = p.tiles_h * p.tiles_w;
  const int num_tiles = p.n_img * tiles_per_img;

  if (tid < STEM_BUILDERS) {
    constexpr int NPRE = (3 * S_PH * S_PW + STEM_BUILDERS - 1) / STEM_BUILDERS;  // 11 loads in flight / thread
    float pre[NPRE];
    // tile-independent part of every patch element this thread owns: offset inside the image and (ph, pw)
    int p_off[NPRE], p_hw[NPRE];
#pragma unroll
    for (int j = 0; j < NPRE; ++j) {
      const int e = tid + j * STEM_BUILDERS;
      const int c = e / (S_PH * S_PW), rem = e - c * (S_PH * S_PW), ph = rem / S_PW, pw = rem - ph * S_PW;
      p_off[j] = (c * p.H + ph) * p.W + pw;
      p_hw[j] = e < 3 * S_PH * S_PW ? ((ph << 16) | pw) : (1 << 30);  // out-of-range marker fails the row test
    }
    auto load_patch = [&](int tile) {  // fp32 NCHW -> registers, zero outside the image
      const int img = tile / tiles_per_img, tr = tile - img * tiles_per_img;
      const int ih0 = 2 * ((tr / p.tiles_w) * S_TH) - 3, iw0 = 2 * ((tr % p.tiles_w) * S_TW) - 3;
      const float* xb = p.x + (size_t)img * 3 * p.H * p.W + (long long)ih0 * p.W + iw0;
#pragma unroll
      for (int j = 0; j < NPRE; ++j) {
        const int ih = ih0 + (p_hw[j] >> 16), iw = iw0 + (p_hw[j] & 0xFFFF);
        float v = 0.f;
        if ((unsigned)ih < (unsigned)p.H && (unsigned)iw < (unsigned)p.W) v = __ldg(xb + p_off[j]);
        pre[j] = v;
      }
    };
    // per-thread constants of the operand assembly: pixel px, (c, r) groups cr = 2 i + hi
    const int px = tid & 127, hi = tid >> 7;
    int src_off[11], dst_off[11];
#pragma unroll
    for (int i = 0; i < 11; ++i) {
      const int cr = 2 * i + hi, c = cr / 7, r = cr - c * 7;
      src_off[i] = (c * S_PH + 2 * (px >> 5) + r) * S_PW + 2 * (px & 31);
      dst_off[i] = (cr >> 3) * A_TILE_BYTES + px * 128 + (((cr & 7) ^ (px & 7)) << 4);
    }
    if ((int)blockIdx.x < num_tiles) load_patch(blockIdx.x);
    int buf = 0;
    uint32_t eph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      __half* patch = patch0 + buf * (S_PATCH_BYTES / 2);
#pragma unroll
      for (int j = 0; j < NPRE; ++j) {
        const int e = tid + j * STEM_BUILDERS;
        if (e < 3 * S_PH * S_PW) patch[e] = __float2half_rn(pre[j]);
      }
      named_bar_sync(2, STEM_BUILDERS);  // patch[buf] complete (its previous readers finished two tiles ago)
      if (tile + (int)gridDim.x < num_tiles) load_patch(tile + gridDim.x);  // next patch travels during the build
      mbar_wait(a_empty(buf), eph ^ 1u);  // the MMAs that read A[buf] two tiles ago have completed
      uint8_t* A = gbase + buf * S_A_BYTES;
#pragma unroll
      for (int i = 0; i < 11; ++i) {
        if (2 * i + hi < 21) {
          const uint32_t* src = reinterpret_cast<const uint32_t*>(patch + src_off[i]);
          *reinterpret_cast<uint4*>(A + dst_off[i]) = make_uint4(src[0], src[1], src[2], src[3]);
        }
      }
      fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
      __syncwarp();
      if (lane == 0) mbar_arrive(a_full(buf));
      if (++buf == 2) {
        buf = 0;
        eph ^= 1u;
      }
    }
  } else {
    const bool leader = tid == STEM_BUILDERS;
    if (leader) {
      mbar_arrive_expect_tx(bar_w, S_B_BYTES);
      for (int kb = 0; kb < 3; ++kb) tma_load_2d(sB + kb * 64 * 128, &p.w_map, bar_w, kb * 64, 0);
    }
    mbar_wait(bar_w, 0);
    float acc[2][32];
    int buf = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int img = tile / tiles_per_img, tr = tile - img * tiles_per_img;
      const int oh0 = (tr / p.tiles_w) * S_TH, ow0 = (tr % p.tiles_w) * S_TW;
      mbar_wait(a_full(buf), ph);  // operand tile assembled
      wgmma_fence();
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int kb = 0; kb < 3; ++kb) {
          const uint64_t da = make_sw128_kmajor_desc(sA + buf * S_A_BYTES + kb * A_TILE_BYTES + h * A_HALF_BYTES);
          const uint64_t db = make_sw128_kmajor_desc(sB + kb * 64 * 128);
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_f16<64>(acc[h], desc_advance_k(da, k), desc_advance_k(db, k), (kb | k) ? 1u : 0u);
        }
      wgmma_commit();
      wgmma_wait<0>();
      if (leader) mbar_arrive(a_empty(buf));
      if (leader) tma_store_wait_read<1>();  // staging slab `buf` was stored two tiles ago
      named_bar_sync(3, 128);
      uint8_t* slab = gbase + 2 * S_A_BYTES + S_B_BYTES + buf * A_TILE_BYTES;
#pragma unroll
      for (int h = 0; h < 2; ++h) store_subtile_f16(acc[h], slab, 64 * h + 16 * (warp & 3), bias_s, 0, p.relu, 0);
      fence_proxy_async();
      named_bar_sync(3, 128);
      if (leader) {
        tma_store_4d(&p.out_map, sO + buf * A_TILE_BYTES, 0, ow0, oh0, img);
        tma_store_commit();
      }
      if (++buf == 2) {
        buf = 0;
        ph ^= 1u;
      }
    }
    if (leader) tma_store_wait<0>();
  }
}

// =======================================================================================
// Fused stem: conv 7x7 / 2 (+folded BN, optional ReLU) -> maxpool 3x3 / 2, for inputs up to 128 pixels wide.
//
// The input is first packed to zero-bordered NHWC4 fp16 (stem_pack_input_kernel: [N][H+6][136][4], 8 bytes per
// pixel, 3 border pixels left/top).  In that layout the 7-pixel window of output column ox starts 16 bytes after
// the window of ox-1 (stride 2 x 8 bytes), which is exactly the row pitch of a K-major NO-SWIZZLE wgmma core
// matrix (8 rows, 16 bytes apart).  So the im2col operand is never built: shared memory holds raw input rows
// (cut into 8 overlapping 192-byte pieces of 8 output columns each by one TMA box with overlapping strides) and
// the A descriptor (LBO = 16 B, SBO = 192 B) walks the windows in place.  Per output-row pair the CTA loads
// 10 input-row slots (15 KiB) instead of a 56 KiB im2col tile; K = 7 kernel rows x (8 px x 4 ch) = 224.
// Even/odd input rows sit in separate slot runs so that "+1 slot" = "+2 input rows" = the second output row
// (rows 64..127 of the M = 128 tile, the second MMA warpgroup).
//
// The epilogue writes the conv tile (2 output rows x 64 columns x 64 ch, fp16) to a triple-buffered smem tile and
// pools it together with the last row of the previous tile; only the pooled tensor goes to HBM.  A CTA walks a
// contiguous range of row pairs; a range that starts inside an image first recomputes the row pair above it.
// =======================================================================================
static constexpr int S3_THREADS = 512;                 // TMA warpgroup, 2 MMA + epilogue warpgroups, 4 pool warps
static constexpr int S3_STAGES = 4;
static constexpr int S3_PIECE = 256;                   // bytes: 8 windows (stride 2 px) of 8 px need 176; 256 keeps core matrices 128 B-aligned
static constexpr int S3_SLOT = 8 * S3_PIECE;           // one input row cut into 8 pieces
static constexpr int S3_STAGE_BYTES = 10 * S3_SLOT;    // 5 even + 5 odd input rows
static constexpr int S3_W_BYTES = 28 * 64 * 16;        // [k chunk of 8][cout][8] fp16
static constexpr int S3_TILE_BYTES = 128 * 128;        // conv tile, one 128-byte line per pixel
static constexpr int S3_WP = 136;                      // padded input row, pixels
static constexpr size_t S3_SMEM = 1024 + S3_STAGES * S3_STAGE_BYTES + S3_W_BYTES + 3 * S3_TILE_BYTES + 256 + 256;

struct Stem3Params {
  CUtensorMap x_map;  // 5-D overlapping view of the packed input: {96 el, 8 pieces, row pair, parity, image}
  const __half* w;    // packed weights [28][64][8]
  const float* bias;
  __half* out;        // pooled NHWC fp16 [n][hp][wp][64]
  int n_img, hp, wp, Wo, relu;
};

// NCHW fp32 -> zero-bordered NHWC4 fp16; block = 64 x 4 threads, a thread converts two adjacent pixels of one row
__global__ void __launch_bounds__(256) stem_pack_input_kernel(const float* __restrict__ x, int N, int H, int W,
                                                              __half* __restrict__ xp) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x * 4 + (threadIdx.x >> 6);  // n * H + y
  const int xw = 2 * (threadIdx.x & 63);
  if (row >= N * H || xw >= W) return;
  const int n = row / H, y = row - n * H;
  const size_t plane = (size_t)H * W;
  const float* src = x + (size_t)n * 3 * plane + (size_t)y * W + xw;
  const float2 c0 = *reinterpret_cast<const float2*>(src);
  const float2 c1 = *reinterpret_cast<const float2*>(src + plane);
  const float2 c2 = *reinterpret_cast<const float2*>(src + 2 * plane);
  const __half2 a0 = __floats2half2_rn(c0.x, c1.x), b0 = __floats2half2_rn(c2.x, 0.f);
  const __half2 a1 = __floats2half2_rn(c0.y, c1.y), b1 = __floats2half2_rn(c2.y, 0.f);
  uint2* dst = reinterpret_cast<uint2*>(xp + (((size_t)n * (H + 6) + y + 3) * S3_WP + xw + 3) * 4);
  dst[0] = make_uint2(*reinterpret_cast<const uint32_t*>(&a0), *reinterpret_cast<const uint32_t*>(&b0));
  dst[1] = make_uint2(*reinterpret_cast<const uint32_t*>(&a1), *reinterpret_cast<const uint32_t*>(&b1));
}

// The same packed layout straight from uint8 HWC crops: ToTensor + Normalize (datasets/transforms/build.py:29-33) folded
// into the pack -- (u / 255 - mean) / std in IEEE fp32 (the arithmetic of augment_kernel, so the fp16 operand is
// bit-identical to normalize_batch followed by stem_pack_input_kernel) without the fp32 NCHW tensor in between
// (3 B read per pixel instead of 12 B written + 12 B read).
__global__ void __launch_bounds__(256) stem_pack_input_u8_kernel(const uint8_t* __restrict__ x, int N, int H, int W, float m0,
                                                                 float m1, float m2, float s0, float s1, float s2,
                                                                 __half* __restrict__ xp) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x * 4 + (threadIdx.x >> 6);  // n * H + y
  const int xw = 2 * (threadIdx.x & 63);
  if (row >= N * H || xw >= W) return;
  const int n = row / H, y = row - n * H;
  const uint16_t* src = reinterpret_cast<const uint16_t*>(x + ((size_t)row * W + xw) * 3);  // 6 bytes, 2-byte aligned
  const uint32_t w0 = src[0], w1 = src[1], w2 = src[2];  // r0 g0 | b0 r1 | g1 b1
  const float r0 = (float)(w0 & 255u) / 255.f, g0 = (float)(w0 >> 8) / 255.f, b0 = (float)(w1 & 255u) / 255.f;
  const float r1 = (float)(w1 >> 8) / 255.f, g1 = (float)(w2 & 255u) / 255.f, b1 = (float)(w2 >> 8) / 255.f;
  const __half2 a0 = __floats2half2_rn((r0 - m0) / s0, (g0 - m1) / s1), c0 = __floats2half2_rn((b0 - m2) / s2, 0.f);
  const __half2 a1 = __floats2half2_rn((r1 - m0) / s0, (g1 - m1) / s1), c1 = __floats2half2_rn((b1 - m2) / s2, 0.f);
  uint2* dst = reinterpret_cast<uint2*>(xp + (((size_t)n * (H + 6) + y + 3) * S3_WP + xw + 3) * 4);
  dst[0] = make_uint2(*reinterpret_cast<const uint32_t*>(&a0), *reinterpret_cast<const uint32_t*>(&c0));
  dst[1] = make_uint2(*reinterpret_cast<const uint32_t*>(&a1), *reinterpret_cast<const uint32_t*>(&c1));
}

__global__ void __launch_bounds__(S3_THREADS, 1) stem_pool_kernel(const __grid_constant__ Stem3Params p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t sA = base, sW = sA + S3_STAGES * S3_STAGE_BYTES, sT = sW + S3_W_BYTES;
  uint8_t* tile_g = gbase + (sT - base);
  float* bias_s = reinterpret_cast<float*>(gbase + (sT - base) + 3 * S3_TILE_BYTES);
  const uint32_t bars = sT + 3 * S3_TILE_BYTES + 256;
  const uint32_t bar_w = bars;
  auto full_bar = [&](int s) { return bars + 8u * (1 + s); };
  auto empty_bar = [&](int s) { return bars + 8u * (1 + S3_STAGES + s); };
  auto sfull_bar = [&](int s) { return bars + 8u * (1 + 2 * S3_STAGES + s); };   // conv tile written (8 warps)
  auto sempty_bar = [&](int s) { return bars + 8u * (4 + 2 * S3_STAGES + s); };  // conv tile no longer needed (4 warps)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid < 64) bias_s[tid] = p.bias[tid];
  if (tid == 0) {
    mbar_init(bar_w, 1);
    for (int s = 0; s < S3_STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);  // one arrive per MMA warpgroup
    }
    for (int s = 0; s < 3; ++s) {
      mbar_init(sfull_bar(s), 8);
      mbar_init(sempty_bar(s), 4);
    }
    fence_barrier_init();
    tma_prefetch_desc(&p.x_map);
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  // contiguous, balanced range of row pairs; a range that starts inside an image recomputes the pair above it
  const int num_tiles = p.n_img * p.hp;
  const int per = num_tiles / (int)gridDim.x, rem = num_tiles - per * (int)gridDim.x;
  const int t_begin = (int)blockIdx.x * per + min((int)blockIdx.x, rem);
  const int t_end = t_begin + per + ((int)blockIdx.x < rem ? 1 : 0);
  const int t_first = (t_begin < t_end && (t_begin % p.hp) != 0) ? t_begin - 1 : t_begin;

  if (warp < 4) {
    if (tid == 0) {
      mbar_arrive_expect_tx(bar_w, S3_W_BYTES);
      bulk_copy_g2s(sW, p.w, S3_W_BYTES, bar_w);
      int stage = 0;
      uint32_t phase = 0;
      for (int t = t_first; t < t_end; ++t) {
        const int n = t / p.hp, py = t - n * p.hp;
        mbar_wait(empty_bar(stage), phase ^ 1u);
        const uint32_t dst = sA + stage * S3_STAGE_BYTES;
        mbar_arrive_expect_tx(full_bar(stage), S3_STAGE_BYTES);
        tma_load_5d(dst, &p.x_map, full_bar(stage), 0, 0, 2 * py, 0, n);                   // padded rows 4py, +2, .., +8
        tma_load_5d(dst + 5 * S3_SLOT, &p.x_map, full_bar(stage), 0, 0, 2 * py, 1, n);     // padded rows 4py+1, .., +9
        if (++stage == S3_STAGES) {
          stage = 0;
          phase ^= 1u;
        }
      }
    }
  } else if (warp < 12) {
    // ---- MMA warpgroups: wg computes output row wg of the pair (tile rows [64 wg, 64 wg + 64)), then
    // +bias (+ReLU) -> fp16 -> conv tile in shared memory (ring of 3) ----
    const int wg = (tid >> 7) - 1;
    const int row0 = 64 * wg + 16 * (warp & 3);
    mbar_wait(bar_w, 0);
    float acc[32];
    int stage = 0, buf = 0;
    uint32_t phase = 0, bphase = 0;
    for (int t = t_first; t < t_end; ++t) {
      mbar_wait(full_bar(stage), phase);
      // output row 1 reads its kernel rows one slot (= two input rows) further
      const uint32_t a0 = sA + stage * S3_STAGE_BYTES + wg * S3_SLOT;
      wgmma_fence();
#pragma unroll
      for (int r = 0; r < 7; ++r) {
        // kernel row r of output row 0 = padded input row 4py + r: slot r/2 of the even or odd run
        const uint32_t arow = a0 + ((r & 1) * 5 + (r >> 1)) * S3_SLOT;
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
          const uint64_t da = make_noswizzle_kmajor_desc(arow + 32 * kk, 16, S3_PIECE);
          const uint64_t db = make_noswizzle_kmajor_desc(sW + (r * 4 + 2 * kk) * 1024, 1024, 128);
          wgmma_f16<64>(acc, da, db, (r > 0 || kk > 0) ? 1u : 0u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      if ((tid & 127) == 0) mbar_arrive(empty_bar(stage));
      if (++stage == S3_STAGES) {
        stage = 0;
        phase ^= 1u;
      }
      mbar_wait(sempty_bar(buf), bphase ^ 1u);  // the pool warps are done with the tile that lived here
      store_subtile_f16(acc, tile_g + buf * S3_TILE_BYTES, row0, bias_s, 0, p.relu, 0);
      __syncwarp();
      if (lane == 0) mbar_arrive(sfull_bar(buf));
      if (++buf == 3) {
        buf = 0;
        bphase ^= 1u;
      }
    }
  } else {
    // ---- pool warps: 3x3/2 max over the conv tile and the last row of the previous one -> HBM ----
    const int pt = tid - 384;  // 0..127
    int buf = 0;
    uint32_t bphase = 0;
    for (int t = t_first; t < t_end; ++t) {
      const int n = t / p.hp, py = t - n * p.hp;
      mbar_wait(sfull_bar(buf), bphase);
      const int pbuf = buf == 0 ? 2 : buf - 1;
      if (t >= t_begin) {
        const uint8_t* tl = tile_g + buf * S3_TILE_BYTES;
        const uint8_t* prev = tile_g + pbuf * S3_TILE_BYTES;
        // Out-of-range taps are replaced by an in-window duplicate (max is idempotent): all 9 loads of an output are
        // unconditional and issued back to back (one shared-memory round trip, not nine).
        const uint8_t* rows[3] = {py == 0 ? tl : prev + 64 * 128, tl, tl + 64 * 128};
#pragma unroll
        for (int it = 0; it < 2; ++it) {
          const int item = pt + it * 128;
          const int ppx = min(item >> 3, p.wp - 1), pch = item & 7;  // pooled column, 8-channel chunk
          const int cxs[3] = {max(2 * ppx - 1, 0), 2 * ppx, min(2 * ppx + 1, p.Wo - 1)};
          uint4 v[9];
#pragma unroll
          for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx)
              v[dy * 3 + dx] = *reinterpret_cast<const uint4*>(rows[dy] + cxs[dx] * 128 + ((pch ^ (cxs[dx] & 7)) << 4));
          uint4 m = v[0];
          __half2* mm = reinterpret_cast<__half2*>(&m);
#pragma unroll
          for (int q = 1; q < 9; ++q) {
            const __half2* vv = reinterpret_cast<const __half2*>(&v[q]);
#pragma unroll
            for (int e = 0; e < 4; ++e) mm[e] = __hmax2(mm[e], vv[e]);
          }
          if ((item >> 3) < p.wp)
            *reinterpret_cast<uint4*>(p.out + (((size_t)n * p.hp + py) * p.wp + ppx) * 64 + pch * 8) = m;
        }
      }
      __syncwarp();
      if (lane == 0 && t > t_first) mbar_arrive(sempty_bar(pbuf));  // the previous tile is no longer needed
      if (++buf == 3) {
        buf = 0;
        bphase ^= 1u;
      }
    }
  }
}

// maxpool 3x3 / 2, pad 1, NHWC fp16; one thread = 8 channels of one output pixel.  Every window has an in-bounds tap,
// so starting from -inf returns -inf only for a window of -inf inputs, as F.max_pool2d does.
__global__ void __launch_bounds__(256) maxpool3x3s2_kernel(const __half* __restrict__ x, int N, int H, int W, int C,
                                                           __half* __restrict__ out, int Ho, int Wo) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int cv = C / 8;
  const size_t total = (size_t)N * Ho * Wo * cv;
  if (i >= total) return;
  const int c8 = (int)(i % cv);
  size_t t = i / cv;
  const int ow = (int)(t % Wo);
  t /= Wo;
  const int oh = (int)(t % Ho);
  const int n = (int)(t / Ho);
  __half2 m[4];
  const __half2 neg = __float2half2_rn(-INFINITY);
#pragma unroll
  for (int j = 0; j < 4; ++j) m[j] = neg;
  for (int r = 0; r < 3; ++r) {
    const int ih = 2 * oh - 1 + r;
    if (ih < 0 || ih >= H) continue;
    for (int s = 0; s < 3; ++s) {
      const int iw = 2 * ow - 1 + s;
      if (iw < 0 || iw >= W) continue;
      const uint4 v = *reinterpret_cast<const uint4*>(x + (((size_t)n * H + ih) * W + iw) * C + c8 * 8);
      const __half2* hv = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) m[j] = __hmax2(m[j], hv[j]);
    }
  }
  uint4 o;
  __half2* po = reinterpret_cast<__half2*>(&o);
#pragma unroll
  for (int j = 0; j < 4; ++j) po[j] = m[j];
  *reinterpret_cast<uint4*>(out + (((size_t)n * Ho + oh) * Wo + ow) * C + c8 * 8) = o;
}

// global average pool over H*W (fp32 accumulate, pixel order) + optional eval BatchNorm1d
// (modelling/baseline.py:93-94, modelling/bases.py:175): one thread = 2 channels of one image
__global__ void __launch_bounds__(256) gap_bn_kernel(const __half* __restrict__ x, int HW, int C,
                                                     const float* __restrict__ bn_scale /*gamma/sqrt(var+eps)*/,
                                                     const float* __restrict__ bn_shift, float* __restrict__ feat,
                                                     float* __restrict__ emb) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.y;
  const int c2 = blockIdx.x * blockDim.x + threadIdx.x;
  if (c2 * 2 >= C) return;
  const __half2* base = reinterpret_cast<const __half2*>(x + (size_t)n * HW * C) + c2;
  float s0 = 0.f, s1 = 0.f;
  for (int p = 0; p < HW; ++p) {
    const float2 v = __half22float2(base[(size_t)p * (C / 2)]);
    s0 += v.x;
    s1 += v.y;
  }
  const float inv = 1.f / (float)HW;
  const float f0 = s0 * inv, f1 = s1 * inv;
  if (feat) {
    feat[(size_t)n * C + 2 * c2] = f0;
    feat[(size_t)n * C + 2 * c2 + 1] = f1;
  }
  if (emb) {
    emb[(size_t)n * C + 2 * c2] = __fmaf_rn(f0, bn_scale[2 * c2], bn_shift[2 * c2]);
    emb[(size_t)n * C + 2 * c2 + 1] = __fmaf_rn(f1, bn_scale[2 * c2 + 1], bn_shift[2 * c2 + 1]);
  }
}

// ---------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------
template <int BN, int N2 = 0>
static int launch_conv(const ConvKernelParams& p, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    CTL_CUDA(cudaFuncSetAttribute(conv_gemm_kernel<BN, N2>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)ConvCfg<BN>::SMEM));
    attr_set = true;
  }
  const long long units = N2 > 0 ? (long long)p.m_tiles : (long long)p.m_tiles * p.n_tiles;
  const int grid = (int)std::min<long long>(units, sm_count());
  CTL_CUDA(launch_k(conv_gemm_kernel<BN, N2>, dim3(grid), dim3(CONV_THREADS), ConvCfg<BN>::SMEM, st, p));
  CTL_LAUNCH_CHECK();
  return 0;
}

// Whether the 1x1 convolution cout -> cout2 that reads a launch's output can be chained into that launch
// (conv_gemm_kernel<128, cout2>).  The kernel's 168 registers per thread (384 threads, one CTA per SM) hold GEMM1's
// 64 accumulators of a 128-wide n-tile plus GEMM2's cout2 / 2 (a 256-wide n-tile's 128 plus 32 already spill); at most
// four n-tiles per m-tile keep the m-tiles (the unit a CTA owns) numerous enough to balance.
static bool chain_fits(int cout, int cout2) {
  return cout % 128 == 0 && cout <= 512 && (cout2 == 64 || cout2 == 128);
}

// The next 1x1 convolution of a chained launch (ctl_conv1x1_chain_nhwc_f16).
struct ChainNext {
  const void* weight;  // [cout2][cout] fp16
  const float* bias;
  void* out;
  int cout2, relu_from;
};

template <bool RES>
static int launch_c64_kernel(const C64Params& p, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    CTL_CUDA(cudaFuncSetAttribute(conv3x3_c64_kernel<RES>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)C64Cfg<RES>::SMEM));
    attr_set = true;
  }
  const long long tiles = (long long)p.n_img * p.tiles_h * p.tiles_w;
  const int grid = (int)std::min<long long>(tiles, sm_count());
  CTL_CUDA(launch_k(conv3x3_c64_kernel<RES>, dim3(grid), dim3(CONV_THREADS), C64Cfg<RES>::SMEM, st, p));
  CTL_LAUNCH_CHECK();
  return 0;
}

// residual (may be null): [n][h][w][64], added before the bias
static int launch_c64(const void* x, int n, int h, int w, const void* weight, const float* bias, const void* residual,
                      void* out, int relu, cudaStream_t st) {
  C64Params p = {};
  p.bias = bias;
  p.n_img = n;
  p.H = h;
  p.W = w;
  p.tiles_h = (h + 15) / 16;
  p.tiles_w = (w + 7) / 8;
  p.relu = relu;
  int rc;
  const uint64_t dims[4] = {64, (uint64_t)w, (uint64_t)h, (uint64_t)n};
  const uint64_t strd[4] = {2, 128, (uint64_t)w * 128, (uint64_t)h * w * 128};
  const uint32_t xbox[4] = {64, 16, 18, 1}, obox[4] = {64, 8, 16, 1};
  if ((rc = encode_tensor_map(&p.x_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, x, dims, strd, xbox, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = encode_tensor_map(&p.out_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, out, dims, strd, obox, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if (residual && (rc = encode_tensor_map(&p.res_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, residual, dims, strd, obox,
                                          CU_TENSOR_MAP_SWIZZLE_128B)))
    return rc;
  const uint64_t wd[2] = {576, 64}, ws[2] = {2, 576 * 2};
  const uint32_t wbox[2] = {64, 64};
  if ((rc = encode_tensor_map(&p.w_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 2, weight, wd, ws, wbox, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  return residual ? launch_c64_kernel<true>(p, st) : launch_c64_kernel<false>(p, st);
}

// Fills the tile geometry, the output / residual / weight maps and dispatches.  The caller has filled the A maps,
// the taps and k_blocks; `ktot` = row length of the weight matrix [Cout][ktot]; `next` (chain_fits(cout, cout2))
// chains the following 1x1 convolution into the launch.
static int finish_and_launch(ConvKernelParams& p, int n, int Ho, int Wo, int cout, int ktot, const void* weight,
                             const float* bias, const void* residual, void* out, int relu, int relu_from,
                             cudaStream_t st, const ChainNext* next = nullptr) {
  int rc;
  p.n_img = n;
  p.Ho = Ho;
  p.Wo = Wo;
  p.Cout = cout;
  p.bias = bias;
  p.has_residual = residual != nullptr;
  p.relu = relu;
  p.relu_from = relu_from;
  p.m_tiles = n * p.tiles_h * p.tiles_w;
  const int BN = next ? 128 : (cout % 256 == 0 ? 256 : (cout % 128 == 0 ? 128 : 64));
  p.n_tiles = cout / BN;
  {
    const uint64_t odims[4] = {(uint64_t)cout, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)n};
    const uint64_t ostr[4] = {2, (uint64_t)cout * 2, (uint64_t)Wo * cout * 2, (uint64_t)Ho * Wo * cout * 2};
    const uint32_t obox[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, 1};
    if ((rc = encode_tensor_map(&p.out_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, out, odims, ostr, obox,
                                CU_TENSOR_MAP_SWIZZLE_128B)))
      return rc;
    if ((rc = encode_tensor_map(&p.res_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, residual ? residual : out, odims,
                                ostr, obox, CU_TENSOR_MAP_SWIZZLE_128B)))
      return rc;
  }
  const uint64_t bdims[2] = {(uint64_t)ktot, (uint64_t)cout};
  const uint64_t bstr[2] = {2, (uint64_t)ktot * 2};
  const uint32_t bbox[2] = {CBK, (uint32_t)BN};
  if ((rc = encode_tensor_map(&p.b_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 2, weight, bdims, bstr, bbox,
                              CU_TENSOR_MAP_SWIZZLE_128B)))
    return rc;
  if (next) {
    const int c2 = next->cout2;
    const uint64_t odims[4] = {(uint64_t)c2, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)n};
    const uint64_t ostr[4] = {2, (uint64_t)c2 * 2, (uint64_t)Wo * c2 * 2, (uint64_t)Ho * Wo * c2 * 2};
    const uint32_t obox[4] = {64, (uint32_t)p.TW, (uint32_t)p.TH, 1};
    if ((rc = encode_tensor_map(&p.out2_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, next->out, odims, ostr, obox,
                                CU_TENSOR_MAP_SWIZZLE_128B)))
      return rc;
    const uint64_t wdims[2] = {(uint64_t)cout, (uint64_t)c2};
    const uint64_t wstr[2] = {2, (uint64_t)cout * 2};
    const uint32_t wbox[2] = {CBK, (uint32_t)c2};
    if ((rc = encode_tensor_map(&p.b2_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 2, next->weight, wdims, wstr, wbox,
                                CU_TENSOR_MAP_SWIZZLE_128B)))
      return rc;
    p.bias2 = next->bias;
    p.relu_from2 = next->relu_from;
    return c2 == 64 ? launch_conv<128, 64>(p, st) : launch_conv<128, 128>(p, st);
  }
  if (BN == 256) return launch_conv<256>(p, st);
  if (BN == 128) return launch_conv<128>(p, st);
  return launch_conv<64>(p, st);
}

// A tensor maps of one NHWC source [n, h, w, cin] read at `stride`: stride 1 -> map 0..3 identical; stride 2 -> the four
// parity views (view (ph, pw) holds input pixels (2i + ph, 2j + pw)), so every box is a dense stride-1 box.
static int encode_source(CUtensorMap* maps, int count, const void* x, int n, int h, int w, int cin, int stride, int TH,
                         int TW) {
  int rc;
  const __half* xb = static_cast<const __half*>(x);
  const uint32_t abox[4] = {CBK, (uint32_t)TW, (uint32_t)TH, 1};
  if (stride == 1) {
    const uint64_t dims[4] = {(uint64_t)cin, (uint64_t)w, (uint64_t)h, (uint64_t)n};
    const uint64_t strd[4] = {2, (uint64_t)cin * 2, (uint64_t)w * cin * 2, (uint64_t)h * w * cin * 2};
    for (int i = 0; i < count; ++i)
      if ((rc = encode_tensor_map(&maps[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, xb, dims, strd, abox,
                                  CU_TENSOR_MAP_SWIZZLE_128B)))
        return rc;
    return 0;
  }
  const uint64_t dims[4] = {(uint64_t)cin, (uint64_t)(w / 2), (uint64_t)(h / 2), (uint64_t)n};
  const uint64_t strd[4] = {2, (uint64_t)cin * 4, (uint64_t)w * cin * 4, (uint64_t)h * w * cin * 2};
  for (int v = 0; v < count; ++v) {
    const int ph = v >> 1, pw = v & 1;
    if ((rc = encode_tensor_map(&maps[v], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, xb + ((size_t)ph * w + pw) * cin, dims,
                                strd, abox, CU_TENSOR_MAP_SWIZZLE_128B)))
      return rc;
  }
  return 0;
}

// Tile geometry, A maps and taps of a k1 x k1 (1 or 3, pad k1 / 2, stride 1) convolution at the output resolution
// Ho x Wo = h2 / stride2 x w2 / stride2: x1 [n][Ho][Wo][cin1] alone, or K-concatenated with the 1x1 of
// x2 [n][h2][w2][cin2] read at stride2 (weight columns k1 * k1 * cin1 ..).
static int setup_dual(ConvKernelParams& p, int k1, const void* x1, int cin1, const void* x2, int h2, int w2, int cin2,
                      int stride2, int n) {
  int rc;
  const int Ho = h2 / stride2, Wo = w2 / stride2;
  pick_tile(Ho, Wo, &p.TH, &p.TW);
  p.tiles_h = (Ho + p.TH - 1) / p.TH;
  p.tiles_w = (Wo + p.TW - 1) / p.TW;
  // map 0: x1 at the output resolution; map 1: x2 (its (0, 0) parity view when strided); unused maps repeat map 0
  if ((rc = encode_source(&p.a_map[0], 1, x1, n, Ho, Wo, cin1, 1, p.TH, p.TW))) return rc;
  p.a_map[1] = p.a_map[0];
  if (x2 && (rc = encode_source(&p.a_map[1], 1, x2, n, h2, w2, cin2, stride2, p.TH, p.TW))) return rc;
  p.a_map[2] = p.a_map[0];
  p.a_map[3] = p.a_map[0];
  const int pad = k1 / 2;
  p.n_taps = 0;
  for (int r = 0; r < k1; ++r)
    for (int s = 0; s < k1; ++s) p.taps[p.n_taps++] = ConvTap{0, r - pad, s - pad, (r * k1 + s) * cin1, cin1 / 64};
  if (x2) {
    const ConvTap shortcut = {1, 0, 0, k1 * k1 * cin1, cin2 / 64};
    if (p.n_taps < 9)
      p.taps[p.n_taps] = shortcut;
    else
      p.tap9 = shortcut;
    ++p.n_taps;
  }
  p.k_blocks = (k1 * k1 * cin1 + (x2 ? cin2 : 0)) / 64;
  return 0;
}

}  // namespace ctl

using namespace ctl;

extern "C" {

int ctl_conv2d_nhwc_f16(const void* x, int32_t n, int32_t h, int32_t w, int32_t cin, const void* weight,
                        const float* bias, const void* residual, void* out, int32_t cout, int32_t ksize,
                        int32_t stride, int32_t relu, int32_t relu_from, ctl_stream_t stream) {
  CTL_CHECK_ARG(x && weight && bias && out, "null pointer");
  CTL_CHECK_ARG(n >= 1 && h >= 1 && w >= 1, "bad activation shape");
  CTL_CHECK_ARG(cin % 64 == 0 && cout % 64 == 0, "Cin=%d and Cout=%d must be multiples of 64", cin, cout);
  CTL_CHECK_ARG(cout <= 2048, "Cout=%d exceeds 2048 (bias staging)", cout);
  CTL_CHECK_ARG((ksize == 1 || ksize == 3) && (stride == 1 || stride == 2), "only 1x1 / 3x3, stride 1 / 2");
  CTL_CHECK_ARG(relu_from % 32 == 0, "relu_from=%d must be a multiple of 32", relu_from);
  CTL_CHECK_ARG(stride == 1 || (h % 2 == 0 && w % 2 == 0), "stride 2 needs even H, W (got %dx%d)", h, w);
  int rc = ctl_device_check();
  if (rc) return rc;
  const int pad = ksize == 3 ? 1 : 0;
  const int Ho = (h + 2 * pad - ksize) / stride + 1, Wo = (w + 2 * pad - ksize) / stride + 1;
  if (ksize == 3 && stride == 1 && cin == 64 && cout == 64 && relu_from == 0)
    return launch_c64(x, n, h, w, weight, bias, residual, out, relu, (cudaStream_t)stream);
  ConvKernelParams p = {};
  pick_tile(Ho, Wo, &p.TH, &p.TW);
  p.tiles_h = (Ho + p.TH - 1) / p.TH;
  p.tiles_w = (Wo + p.TW - 1) / p.TW;
  if ((rc = encode_source(p.a_map, 4, x, n, h, w, cin, stride, p.TH, p.TW))) return rc;
  p.n_taps = ksize * ksize;
  p.k_blocks = p.n_taps * (cin / 64);
  for (int r = 0; r < ksize; ++r)
    for (int s = 0; s < ksize; ++s) {
      if (stride == 1) {
        p.taps[r * ksize + s] = ConvTap{0, r - pad, s - pad, (r * ksize + s) * cin, cin / 64};
      } else {
        // input row 2*ho + r - pad = 2*(ho + dh) + ph
        const int ar = r - pad, as = s - pad;
        const int ph = ((ar % 2) + 2) % 2, pw = ((as % 2) + 2) % 2;
        const int dh = (ar - ph) / 2, dw = (as - pw) / 2;
        p.taps[r * ksize + s] = ConvTap{ph * 2 + pw, dh, dw, (r * ksize + s) * cin, cin / 64};
      }
    }
  return finish_and_launch(p, n, Ho, Wo, cout, ksize * ksize * cin, weight, bias, residual, out, relu, relu_from,
                           (cudaStream_t)stream);
}

int ctl_conv1x1_dual_nhwc_f16(const void* x1, int32_t cin1, const void* x2, int32_t h2, int32_t w2, int32_t cin2,
                              int32_t stride2, int32_t n, const void* weight_cat, const float* bias, void* out,
                              int32_t cout, int32_t relu, ctl_stream_t stream) {
  CTL_CHECK_ARG(x1 && x2 && weight_cat && bias && out, "null pointer");
  CTL_CHECK_ARG(n >= 1 && h2 >= 1 && w2 >= 1, "bad activation shape");
  CTL_CHECK_ARG(cin1 % 64 == 0 && cin2 % 64 == 0 && cout % 64 == 0 && cin1 >= 64 && cin2 >= 64,
                "Cin1=%d, Cin2=%d and Cout=%d must be multiples of 64", cin1, cin2, cout);
  CTL_CHECK_ARG(cout <= 2048, "Cout=%d exceeds 2048 (bias staging)", cout);
  CTL_CHECK_ARG(stride2 == 1 || (stride2 == 2 && h2 % 2 == 0 && w2 % 2 == 0), "stride2 must be 1, or 2 with even H2, W2");
  int rc = ctl_device_check();
  if (rc) return rc;
  ConvKernelParams p = {};
  if ((rc = setup_dual(p, 1, x1, cin1, x2, h2, w2, cin2, stride2, n))) return rc;
  return finish_and_launch(p, n, h2 / stride2, w2 / stride2, cout, cin1 + cin2, weight_cat, bias, nullptr, out, relu, 0,
                           (cudaStream_t)stream);
}

int ctl_conv3x3_dual_nhwc_f16(const void* x1, int32_t cin1, const void* x2, int32_t h2, int32_t w2, int32_t cin2,
                              int32_t stride2, int32_t n, const void* weight_cat, const float* bias, void* out,
                              int32_t cout, int32_t relu, ctl_stream_t stream) {
  CTL_CHECK_ARG(x1 && x2 && weight_cat && bias && out, "null pointer");
  CTL_CHECK_ARG(n >= 1 && h2 >= 1 && w2 >= 1, "bad activation shape");
  CTL_CHECK_ARG(cin1 % 64 == 0 && cin2 % 64 == 0 && cout % 64 == 0 && cin1 >= 64 && cin2 >= 64,
                "Cin1=%d, Cin2=%d and Cout=%d must be multiples of 64", cin1, cin2, cout);
  CTL_CHECK_ARG(cout <= 2048, "Cout=%d exceeds 2048 (bias staging)", cout);
  CTL_CHECK_ARG(stride2 == 1 || (stride2 == 2 && h2 % 2 == 0 && w2 % 2 == 0), "stride2 must be 1, or 2 with even H2, W2");
  int rc = ctl_device_check();
  if (rc) return rc;
  ConvKernelParams p = {};
  if ((rc = setup_dual(p, 3, x1, cin1, x2, h2, w2, cin2, stride2, n))) return rc;
  return finish_and_launch(p, n, h2 / stride2, w2 / stride2, cout, 9 * cin1 + cin2, weight_cat, bias, nullptr, out, relu, 0,
                           (cudaStream_t)stream);
}

int32_t ctl_conv1x1_chain_supported(int32_t cout, int32_t cout2) { return chain_fits(cout, cout2) ? 1 : 0; }

int ctl_conv1x1_chain_nhwc_f16(const void* x1, int32_t cin1, const void* x2, int32_t h2, int32_t w2, int32_t cin2,
                               int32_t stride2, int32_t n, const void* weight, const float* bias, const void* residual,
                               void* out, int32_t cout, const void* weight2, const float* bias2, int32_t cout2,
                               int32_t relu_from2, void* out2, ctl_stream_t stream) {
  CTL_CHECK_ARG(x1 && weight && bias && out && weight2 && bias2 && out2, "null pointer");
  CTL_CHECK_ARG(!(x2 && residual), "the K-concatenated form (x2) takes no residual");
  CTL_CHECK_ARG(n >= 1 && h2 >= 1 && w2 >= 1, "bad activation shape");
  CTL_CHECK_ARG(cin1 % 64 == 0 && cin1 >= 64 && (!x2 || (cin2 % 64 == 0 && cin2 >= 64)),
                "Cin1=%d and Cin2=%d must be multiples of 64", cin1, cin2);
  CTL_CHECK_ARG(chain_fits(cout, cout2), "Cout=%d -> Cout2=%d cannot be chained (see ctl_conv1x1_chain_supported)", cout,
                cout2);
  CTL_CHECK_ARG(relu_from2 % 32 == 0, "relu_from2=%d must be a multiple of 32", relu_from2);
  CTL_CHECK_ARG(x2 ? (stride2 == 1 || (stride2 == 2 && h2 % 2 == 0 && w2 % 2 == 0)) : stride2 == 1,
                "stride2 must be 1, or 2 with even H2, W2 and a second source");
  int rc = ctl_device_check();
  if (rc) return rc;
  ConvKernelParams p = {};
  if ((rc = setup_dual(p, 1, x1, cin1, x2, h2, w2, cin2, stride2, n))) return rc;
  const ChainNext next = {weight2, bias2, out2, cout2, relu_from2};
  return finish_and_launch(p, n, h2 / stride2, w2 / stride2, cout, cin1 + (x2 ? cin2 : 0), weight, bias, residual, out, 1,
                           0, (cudaStream_t)stream, &next);
}

int ctl_stem_conv7x7_tc(const float* x_nchw, int32_t n, int32_t h, int32_t w, const void* weight_k192_f16,
                        const float* bias, int32_t relu, void* out_nhwc_f16, ctl_stream_t stream) {
  CTL_CHECK_ARG(x_nchw && weight_k192_f16 && bias && out_nhwc_f16, "null pointer");
  CTL_CHECK_ARG(n >= 1 && h >= 7 && w >= 7, "bad input shape");
  int rc = ctl_device_check();
  if (rc) return rc;
  StemParams p = {};
  p.x = x_nchw;
  p.bias = bias;
  p.out = static_cast<__half*>(out_nhwc_f16);
  p.n_img = n;
  p.H = h;
  p.W = w;
  p.Ho = (h + 6 - 7) / 2 + 1;
  p.Wo = (w + 6 - 7) / 2 + 1;
  p.tiles_h = (p.Ho + S_TH - 1) / S_TH;
  p.tiles_w = (p.Wo + S_TW - 1) / S_TW;
  p.relu = relu;
  const uint64_t dims[2] = {SK, 64};
  const uint64_t strd[2] = {2, SK * 2};
  const uint32_t box[2] = {64, 64};
  if ((rc = encode_tensor_map(&p.w_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 2, weight_k192_f16, dims, strd, box,
                              CU_TENSOR_MAP_SWIZZLE_128B)))
    return rc;
  {
    const uint64_t odims[4] = {64, (uint64_t)p.Wo, (uint64_t)p.Ho, (uint64_t)n};
    const uint64_t ostr[4] = {2, 128, (uint64_t)p.Wo * 128, (uint64_t)p.Ho * p.Wo * 128};
    const uint32_t obox[4] = {64, S_TW, S_TH, 1};
    if ((rc = encode_tensor_map(&p.out_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, out_nhwc_f16, odims, ostr, obox,
                                CU_TENSOR_MAP_SWIZZLE_128B)))
      return rc;
  }
  static bool attr_set = false;
  if (!attr_set) {
    CTL_CUDA(cudaFuncSetAttribute(stem_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)STEM_TC_SMEM));
    attr_set = true;
  }
  const long long tiles = (long long)n * p.tiles_h * p.tiles_w;
  const int grid = (int)std::min<long long>(tiles, (long long)sm_count());
  CTL_CUDA(launch_k(stem_tc_kernel, dim3(grid), dim3(STEM_TC_THREADS), STEM_TC_SMEM, (cudaStream_t)stream, p));
  CTL_LAUNCH_CHECK();
  return 0;
}

size_t ctl_stem_pad_bytes(int32_t n, int32_t h, int32_t w) {
  (void)w;
  if (n < 1 || h < 1) return 0;
  return (size_t)n * (h + 6) * S3_WP * 4 * sizeof(__half) + 256;  // + slack: the last piece of a row is read 256 B wide
}

// the conv + pool kernel on an already packed input (shared by the fp32 and the uint8 entry points)
static int stem_pool_launch(int32_t n, int32_t h, int32_t w, void* xpad, const void* weight_packed_f16, const float* bias,
                            int32_t relu, void* out_pooled_nhwc_f16, cudaStream_t st) {
  int rc;
  Stem3Params p = {};
  p.w = static_cast<const __half*>(weight_packed_f16);
  p.bias = bias;
  p.out = static_cast<__half*>(out_pooled_nhwc_f16);
  p.n_img = n;
  const int Ho = h / 2;
  p.Wo = w / 2;
  p.hp = Ho / 2;
  p.wp = (p.Wo + 2 - 3) / 2 + 1;
  p.relu = relu;
  const uint64_t pitch = (uint64_t)S3_WP * 8, hp_rows = (uint64_t)h + 6;
  // overlapping view: piece g of a row starts 128 bytes (16 pixels) after piece g-1 and is 192 bytes long
  const uint64_t dims[5] = {(uint64_t)S3_WP * 4, 8, hp_rows / 2, 2, (uint64_t)n};
  const uint64_t strd[5] = {2, 128, 2 * pitch, pitch, hp_rows * pitch};
  const uint32_t box[5] = {S3_PIECE / 2, 8, 5, 1, 1};
  if ((rc = encode_tensor_map(&p.x_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 5, xpad, dims, strd, box, CU_TENSOR_MAP_SWIZZLE_NONE)))
    return rc;
  static bool attr_set = false;
  if (!attr_set) {
    CTL_CUDA(cudaFuncSetAttribute(stem_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S3_SMEM));
    attr_set = true;
  }
  const long long tiles = (long long)n * p.hp;
  const int grid = (int)std::min<long long>(tiles, (long long)sm_count());
  CTL_CUDA(launch_k(stem_pool_kernel, dim3(grid), dim3(S3_THREADS), S3_SMEM, st, p));
  return 0;
}

static int stem_fused_check(const void* x, int32_t n, int32_t h, int32_t w, const void* xpad, const void* wt, const float* bias,
                            const void* out) {
  CTL_CHECK_ARG(x && xpad && wt && bias && out, "null pointer");
  CTL_CHECK_ARG(n >= 1 && h >= 8 && w >= 8 && h % 4 == 0 && w % 2 == 0 && w <= 128,
                "the fused stem needs h % 4 == 0, even w <= 128 (use ctl_stem_conv7x7_tc + ctl_maxpool3x3s2_nhwc_f16)");
  return ctl_device_check();
}

int ctl_stem_pool_fused(const float* x_nchw, int32_t n, int32_t h, int32_t w, void* xpad, const void* weight_packed_f16,
                        const float* bias, int32_t relu, void* out_pooled_nhwc_f16, ctl_stream_t stream) {
  int rc = stem_fused_check(x_nchw, n, h, w, xpad, weight_packed_f16, bias, out_pooled_nhwc_f16);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  CTL_CUDA(launch_k(stem_pack_input_kernel, dim3((unsigned)(((size_t)n * h + 3) / 4)), dim3(256), 0, st, x_nchw, (int)n, (int)h,
                    (int)w, static_cast<__half*>(xpad)));
  return stem_pool_launch(n, h, w, xpad, weight_packed_f16, bias, relu, out_pooled_nhwc_f16, st);
}

int ctl_stem_pool_fused_u8(const void* x_u8_nhwc, int32_t n, int32_t h, int32_t w, const float* mean3_host, const float* std3_host,
                           void* xpad, const void* weight_packed_f16, const float* bias, int32_t relu, void* out_pooled_nhwc_f16,
                           ctl_stream_t stream) {
  CTL_CHECK_ARG(mean3_host && std3_host, "null pointer");
  CTL_CHECK_ARG(std3_host[0] > 0 && std3_host[1] > 0 && std3_host[2] > 0, "std must be positive");
  int rc = stem_fused_check(x_u8_nhwc, n, h, w, xpad, weight_packed_f16, bias, out_pooled_nhwc_f16);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  CTL_CUDA(launch_k(stem_pack_input_u8_kernel, dim3((unsigned)(((size_t)n * h + 3) / 4)), dim3(256), 0, st,
                    static_cast<const uint8_t*>(x_u8_nhwc), (int)n, (int)h, (int)w, mean3_host[0], mean3_host[1], mean3_host[2],
                    std3_host[0], std3_host[1], std3_host[2], static_cast<__half*>(xpad)));
  return stem_pool_launch(n, h, w, xpad, weight_packed_f16, bias, relu, out_pooled_nhwc_f16, st);
}

int ctl_maxpool3x3s2_nhwc_f16(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, void* out,
                              ctl_stream_t stream) {
  CTL_CHECK_ARG(x && out && c % 8 == 0, "bad arguments");
  int rc = ctl_device_check();
  if (rc) return rc;
  const int Ho = (h + 2 - 3) / 2 + 1, Wo = (w + 2 - 3) / 2 + 1;
  const size_t total = (size_t)n * Ho * Wo * (c / 8);
  CTL_CUDA(launch_k(maxpool3x3s2_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, (cudaStream_t)stream,
                    static_cast<const __half*>(x), (int)n, (int)h, (int)w, (int)c, static_cast<__half*>(out), Ho, Wo));
  CTL_LAUNCH_CHECK();
  return 0;
}

int ctl_gap_bn_nhwc_f16(const void* x, int32_t n, int32_t hw, int32_t c, const float* bn_scale, const float* bn_shift,
                        float* feat, float* emb, ctl_stream_t stream) {
  CTL_CHECK_ARG(x && (feat || emb) && c % 2 == 0, "bad arguments");
  CTL_CHECK_ARG(emb == nullptr || (bn_scale && bn_shift), "emb needs the folded BatchNorm1d scale/shift");
  int rc = ctl_device_check();
  if (rc) return rc;
  dim3 grid((c / 2 + 255) / 256, n);
  CTL_CUDA(launch_k(gap_bn_kernel, grid, dim3(256), 0, (cudaStream_t)stream, static_cast<const __half*>(x), (int)hw, (int)c,
                    bn_scale, bn_shift, feat, emb));
  CTL_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
