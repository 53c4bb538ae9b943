// Ranked-result grids of utils/visrank.py (visualize_ranked_results, :161-236) on the device: OpenCV's
// cv2.resize(img, (w, h)) with INTER_LINEAR on 8UC3 images, bit for bit, the bordered second resize of every grid cell,
// the grid composition, and the per-query ranked list without junk entries.
//
// cv2's INTER_LINEAR is not PIL's BILINEAR (resize.cu): it always blends 2 taps per axis, with 11-bit fixed-point
// weights.  Per axis (`in` -> `out` pixels), o the output index:
//   f = (float)((o + 0.5) * (in / out) - 0.5)   (double arithmetic, one rounding per operation, then float)
//   s = floor(f), f -= s (float), a0 = rint((float)(1 - f) * 2048), a1 = 2048 - a0 (rint: half to even)
// Along x (only) the weights are clamped: s < 0 -> s = 0, f = 0; s >= in - 1 -> s = in - 1, f = 0.  Along y the
// weights are kept and the two source rows are clamped to [0, in - 1].  Then, per channel (all integers >= 0):
//   hrow(y) = S[y][s] * a0 + S[y][min(s + 1, in - 1)] * a1
//   out = min((((b0 * (hrow(y0) >> 4)) >> 16) + ((b1 * (hrow(y1) >> 4)) >> 16) + 2) >> 2, 255)
#include <stdint.h>

#include <algorithm>

#include "common.h"

namespace ctl {

constexpr int VR_THREADS = 256;
constexpr long long VR_MAX_SIDE = 1 << 24;

struct LinTap {
  int i0, i1, w0, w1;  // source indices and weights (w0 + w1 = 2048)
};

__device__ __forceinline__ LinTap lin_tap(int o, int in, int out, bool clamp_weights) {
  const double scale = __ddiv_rn((double)in, (double)out);
  float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)o, 0.5), scale), 0.5));
  int s = __float2int_rd(f);
  f = __fsub_rn(f, (float)s);
  if (clamp_weights) {
    if (s < 0) s = 0, f = 0.f;
    if (s >= in - 1) s = in - 1, f = 0.f;
  }
  LinTap t;
  t.w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  t.w1 = 2048 - t.w0;
  t.i0 = min(max(s, 0), in - 1);
  t.i1 = min(max(s + 1, 0), in - 1);
  return t;
}

__device__ __forceinline__ uint8_t lin_out(int b0, int h0, int b1, int h1) {
  return (uint8_t)min((((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2, 255);
}

// one output pixel of a W x H source whose pixel (y, x) channel c is px(y, x, c)
template <typename Px>
__device__ __forceinline__ void lin_pixel(const Px& px, int H, int W, int h, int w, int y, int x, uint8_t* d) {
  const LinTap tx = lin_tap(x, W, w, true), ty = lin_tap(y, H, h, false);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int h0 = px(ty.i0, tx.i0, c) * tx.w0 + px(ty.i0, tx.i1, c) * tx.w1;
    const int h1 = px(ty.i1, tx.i0, c) * tx.w0 + px(ty.i1, tx.i1, c) * tx.w1;
    d[c] = lin_out(ty.w0, h0, ty.w1, h1);
  }
}

// 0: a real image inside src_bytes; 1: a mock row (zeros); 2: an entry that does not fit
__device__ __forceinline__ int vr_entry_kind(const ctl_resize_entry& e, long long src_bytes) {
  if (e.h < 0 || e.w < 0 || e.h > VR_MAX_SIDE || e.w > VR_MAX_SIDE) return 2;
  if (e.h == 0 || e.w == 0) return 1;
  if (e.offset < 0 || e.offset > src_bytes || e.h * e.w * 3 > src_bytes - e.offset) return 2;
  return 0;
}

// one CTA row per image; every thread of it writes pixels of that image
__global__ void __launch_bounds__(VR_THREADS) resize_linear_cv_kernel(const uint8_t* __restrict__ src, long long src_bytes,
                                                                     const ctl_resize_entry* __restrict__ table, int out_h,
                                                                     int out_w, uint8_t* __restrict__ out,
                                                                     int* __restrict__ status) {
  const int b = blockIdx.x;
  const ctl_resize_entry e = table[b];
  const int kind = vr_entry_kind(e, src_bytes);
  if (blockIdx.y == 0 && threadIdx.x == 0) status[b] = kind == 2 ? 1 : 0;
  const long long units = (long long)out_h * out_w;
  uint8_t* img = out + (size_t)b * units * 3;
  const int H = (int)e.h, W = (int)e.w;
  const uint8_t* s = src + (kind == 0 ? e.offset : 0);
  auto px = [&](int y, int x, int c) -> int { return s[((size_t)y * W + x) * 3 + c]; };
  for (long long u = (long long)blockIdx.y * blockDim.x + threadIdx.x; u < units; u += (long long)gridDim.y * blockDim.x) {
    uint8_t* d = img + u * 3;
    if (kind != 0) {
      d[0] = d[1] = d[2] = 0;
      continue;
    }
    lin_pixel(px, H, W, out_h, out_w, (int)(u / out_w), (int)(u % out_w), d);
  }
}

constexpr int VR_BW = 3;           // border width, visrank.py:18
constexpr int VR_SPACING = 2;      // GRID_SPACING, visrank.py:16
constexpr int VR_QUERY_EXTRA = 8;  // QUERY_EXTRA_SPACING, visrank.py:17

// one CTA row per cell: cv2.resize(copyMakeBorder(cell image, 3, 3, 3, 3, colour), (w, h)) into its grid slot, the
// bordered (h + 6) x (w + 6) source read on the fly from the resized batch
__global__ void __launch_bounds__(VR_THREADS) visrank_compose_kernel(const uint8_t* __restrict__ resized, long long n_rows,
                                                                    int h, int w, const int32_t* __restrict__ cells,
                                                                    int n_grids, int topk, uint8_t* __restrict__ out,
                                                                    int* __restrict__ status) {
  const int4 cell = reinterpret_cast<const int4*>(cells)[blockIdx.x];
  const int row = cell.x, grid = cell.y, col = cell.z;
  if (row < 0 || row >= n_rows || grid < 0 || grid >= n_grids || col < 0 || col > topk) {
    if (blockIdx.y == 0 && threadIdx.x == 0) atomicOr(status, 1);
    return;
  }
  const uint8_t colour[3] = {(uint8_t)(cell.w >> 16), (uint8_t)(cell.w >> 8), (uint8_t)cell.w};
  const uint8_t* img = resized + (size_t)row * h * w * 3;
  auto px = [&](int y, int x, int c) -> int {
    const int yy = y - VR_BW, xx = x - VR_BW;
    return (yy >= 0 && yy < h && xx >= 0 && xx < w) ? img[((size_t)yy * w + xx) * 3 + c] : colour[c];
  };
  const long long gw = (long long)(topk + 1) * w + (long long)topk * VR_SPACING + VR_QUERY_EXTRA;
  const long long x0 = col == 0 ? 0 : (long long)col * w + (long long)col * VR_SPACING + VR_QUERY_EXTRA;
  uint8_t* dst = out + (size_t)grid * h * gw * 3;
  const long long units = (long long)h * w;
  for (long long u = (long long)blockIdx.y * blockDim.x + threadIdx.x; u < units; u += (long long)gridDim.y * blockDim.x) {
    const int y = (int)(u / w), x = (int)(u % w);
    lin_pixel(px, h + 2 * VR_BW, w + 2 * VR_BW, h, w, y, x, dst + ((size_t)y * gw + x0 + x) * 3);
  }
}

// one thread per query: the first topk non-junk entries of its ascending top-k list
__global__ void visrank_select_kernel(const int64_t* __restrict__ topk_idx, long long nq, int k, const int32_t* __restrict__ q_pid,
                                      const int32_t* __restrict__ q_cam, const int32_t* __restrict__ g_pid,
                                      const uint64_t* __restrict__ g_cammask, long long ng, int topk,
                                      int64_t* __restrict__ out_idx, int8_t* __restrict__ out_matched,
                                      int* __restrict__ status) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  const int qp = q_pid[q], qc = q_cam[q];
  int r = 0;
  for (int j = 0; j < k && r < topk; ++j) {
    const int64_t g = topk_idx[q * k + j];
    if (g < 0 || g >= ng) {
      atomicOr(status, 1);
      break;
    }
    const bool same = g_pid[g] == qp;
    if (same && ((g_cammask[g] >> qc) & 1ull)) continue;  // junk: same identity seen by the query's camera
    out_idx[q * topk + r] = g;
    out_matched[q * topk + r] = same ? 1 : 0;
    ++r;
  }
  for (; r < topk; ++r) {
    out_idx[q * topk + r] = -1;
    out_matched[q * topk + r] = 0;
  }
}

static unsigned vr_grid_y(long long units) {
  return (unsigned)std::min<long long>(std::max<long long>((units + VR_THREADS - 1) / VR_THREADS, 1), 65535);
}

static bool vr_size_ok(int32_t h, int32_t w) { return h >= 1 && w >= 1 && h <= 16384 && w <= 16384; }

}  // namespace ctl

using namespace ctl;

extern "C" {

int ctl_resize_linear_cv_u8(const void* src, int64_t src_bytes, const void* table_device, int64_t n, int32_t out_h,
                            int32_t out_w, void* out_u8_nhwc, int32_t* status, ctl_stream_t stream) {
  CTL_CHECK_ARG(src && table_device && out_u8_nhwc && status, "null pointer");
  CTL_CHECK_ARG(n >= 1 && n <= INT32_MAX, "n = %lld: expected 1 <= n < 2^31", (long long)n);
  CTL_CHECK_ARG(vr_size_ok(out_h, out_w), "output size %d x %d: expected 1..16384 on each side", out_h, out_w);
  CTL_CHECK_ARG(src_bytes >= 0, "src_bytes < 0");
  int rc = ctl_device_check();
  if (rc) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  resize_linear_cv_kernel<<<dim3((unsigned)n, vr_grid_y((long long)out_h * out_w)), VR_THREADS, 0, st>>>(
      static_cast<const uint8_t*>(src), (long long)src_bytes, static_cast<const ctl_resize_entry*>(table_device), out_h,
      out_w, static_cast<uint8_t*>(out_u8_nhwc), reinterpret_cast<int*>(status));
  CTL_LAUNCH_CHECK();
  return 0;
}

int ctl_visrank_compose(const void* resized_u8, int64_t n_rows, int32_t h, int32_t w, const int32_t* cells_device,
                        int64_t n_cells, int64_t n_grids, int32_t topk, void* out_u8, int32_t* status,
                        ctl_stream_t stream) {
  CTL_CHECK_ARG(resized_u8 && out_u8 && status && (cells_device || n_cells == 0), "null pointer");
  CTL_CHECK_ARG(vr_size_ok(h, w), "cell size %d x %d: expected 1..16384 on each side", h, w);
  CTL_CHECK_ARG(topk >= 1 && topk <= 1024, "topk = %d: expected 1..1024", topk);
  CTL_CHECK_ARG(n_rows >= 1 && n_grids >= 1 && n_grids <= INT32_MAX && n_cells >= 0 && n_cells <= INT32_MAX,
                "n_rows = %lld, n_grids = %lld, n_cells = %lld", (long long)n_rows, (long long)n_grids,
                (long long)n_cells);
  int rc = ctl_device_check();
  if (rc) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  const size_t gw = (size_t)(topk + 1) * w + (size_t)topk * VR_SPACING + VR_QUERY_EXTRA;
  CTL_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
  CTL_CUDA(cudaMemsetAsync(out_u8, 255, (size_t)n_grids * h * gw * 3, st));  // visrank.py:176: a white grid
  if (n_cells == 0) return 0;
  visrank_compose_kernel<<<dim3((unsigned)n_cells, vr_grid_y((long long)h * w)), VR_THREADS, 0, st>>>(
      static_cast<const uint8_t*>(resized_u8), (long long)n_rows, h, w, cells_device, (int)n_grids, topk,
      static_cast<uint8_t*>(out_u8), reinterpret_cast<int*>(status));
  CTL_LAUNCH_CHECK();
  return 0;
}

int ctl_visrank_select(const int64_t* topk_idx, int64_t nq, int32_t k, const int32_t* q_pid, const int32_t* q_cam,
                       const int32_t* g_pid, const uint64_t* g_cammask, int64_t ng, int32_t topk, int64_t* out_idx,
                       int8_t* out_matched, int32_t* status, ctl_stream_t stream) {
  CTL_CHECK_ARG(topk_idx && q_pid && q_cam && g_pid && g_cammask && out_idx && out_matched && status, "null pointer");
  CTL_CHECK_ARG(nq >= 1 && k >= 1 && ng >= 1 && topk >= 1, "nq = %lld, k = %d, ng = %lld, topk = %d: expected >= 1",
                (long long)nq, k, (long long)ng, topk);
  int rc = ctl_device_check();
  if (rc) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  CTL_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
  visrank_select_kernel<<<(unsigned)((nq + 127) / 128), 128, 0, st>>>(topk_idx, (long long)nq, k, q_pid, q_cam, g_pid,
                                                                     g_cammask, (long long)ng, topk, out_idx,
                                                                     out_matched, reinterpret_cast<int*>(status));
  CTL_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
