// `T.Resize((h, w))` of the eval and training transforms (datasets/transforms/build.py:19,29) on the device: PIL's
// BILINEAR resampler (Image.resize on an RGB image), bit for bit, for a ragged batch of native-size HWC uint8 images.
//
// PIL resamples each axis separately with fixed-point weights: the width pass first, then the height pass over the
// width pass's output clipped to uint8.  Per axis (`in` source pixels -> `out` output pixels), in IEEE double:
//   scale = in / out, fs = max(scale, 1), support = fs, ss = 1 / fs, center = (o + 0.5) scale,
//   xmin = max((int)(center - support + 0.5), 0), taps = min((int)(center + support + 0.5), in) - xmin,
//   w[t] = tri((t + xmin - center + 0.5) ss), normalised by their sum taken in tap order,
//   k[t] = (int)(0.5 + w[t] 2^22), pixel = clamp((2^21 + sum_t src[xmin + t] k[t]) >> 22, 0, 255).
// Every double operation is an explicit round-to-nearest intrinsic, so nvcc cannot contract a multiply and an add into
// an FMA: the weights are the ones PIL computes.  PIL skips a pass whose size does not change; a pass with in == out
// has the taps {1, 0} and copies, so running both passes always gives the same bytes.
//
// Each thread derives the taps of its own output index inline (no coefficient tables) and applies them to several
// rows (width pass) or columns (height pass).  One CTA row per image: the image's first row in the uint8 intermediate
// [sum of h, out_w, 3] is the sum of the heights of the valid images before it, reduced by each CTA from the table.
#include <stdint.h>

#include <algorithm>

#include "common.h"
#include "wgmma.cuh"

namespace ctl {

constexpr int RS_THREADS = 256;
constexpr int RS_PER = 4;                // rows per thread (width pass), columns per thread (height pass)
constexpr long long RS_MAX_SIDE = 1 << 24;

using ResizeEntry = ctl_resize_entry;

// 0: a real image inside src_bytes; 1: a mock row (h == 0 or w == 0, zeros); 2: an entry that does not fit
__device__ __forceinline__ int entry_kind(const ResizeEntry& e, long long src_bytes) {
  if (e.h < 0 || e.w < 0 || e.h > RS_MAX_SIDE || e.w > RS_MAX_SIDE) return 2;
  if (e.h == 0 || e.w == 0) return 1;
  if (e.offset < 0 || e.offset > src_bytes || e.h * e.w * 3 > src_bytes - e.offset) return 2;
  return 0;
}

// first intermediate row of image b: the heights of the real images before it, summed by the whole CTA
static __device__ long long first_row(const ResizeEntry* __restrict__ table, int b, long long src_bytes) {
  __shared__ long long part[RS_THREADS / 32];
  long long acc = 0;
  for (int j = threadIdx.x; j < b; j += blockDim.x) {
    const ResizeEntry e = table[j];
    if (entry_kind(e, src_bytes) == 0) acc += e.h;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  long long row0 = 0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) row0 += part[i];
  return row0;
}

struct Taps {
  double center, ss, ww;
  int xmin, n;
};

__device__ __forceinline__ double tap_weight(const Taps& t, int x) {
  const double v = fabs(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + t.xmin), t.center), 0.5), t.ss));
  return v < 1.0 ? __dsub_rn(1.0, v) : 0.0;
}

__device__ __forceinline__ Taps make_taps(int o, int in, int out) {
  Taps t;
  const double scale = __ddiv_rn((double)in, (double)out);
  const double support = fmax(scale, 1.0);  // the triangle's support (1) times the filter scale
  t.ss = __ddiv_rn(1.0, support);
  t.center = __dmul_rn(__dadd_rn((double)o, 0.5), scale);
  t.xmin = max(__double2int_rz(__dadd_rn(__dsub_rn(t.center, support), 0.5)), 0);
  t.n = min(__double2int_rz(__dadd_rn(__dadd_rn(t.center, support), 0.5)), in) - t.xmin;
  t.ww = 0.0;
  for (int x = 0; x < t.n; ++x) t.ww = __dadd_rn(t.ww, tap_weight(t, x));
  return t;
}

// fixed-point weight of tap x (PRECISION_BITS = 22); weights are never negative
__device__ __forceinline__ int tap_coeff(const Taps& t, int x) {
  double w = tap_weight(t, x);
  if (t.ww != 0.0) w = __ddiv_rn(w, t.ww);
  return __double2int_rz(__dadd_rn(0.5, __dmul_rn(w, 4194304.0)));
}

__device__ __forceinline__ uint8_t clip8(int acc) { return (uint8_t)min(max(acc >> 22, 0), 255); }

// width pass: image b's rows resampled from w to out_w into mid rows [row0, row0 + h); a thread owns one output
// column x of RS_PER consecutive rows
__global__ void __launch_bounds__(RS_THREADS) resize_width_kernel(const uint8_t* __restrict__ src, long long src_bytes,
                                                                  const ResizeEntry* __restrict__ table, int out_w,
                                                                  uint8_t* __restrict__ mid, long long mid_rows) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const ResizeEntry e = table[b];
  const long long row0 = first_row(table, b, src_bytes);
  if (entry_kind(e, src_bytes) != 0 || row0 + e.h > mid_rows) return;  // the height pass writes zeros and the status
  const int h = (int)e.h, w = (int)e.w;
  const uint8_t* img = src + e.offset;
  const long long units = (long long)((h + RS_PER - 1) / RS_PER) * out_w;
  for (long long u = (long long)blockIdx.y * blockDim.x + threadIdx.x; u < units; u += (long long)gridDim.y * blockDim.x) {
    const int x = (int)(u % out_w), y0 = (int)(u / out_w) * RS_PER;
    const int rows = min(RS_PER, h - y0);
    const Taps t = make_taps(x, w, out_w);
    int acc[RS_PER][3];
#pragma unroll
    for (int r = 0; r < RS_PER; ++r) acc[r][0] = acc[r][1] = acc[r][2] = 1 << 21;
    for (int k = 0; k < t.n; ++k) {
      const int c = tap_coeff(t, k);
      const uint8_t* s = img + ((size_t)y0 * w + t.xmin + k) * 3;
#pragma unroll
      for (int r = 0; r < RS_PER; ++r) {
        if (r < rows) {
          const uint8_t* p = s + (size_t)r * w * 3;
          acc[r][0] += p[0] * c;
          acc[r][1] += p[1] * c;
          acc[r][2] += p[2] * c;
        }
      }
    }
#pragma unroll
    for (int r = 0; r < RS_PER; ++r) {
      if (r < rows) {
        uint8_t* d = mid + ((size_t)(row0 + y0 + r) * out_w + x) * 3;
        d[0] = clip8(acc[r][0]);
        d[1] = clip8(acc[r][1]);
        d[2] = clip8(acc[r][2]);
      }
    }
  }
}

// height pass: mid rows [row0, row0 + h) resampled from h to out_h into out[b]; a thread owns one output row y of
// RS_PER consecutive columns.  Mock rows and entries that do not fit become zeros; the latter set *status.
__global__ void __launch_bounds__(RS_THREADS) resize_height_kernel(const uint8_t* __restrict__ mid, long long mid_rows,
                                                                   const ResizeEntry* __restrict__ table,
                                                                   long long src_bytes, int out_h, int out_w,
                                                                   uint8_t* __restrict__ out, int* __restrict__ status) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const ResizeEntry e = table[b];
  const long long row0 = first_row(table, b, src_bytes);
  const int kind = entry_kind(e, src_bytes);
  const bool fits = kind == 0 && row0 + e.h <= mid_rows;
  if (!fits && kind != 1 && blockIdx.y == 0 && threadIdx.x == 0) atomicOr(status, kind == 2 ? 1 : 2);
  const int groups = (out_w + RS_PER - 1) / RS_PER;
  const long long units = (long long)out_h * groups;
  uint8_t* img = out + (size_t)b * out_h * out_w * 3;
  for (long long u = (long long)blockIdx.y * blockDim.x + threadIdx.x; u < units; u += (long long)gridDim.y * blockDim.x) {
    const int y = (int)(u / groups), x0 = (int)(u % groups) * RS_PER;
    const int cols = min(RS_PER, out_w - x0);
    uint8_t* d = img + ((size_t)y * out_w + x0) * 3;
    if (!fits) {
      for (int i = 0; i < cols * 3; ++i) d[i] = 0;
      continue;
    }
    const Taps t = make_taps(y, (int)e.h, out_h);
    int acc[RS_PER][3];
#pragma unroll
    for (int i = 0; i < RS_PER; ++i) acc[i][0] = acc[i][1] = acc[i][2] = 1 << 21;
    for (int k = 0; k < t.n; ++k) {
      const int c = tap_coeff(t, k);
      const uint8_t* s = mid + ((size_t)(row0 + t.xmin + k) * out_w + x0) * 3;
#pragma unroll
      for (int i = 0; i < RS_PER; ++i) {
        if (i < cols) {
          acc[i][0] += s[3 * i] * c;
          acc[i][1] += s[3 * i + 1] * c;
          acc[i][2] += s[3 * i + 2] * c;
        }
      }
    }
#pragma unroll
    for (int i = 0; i < RS_PER; ++i) {
      if (i < cols) {
        d[3 * i] = clip8(acc[i][0]);
        d[3 * i + 1] = clip8(acc[i][1]);
        d[3 * i + 2] = clip8(acc[i][2]);
      }
    }
  }
}

static bool resize_size_ok(int32_t out_h, int32_t out_w) { return out_h >= 1 && out_w >= 1 && out_h <= 16384 && out_w <= 16384; }

static unsigned grid_y(long long units) { return (unsigned)std::min<long long>(std::max<long long>((units + RS_THREADS - 1) / RS_THREADS, 1), 65535); }

}  // namespace ctl

using namespace ctl;

extern "C" {

size_t ctl_resize_bilinear_u8_workspace_bytes(int64_t total_rows, int32_t out_h, int32_t out_w) {
  if (total_rows < 0 || !resize_size_ok(out_h, out_w)) return 0;
  const size_t bytes = (size_t)std::max<int64_t>(total_rows, 1) * out_w * 3;
  return (bytes + 255) & ~size_t(255);
}

int ctl_resize_bilinear_u8(const void* src, int64_t src_bytes, const void* table_device, int64_t n, int32_t out_h,
                           int32_t out_w, void* out_u8_nhwc, int32_t* status, void* workspace, size_t workspace_bytes,
                           ctl_stream_t stream) {
  CTL_CHECK_ARG(src && table_device && out_u8_nhwc && status && workspace, "null pointer");
  CTL_CHECK_ARG(n >= 1 && n <= INT32_MAX, "n = %lld: expected 1 <= n < 2^31", (long long)n);
  CTL_CHECK_ARG(resize_size_ok(out_h, out_w), "output size %d x %d: expected 1..16384 on each side", out_h, out_w);
  CTL_CHECK_ARG(src_bytes >= 0, "src_bytes < 0");
  CTL_CHECK_ARG(workspace_bytes >= (size_t)out_w * 3,
                "workspace of %zu bytes holds no intermediate row of %d bytes (ctl_resize_bilinear_u8_workspace_bytes)",
                workspace_bytes, out_w * 3);
  int rc = ctl_device_check();
  if (rc) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  const long long mid_rows = (long long)(workspace_bytes / ((size_t)out_w * 3));
  const auto* table = static_cast<const ResizeEntry*>(table_device);
  auto* mid = static_cast<uint8_t*>(workspace);
  CTL_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
  // width pass: sized for the mean height the workspace was planned for; taller images loop
  const long long mean_h = (mid_rows + n - 1) / n;
  CTL_CUDA(launch_k(resize_width_kernel, dim3((unsigned)n, grid_y((mean_h + RS_PER - 1) / RS_PER * out_w)), dim3(RS_THREADS),
                    0, st, static_cast<const uint8_t*>(src), (long long)src_bytes, table, (int)out_w, mid, mid_rows));
  CTL_CUDA(launch_k(resize_height_kernel, dim3((unsigned)n, grid_y((long long)out_h * ((out_w + RS_PER - 1) / RS_PER))),
                    dim3(RS_THREADS), 0, st, static_cast<const uint8_t*>(mid), mid_rows, table, (long long)src_bytes,
                    (int)out_h, (int)out_w, static_cast<uint8_t*>(out_u8_nhwc), reinterpret_cast<int*>(status)));
  return 0;
}

}  // extern "C"
