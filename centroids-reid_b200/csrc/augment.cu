// Training-time augmentation on the device (datasets/transforms/build.py:15-27, random_erasing.py:30-55): from a batch
// of already-resized uint8 HWC crops and host-drawn per-image parameters to the normalised fp32 NCHW tensor the trunk
// consumes -- RandomHorizontalFlip -> Pad(p, fill 0) -> RandomCrop -> ToTensor -> Normalize -> RandomErasing
// (erased pixels take the raw PIXEL_MEAN value, after normalisation, like the reference) in ONE pass:
// 3 B read + 12 B written per pixel (the uint8 batch also cuts the H2D copy 4x against fp32 crops).
#include <stdint.h>

#include <algorithm>

#include "common.h"
#include "wgmma.cuh"

namespace ctl {

// per image: flip, crop_top, crop_left (in the padded image), erase_x1 (row), erase_y1 (col), erase_h, erase_w
// (erase_h == 0: no erasing), is_real (0: mock image -> all zeros, datasets/bases.py:378-391)
struct AugParams {
  int v[8];
};

__global__ void __launch_bounds__(256) augment_kernel(const uint8_t* __restrict__ src, int B, int H, int W, int pad,
                                                      const AugParams* __restrict__ params, float m0, float m1, float m2,
                                                      float is0, float is1, float is2 /* std */, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = (long long)B * H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const int y = (int)((i / W) % H);
    const int b = (int)(i / ((long long)W * H));
    const AugParams p = params[b];
    float o0 = 0.f, o1 = 0.f, o2 = 0.f;
    if (p.v[7]) {
      const bool erased = p.v[5] > 0 && y >= p.v[3] && y < p.v[3] + p.v[5] && x >= p.v[4] && x < p.v[4] + p.v[6];
      if (erased) {
        o0 = m0;
        o1 = m1;
        o2 = m2;
      } else {
        const int yy = y + p.v[1] - pad, xx = x + p.v[2] - pad;  // coordinate in the (flipped) unpadded image
        float r = 0.f, g = 0.f, bl = 0.f;                        // Pad(fill = 0)
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
          const int sx = p.v[0] ? W - 1 - xx : xx;
          const uint8_t* s = src + (((size_t)b * H + yy) * W + sx) * 3;
          r = s[0] / 255.f;  // IEEE divisions: bit-identical to ToTensor + Normalize on the host
          g = s[1] / 255.f;
          bl = s[2] / 255.f;
        }
        o0 = (r - m0) / is0;
        o1 = (g - m1) / is1;
        o2 = (bl - m2) / is2;
      }
    }
    const size_t plane = (size_t)H * W, base = (size_t)b * 3 * plane + (size_t)y * W + x;
    out[base] = o0;
    out[base + plane] = o1;
    out[base + 2 * plane] = o2;
  }
}

}  // namespace ctl

using namespace ctl;

extern "C" {

int ctl_augment_batch_u8(const void* images_u8_nhwc, int32_t n, int32_t h, int32_t w, int32_t pad, const int32_t* params_device,
                         const float* mean3_host, const float* std3_host, float* out_nchw, ctl_stream_t stream) {
  CTL_CHECK_ARG(images_u8_nhwc && params_device && mean3_host && std3_host && out_nchw, "null pointer");
  CTL_CHECK_ARG(n >= 1 && h >= 1 && w >= 1 && pad >= 0, "bad shape");
  CTL_CHECK_ARG(std3_host[0] > 0 && std3_host[1] > 0 && std3_host[2] > 0, "std must be positive");
  int rc = ctl_device_check();
  if (rc) return rc;
  const long long total = (long long)n * h * w;
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
  CTL_CUDA(launch_k(augment_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, static_cast<const uint8_t*>(images_u8_nhwc),
                    (int)n, (int)h, (int)w, (int)pad, reinterpret_cast<const AugParams*>(params_device), mean3_host[0],
                    mean3_host[1], mean3_host[2], std3_host[0], std3_host[1], std3_host[2], out_nchw));
  return 0;
}

}  // extern "C"
