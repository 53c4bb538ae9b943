// Optimizer step of the training loop (solver/build.py:9-47, train_ctl_model.py:155-159): torch.optim.Adam with L2
// weight decay over the ~160 trunk / head tensors as ONE multi-tensor launch, and the plain SGD step of the center
// parameters (gradient pre-multiplied by 1 / CENTER_LOSS_WEIGHT).  fp32 throughout; HBM-bound: 16 B read + 12 B
// written per parameter.
#include <stdint.h>

#include <algorithm>

#include "common.h"
#include "wgmma.cuh"

namespace ctl {

static constexpr int OPT_CHUNK = 8192;  // elements per CTA iteration

// one entry per tensor; chunk_begin = prefix sum of ceil(numel / OPT_CHUNK)
struct AdamEntry {
  float* p;
  const float* g;
  float* m;
  float* v;
  long long numel;
  long long chunk_begin;
};

__global__ void __launch_bounds__(256) adam_multi_kernel(const AdamEntry* __restrict__ table, int n_tensors, long long n_chunks,
                                                         float lr, float beta1, float beta2, float eps, float weight_decay,
                                                         float bc1, float bc2_sqrt, float grad_mul,
                                                         const int* __restrict__ skip_flag) {
  pdl_launch_dependents();
  pdl_wait();
  if (skip_flag != nullptr && *skip_flag != 0) return;  // overflowing gradients: GradScaler.step skips the update
  for (long long chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
    // the tensor that owns this chunk: last entry with chunk_begin <= chunk
    int lo = 0, hi = n_tensors - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (table[mid].chunk_begin <= chunk) lo = mid; else hi = mid - 1;
    }
    const AdamEntry e = table[lo];
    const long long base = (chunk - e.chunk_begin) * OPT_CHUNK;
    const long long end = min(e.numel, base + OPT_CHUNK);
    for (long long i = base + threadIdx.x; i < end; i += blockDim.x) {
      // torch/optim/_functional.py adam(): grad += wd * p; m, v updates; denom = sqrt(v) / sqrt(bc2) + eps;
      // p -= (lr / bc1) * m / denom
      float g = e.g[i] * grad_mul;
      const float p = e.p[i];
      g = fmaf(weight_decay, p, g);
      const float m = fmaf(beta1, e.m[i], (1.f - beta1) * g);
      const float v = fmaf(beta2, e.v[i], (1.f - beta2) * g * g);
      e.m[i] = m;
      e.v[i] = v;
      const float denom = sqrtf(v) / bc2_sqrt + eps;
      e.p[i] = p - (lr / bc1) * (m / denom);
    }
  }
}

__global__ void __launch_bounds__(256) sgd_kernel(float* __restrict__ p, const float* __restrict__ g, long long numel, float lr,
                                                  float grad_mul, const int* __restrict__ skip_flag) {
  pdl_launch_dependents();
  pdl_wait();
  if (skip_flag != nullptr && *skip_flag != 0) return;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += (long long)gridDim.x * blockDim.x)
    p[i] = fmaf(-lr, g[i] * grad_mul, p[i]);
}

// found-inf check (and optional in-place rescale) over a list of gradient tensors: the role of
// torch.cuda.amp.GradScaler.unscale_ in the reference's PL native-AMP trainer (utils/misc.py:111)
struct GradEntry {
  float* g;
  long long numel;
  long long chunk_begin;
};

__global__ void __launch_bounds__(256) grad_check_multi_kernel(const GradEntry* __restrict__ table, int n_tensors,
                                                               long long n_chunks, float mul,
                                                               const float* __restrict__ mul_dev, int* __restrict__ found_inf) {
  pdl_launch_dependents();
  pdl_wait();
  if (mul_dev != nullptr) mul *= *mul_dev;  // e.g. base_scale / scale of the dynamic loss scaler (a device scalar)
  bool bad = false;
  for (long long chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
    int lo = 0, hi = n_tensors - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (table[mid].chunk_begin <= chunk) lo = mid; else hi = mid - 1;
    }
    const GradEntry e = table[lo];
    const long long base = (chunk - e.chunk_begin) * OPT_CHUNK;
    const long long end = min(e.numel, base + OPT_CHUNK);
    for (long long i = base + threadIdx.x; i < end; i += blockDim.x) {
      float g = e.g[i];
      if (mul != 1.f) {
        g *= mul;
        e.g[i] = g;
      }
      bad |= !isfinite(g);
    }
  }
  if (__syncthreads_or(bad ? 1 : 0) && threadIdx.x == 0) atomicOr(found_inf, 1);
}

// torch.cuda.amp.GradScaler.update() on the device: state = {scale, scale / base, base / scale}
__global__ void loss_scale_update_kernel(float* __restrict__ state, int* __restrict__ tracker, int* __restrict__ found_inf,
                                         int* __restrict__ last_found, float base, float growth, float backoff, int interval) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int found = *found_inf;
  float scale = state[0];
  if (found) {
    scale *= backoff;
    *tracker = 0;
  } else if (++(*tracker) >= interval) {
    const float grown = scale * growth;
    if (isfinite(grown)) scale = grown;  // like GradScaler: a growth that would overflow keeps the current scale
    *tracker = 0;
  }
  state[0] = scale;
  state[1] = scale / base;
  state[2] = base / scale;
  *last_found = found;
  *found_inf = 0;
}

}  // namespace ctl

using namespace ctl;

extern "C" {

int ctl_adam_multi_step(const void* table_device, int32_t n_tensors, int64_t n_chunks, float lr, float beta1, float beta2,
                        float eps, float weight_decay, int64_t step, float grad_mul, const int32_t* skip_flag,
                        ctl_stream_t stream) {
  CTL_CHECK_ARG(table_device && n_tensors >= 1 && n_chunks >= 1 && step >= 1, "bad arguments");
  static_assert(sizeof(AdamEntry) == 48, "ctl_adam_entry layout");
  int rc = ctl_device_check();
  if (rc) return rc;
  const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
  const int grid = (int)std::min<long long>(n_chunks, (long long)sm_count() * 8);
  CTL_CUDA(launch_k(adam_multi_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream,
                    static_cast<const AdamEntry*>(table_device), (int)n_tensors, (long long)n_chunks, lr, beta1, beta2, eps,
                    weight_decay, (float)bc1, (float)sqrt(bc2), grad_mul, skip_flag));
  return 0;
}

int ctl_loss_scale_update(float* state3, int32_t* tracker, int32_t* found_inf, int32_t* last_found, float base_scale,
                          float growth_factor, float backoff_factor, int32_t growth_interval, ctl_stream_t stream) {
  CTL_CHECK_ARG(state3 && tracker && found_inf && last_found, "null pointer");
  CTL_CHECK_ARG(base_scale > 0 && growth_factor >= 1 && backoff_factor > 0 && backoff_factor <= 1 && growth_interval >= 1,
                "bad loss-scale hyper-parameters");
  int rc = ctl_device_check();
  if (rc) return rc;
  CTL_CUDA(launch_k(loss_scale_update_kernel, dim3(1), dim3(32), 0, (cudaStream_t)stream, state3, tracker, found_inf, last_found,
                    base_scale, growth_factor, backoff_factor, (int)growth_interval));
  return 0;
}

int ctl_grad_check_multi(const void* table_device, int32_t n_tensors, int64_t n_chunks, float mul, const float* mul_device,
                         int32_t* found_inf, ctl_stream_t stream) {
  CTL_CHECK_ARG(table_device && found_inf && n_tensors >= 1 && n_chunks >= 1, "bad arguments");
  static_assert(sizeof(GradEntry) == 24, "ctl_grad_entry layout");
  int rc = ctl_device_check();
  if (rc) return rc;
  const int grid = (int)std::min<long long>(n_chunks, (long long)sm_count() * 8);
  CTL_CUDA(launch_k(grad_check_multi_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream,
                    static_cast<const GradEntry*>(table_device), (int)n_tensors, (long long)n_chunks, mul, mul_device,
                    found_inf));
  return 0;
}

int ctl_sgd_step(float* param, const float* grad, int64_t numel, float lr, float grad_mul, const int32_t* skip_flag,
                 ctl_stream_t stream) {
  CTL_CHECK_ARG(param && grad && numel >= 1, "bad arguments");
  int rc = ctl_device_check();
  if (rc) return rc;
  const int grid = (int)std::min<long long>((numel + 255) / 256, (long long)sm_count() * 8);
  CTL_CUDA(launch_k(sgd_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, param, grad, (long long)numel, lr, grad_mul,
                    skip_flag));
  return 0;
}

}  // extern "C"
