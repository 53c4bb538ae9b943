// Host-side plumbing shared by every translation unit of libctl_b200.so: status codes,
// the thread-local error string behind ctl_last_error(), and cuTensorMapEncodeTiled
// resolved at run time through the CUDA runtime (no link-time dependency on libcuda).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <utility>

#include "../../include/ctl_b200.h"

namespace ctl {

void set_error(const char* fmt, ...);

#define CTL_CHECK_ARG(cond, ...)         \
  do {                                   \
    if (!(cond)) {                       \
      ::ctl::set_error(__VA_ARGS__);     \
      return CTL_ERR_INVALID_ARGUMENT;   \
    }                                    \
  } while (0)

#define CTL_CUDA(expr)                                                                      \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      ::ctl::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return static_cast<int>(_e);                                                          \
    }                                                                                       \
  } while (0)

#define CTL_LAUNCH_CHECK()                                                                  \
  do {                                                                                      \
    cudaError_t _e = cudaGetLastError();                                                    \
    if (_e != cudaSuccess) {                                                                \
      ::ctl::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return static_cast<int>(_e);                                                          \
    }                                                                                       \
  } while (0)

// Encodes a tiled tensor map (rank <= 5).  dims/strides innermost-first; strides[0] is implied
// by the element size and not passed to the driver.  Returns 0 or a CTL/CUDA status.
int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType dtype, uint32_t elem_bytes, uint32_t rank,
                      const void* base, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                      CUtensorMapSwizzle swizzle);

int sm_count();

// retrieval.cu: distances of rows [r0, r0 + rows) against rows [c0, c0 + cols) of one planes buffer of n rows (the
// row-sliced planes go straight to the GEMM, nothing is copied), bit-identical to those rows of ctl_dist_matrix.
int dist_matrix_rows(const void* planes, int64_t n, int32_t d, int32_t flags, int64_t r0, int64_t rows, int64_t c0,
                     int64_t cols, float* out, int64_t ld_out, cudaStream_t stream);

// bump allocator over a caller-provided workspace (256-byte aligned slices)
struct Workspace {
  char* base;
  size_t size;
  size_t off;
  Workspace(void* p, size_t n) : base(static_cast<char*>(p)), size(n), off(0) {}
  template <typename T>
  T* take(size_t count) {
    size_t bytes = (count * sizeof(T) + 255) & ~size_t(255);
    if (base == nullptr || off + bytes > size) {
      off += bytes;  // keep counting so the caller learns the required size
      return nullptr;
    }
    T* p = reinterpret_cast<T*>(base + off);
    off += bytes;
    return p;
  }
};

// ---- shared by conv.cu / train.cu ----
// pixel tile TH x TW = 128 of an Ho x Wo map
inline void pick_tile(int Ho, int Wo, int* TH, int* TW) {
  // TH*TW = 128, minimise the over-covered area; prefer wide tiles (longer contiguous runs)
  int best = -1, bth = 1, btw = 128;
  for (int tw = 128; tw >= 1; tw >>= 1) {
    const int th = 128 / tw;
    const long long cover = (long long)((Ho + th - 1) / th) * th * ((Wo + tw - 1) / tw) * tw;
    if (best < 0 || cover < best) {
      best = (int)cover;
      bth = th;
      btw = tw;
    }
  }
  *TH = bth;
  *TW = btw;
}

// Launch with programmatic stream serialization (PDL): the next kernel's prologue overlaps this one's drain; every
// kernel of this file calls pdl_wait() before it touches activations.  CTL_PDL=0 restores ordinary launches.
inline bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("CTL_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v == 1;
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}


}  // namespace ctl
