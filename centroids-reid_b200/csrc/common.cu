// Error reporting, device checks and the run-time resolved cuTensorMapEncodeTiled.
#include "common.h"

#include <cudaTypedefs.h>
#include <string.h>

namespace ctl {

static thread_local char g_error[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}

int sm_count() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      cached = n;
    else
      return 132;  // H100 SXM
  }
  return cached;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn resolve_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess || p == nullptr)
    return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType dtype, uint32_t elem_bytes, uint32_t rank,
                      const void* base, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                      CUtensorMapSwizzle swizzle) {
  EncodeTiledFn fn = resolve_encode();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled is not available from the CUDA driver");
    return CTL_ERR_NO_DEVICE;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15u) != 0) {
    set_error("tensor base %p is not 16-byte aligned", base);
    return CTL_ERR_INVALID_ARGUMENT;
  }
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bx[5], es[5];
  for (uint32_t i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) {
      gstr[i - 1] = strides_bytes[i];
      if (strides_bytes[i] % 16 != 0) {
        set_error("tensor stride %llu of dim %u is not a multiple of 16 bytes", (unsigned long long)strides_bytes[i], i);
        return CTL_ERR_INVALID_ARGUMENT;
      }
    }
  }
  (void)elem_bytes;
  CUresult r = fn(map, dtype, rank, const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %u, dims %llu x %llu, box %u x %u)", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 1), box[0], rank > 1 ? box[1] : 1);
    return CTL_ERR_INVALID_ARGUMENT;
  }
  return 0;
}

}  // namespace ctl

extern "C" {

const char* ctl_last_error(void) { return ctl::g_error; }

int ctl_abi_version(void) { return CTL_ABI_VERSION; }

int ctl_device_check(void) {
  static int cached = 1;  // 1 = unknown
  if (cached != 1) return cached;
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) {
    ctl::set_error("no CUDA device: libctl_b200 has no CPU fallback");
    cudaGetLastError();
    return CTL_ERR_NO_DEVICE;  // not cached: a device may appear later in the process
  }
  if (major != 9) {
    ctl::set_error("device compute capability %d.x is not sm_90 (H100); kernels are built for sm_90a only", major);
    return CTL_ERR_NO_DEVICE;
  }
  cached = 0;
  return 0;
}

}  // extern "C"
