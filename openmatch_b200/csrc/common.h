// Shared host-side plumbing of libopenmatch_b200.so: thread-local error message, CUDA error mapping,
// device-property cache.
#pragma once
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/openmatch_b200.h"

namespace om {

char* err_buf();  // thread-local, 512 bytes (defined in api.cu)

static inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(err_buf(), 512, fmt, ap);
  va_end(ap);
  return code;
}

#define OM_CUDA(expr)                                                                             \
  do {                                                                                            \
    cudaError_t e__ = (expr);                                                                     \
    if (e__ != cudaSuccess) {                                                                     \
      cudaGetLastError();                                                                         \
      return ::om::fail(e__ == cudaErrorMemoryAllocation ? OM_ENOMEM : OM_ECUDA, "%s failed: %s (%s:%d)", #expr, \
                        cudaGetErrorString(e__), __FILE__, __LINE__);                             \
    }                                                                                             \
  } while (0)

#define OM_TRY(expr)            \
  do {                          \
    int rc__ = (expr);          \
    if (rc__ < 0) return rc__;  \
  } while (0)

// Number of SMs of the current device (cached); negative OM_E* when no usable sm_90 device exists.
int device_sm_count();

static inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

// NVTX range (header-only NVTX3: a no-op unless a profiler injects itself) around the host-side enqueue of a phase;
// names: om.encode[.layer], om.search[.scan|.select|.rescore|.exchange|.certify|.level*], om.loss
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
  NvtxRange(const NvtxRange&) = delete;
  NvtxRange& operator=(const NvtxRange&) = delete;
};

}  // namespace om
