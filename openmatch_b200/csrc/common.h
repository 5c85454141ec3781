// Shared host-side plumbing of libopenmatch_b200.so: thread-local error message, CUDA error mapping,
// device-property cache.
#pragma once
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

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

// cudaMalloc for the handles' storage and workspaces.  With OPENMATCH_B200_POISON_ALLOC=1 in the environment every fresh
// buffer is first filled with 0xFF bytes (NaN in fp32, bf16 and fp16), so that tests can tell a read of never-written
// memory from the driver's zero-filled pages.  Testing only: it synchronises the device on every allocation.
static inline cudaError_t dev_malloc(void** p, size_t bytes) {
  cudaError_t e = cudaMalloc(p, bytes);
  const char* poison = getenv("OPENMATCH_B200_POISON_ALLOC");
  if (e == cudaSuccess && bytes > 0 && poison && poison[0] == '1') {
    e = cudaMemset(*p, 0xFF, bytes);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
  }
  return e;
}
template <class T>
static inline cudaError_t dev_malloc(T** p, size_t bytes) {
  return dev_malloc(reinterpret_cast<void**>(p), bytes);
}

// NVTX range (header-only NVTX3: a no-op unless a profiler injects itself) around the host-side enqueue of a phase;
// names: om.encode[.layer], om.search[.scan|.select|.rescore|.exchange|.certify|.level*], om.loss
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
  NvtxRange(const NvtxRange&) = delete;
  NvtxRange& operator=(const NvtxRange&) = delete;
};

}  // namespace om
