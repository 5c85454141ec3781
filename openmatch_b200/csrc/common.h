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

// Layout of one device workspace: add() places a region of `region_bytes` at the next 256-byte boundary and returns its
// byte offset; `bytes` is the size the regions need.
struct Layout {
  size_t bytes = 0;
  size_t add(size_t region_bytes) {
    const size_t o = bytes;
    bytes += round_up(region_bytes, 256);
    return o;
  }
};
// The region at byte offset `off` of the workspace at `base`.
template <class T>
static inline T* region(void* base, size_t off) {
  return reinterpret_cast<T*>(static_cast<uint8_t*>(base) + off);
}

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
