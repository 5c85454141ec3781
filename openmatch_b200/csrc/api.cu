// Library-level entry points of libopenmatch_b200.so (error string, ABI version, device probe).
#include "common.h"

namespace om {

char* err_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}

int device_sm_count() {
  static int cached_dev = -1, cached_sms = 0;
  int dev = -1;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(OM_ENODEVICE, "no CUDA device available: %s (this library has no CPU path)", cudaGetErrorString(e));
  }
  if (dev == cached_dev) return cached_sms;
  // Launcher state (tile-counter pool, loss workspace, one-time cudaFuncSetAttribute guards) is per process and
  // therefore per device: one process drives ONE GPU (torchrun's model).  A second device is refused loudly
  // instead of launching with another device's buffers / missing shared-memory opt-ins.
  if (cached_dev >= 0)
    return fail(OM_ESTATE, "libopenmatch_b200 is bound to CUDA device %d in this process; device %d is current "
                "(one process per GPU)", cached_dev, dev);
  cudaDeviceProp p;
  e = cudaGetDeviceProperties(&p, dev);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(OM_ENODEVICE, "cudaGetDeviceProperties failed: %s", cudaGetErrorString(e));
  }
  if (p.major != 9 || p.minor != 0)
    return fail(OM_ENODEVICE, "device %d is sm_%d%d; libopenmatch_b200 is built for sm_90a (H100) only", dev, p.major,
                p.minor);
  cached_dev = dev;
  cached_sms = p.multiProcessorCount;
  return cached_sms;
}

}  // namespace om

extern "C" {
int om_abi_version(void) { return OM_ABI_VERSION; }
const char* om_last_error(void) { return om::err_buf(); }
int om_device_sm_count(void) { return om::device_sm_count(); }
}
