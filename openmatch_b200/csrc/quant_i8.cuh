// Row quantisation of int8 index storage (om_index_create_typed(d, OM_I8)), shared by the index's add and the encoder's
// OM_I8 output so that both store the same bytes for the same fp32 values.
//
// Row layout (pitch dpad + 16 bytes, dpad = d rounded up to 16, so TMA row strides stay multiples of 16):
//   bytes [0, d)            codes c_j = clamp(rint(x_j / s), -127, 127): IEEE division, round half to even
//   bytes [d, dpad)         0
//   bytes [dpad, dpad + 4)  fp32 scale s = amax / 127 (IEEE division), amax = max_j |x_j|; a zero row has s = 0, codes 0
//   bytes [dpad + 4, +16)   0
// The stored value of element j is fp32(s * c_j).  A row holding inf or NaN gets a NaN scale and zero codes, so that
// om_index_commit counts it and searches refuse the index (an fp32 scale cannot be NaN otherwise).
#pragma once
#include <math.h>
#include <stdint.h>

namespace om {

__host__ __device__ constexpr int i8_dpad(int d) { return (d + 15) & ~15; }

// One warp quantises one row; get(j) returns element j (fp32) for j < d and may be called twice per element.  Returns
// whether every element was finite (warp-uniform).
template <class Get>
__device__ __forceinline__ bool quantize_row_i8(Get&& get, int d, int dpad, int8_t* dst, int lane) {
  float amax = 0.f;
  bool finite = true;
  for (int j = lane; j < d; j += 32) {
    const float x = get(j);
    finite = finite && isfinite(x);
    amax = fmaxf(amax, fabsf(x));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  finite = __all_sync(0xffffffffu, finite);
  const float s = finite ? __fdiv_rn(amax, 127.f) : __int_as_float(0x7fc00000);
  for (int j = lane; j < dpad; j += 32) {
    float c = 0.f;
    if (j < d && s > 0.f) c = fminf(fmaxf(rintf(__fdiv_rn(get(j), s)), -127.f), 127.f);
    dst[j] = static_cast<int8_t>(c);
  }
  if (lane < 4) reinterpret_cast<float*>(dst + dpad)[lane] = lane == 0 ? s : 0.f;
  return finite;
}

}  // namespace om
