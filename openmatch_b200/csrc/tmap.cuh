// Host-side TMA tensor-map construction.  cuTensorMapEncodeTiled is fetched through
// cudaGetDriverEntryPoint so the library links against the CUDA runtime only (no -lcuda needed;
// the build container has no driver).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace om {

typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                         const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                         CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                         CUtensorMapFloatOOBfill);

static inline PFN_tmapEncodeTiled tmap_encode_fn() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
  }
  return fn;
}

// 2-D row-major bf16 tensor [rows, inner] with row pitch `row_stride_bytes` (multiple of 16), tiled into
// boxes of {box_inner (= 64 elements = 128 B), box_rows (<= 256)} with the 128-byte swizzle — the layout
// wgmma consumes as a K-major SWIZZLE_128B operand.  Out-of-bounds elements read as zero.
// Returns 0 on success, else the CUresult (or -1 when the driver entry point is unavailable).
// (also used for TMA stores: box {64, 32} of a bf16 output matrix)
static inline int make_tmap_bf16_2d(CUtensorMap* out, const void* gptr, uint64_t inner, uint64_t rows,
                                    uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_rows) {
  PFN_tmapEncodeTiled fn = tmap_encode_fn();
  if (!fn) return -1;
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(gptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return static_cast<int>(r);
}

// Generic 2-D row-major tiled map: `elem_bytes` 1 (int8), 2 (bf16) or 4 (fp32); swizzle_bytes 128 or 64 (= the box's
// inner extent in bytes).  Used by the residual epilogue: fp32 boxes {32 cols, 32 rows} with SWIZZLE_128B (TMA load +
// in-place TMA store of the residual stream) and bf16 boxes {32 cols, 32 rows} with SWIZZLE_64B (one chunk of a bf16
// output); and by the int8 search scan: boxes {128 codes, 128 rows} with SWIZZLE_128B.
static inline int make_tmap_2d(CUtensorMap* out, const void* gptr, int elem_bytes, uint64_t inner, uint64_t rows,
                               uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_rows, int swizzle_bytes) {
  PFN_tmapEncodeTiled fn = tmap_encode_fn();
  if (!fn) return -1;
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_rows};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType type = elem_bytes == 4   ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                   : elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                                     : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUresult r = fn(out, type, 2,
                  const_cast<void*>(gptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return static_cast<int>(r);
}

}  // namespace om
