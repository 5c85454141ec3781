// Search scan of an int8 index (quant_i8.cuh row layout): s8 x s8 wgmma with exact int32 accumulation, the top-k filter
// applied to the combined fp32 score on the accumulator registers.  One kernel serves every round of an int8 index: the
// dense first round (every score stored) and the threshold rounds, for any number of queries.  The fp16 scan kernels
// (gemm.cuh, scan_gemm.cuh) and their options (pair_scan, scan_cluster_*) do not apply to int8 indices.
//
//   query      q ~ q_h = sig_hi * q_hi + sig_lo * q_lo: two int8 vectors, sig_hi = amax / 127, sig_lo = sig_hi / 254, so
//              q_h carries ~15 bits and the certificate's query term ||q - q_h|| * max ||x^|| stays far below the rank gaps
//   operands   per k block of 128 codes (one 128-byte SW128 row, the fp16 boxes' swizzle and descriptors; a k32 step
//              advances 32 B): the tile's 128 query rows of q_hi and of q_lo and 128 corpus rows, 48 KB per ring slot
//   tile       one CTA: 128 queries x 128 corpus rows; consumer warpgroup g owns queries [64 g, +64) and holds two
//              m64n128 int32 accumulator sets A_hi, A_lo (128 registers, the fp16 wide scan's m64n256 budget).  Products
//              and sums are exact: 127^2 * 16384 < 2^31
//   score      fp32(s_r * fp32(sig_hi * A_hi + fp32(sig_lo * A_lo))), s_r the row's scale: a few roundings of 2^-24 that
//              certify_kernel's bound covers (csrc/search.cu)
//   schedule   persistent, static, queries fastest: every CTA works on neighbouring corpus tiles
//   filter     FragFilter<32> (scan_epilogue.cuh) on the combined scores in accumulator fragment order: a thread owns two
//              query rows x 32 columns, as in scan_wide_kernel.  DENSE: every score stored at position = column
#pragma once
#include <stdint.h>

#include <type_traits>

#include "scan_epilogue.cuh"

namespace om {

constexpr int kI8BlockK = 128;                        // codes per k block
constexpr int kI8BlockN = 128;                        // corpus rows per tile
constexpr int kI8Stages = 4;
constexpr int kI8BoxBytes = kBlockM * kI8BlockK;      // 16 KB: 128 rows of one operand
constexpr int kI8StageBytes = 3 * kI8BoxBytes;        // q_hi, q_lo, corpus
constexpr int kI8Consumers = kStashThreads;           // two consumer warpgroups
constexpr int kI8StashOffset = kI8Stages * kI8StageBytes;
constexpr int kI8BarOffset = kI8StashOffset + kFragStashBytes;
constexpr int kI8SmemBytes = kI8BarOffset + 2 * kI8Stages * 8 + 1024;  // + slack for 1024-B alignment of the base
static_assert(kI8SmemBytes <= 232448, "int8 scan ring + stash exceed the 227 KB of shared memory an H100 block may use");

// ALLOW (threshold rounds only): filtered search, survivors are also masked by the allowed-row bitmap `allow`.
template <bool DENSE, bool ALLOW>
__global__ void __launch_bounds__(kGemmProducerThreads + kI8Consumers, 1)
scan_i8_kernel(const __grid_constant__ CUtensorMap tmQh, const __grid_constant__ CUtensorMap tmQl,
               const __grid_constant__ CUtensorMap tmX, int K, const int8_t* __restrict__ xrows, int64_t pitch, int dpad,
               const float2* __restrict__ qsig, const float* __restrict__ thr, unsigned long long* cand, int* count,
               int* overflow, int nq, int n_cols, int C, uint32_t row_base, const uint32_t* __restrict__ allow) {
  static_assert(!(DENSE && ALLOW), "a filtered first round runs as a threshold round at -inf");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  unsigned long long* stash = reinterpret_cast<unsigned long long*>(smem + kI8StashOffset);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kI8BarOffset);
  uint64_t* empty_bar = full_bar + kI8Stages;
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = static_cast<int>(threadIdx.x & 31);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmQh);
    tma_prefetch_desc(&tmQl);
    tma_prefetch_desc(&tmX);
  }
  if (warp == 1 && lane == 0) {
    ring_init(full_bar, empty_bar, kI8Stages, kI8Consumers / 32);
    fence_barrier_init();
  }
  __syncthreads();

  const int qgroups = (nq + kBlockM - 1) / kBlockM;
  const int num_tiles = qgroups * ((n_cols + kI8BlockN - 1) / kI8BlockN);
  const int num_k = (K + kI8BlockK - 1) / kI8BlockK;

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      // ------------------------------ TMA producer ------------------------------
      Ring<kI8Stages> ring;
      for (int tile = static_cast<int>(blockIdx.x); tile < num_tiles; tile += static_cast<int>(gridDim.x)) {
        const int m_blk = tile % qgroups, n_blk = tile / qgroups;
        for (int kb = 0; kb < num_k; ++kb) {
          uint64_t* bar = ring_acquire_tx(full_bar, empty_bar, ring, kI8StageBytes, 40);
          uint8_t* s = smem + ring.stage * kI8StageBytes;
          tma_load_2d(s, &tmQh, bar, kb * kI8BlockK, m_blk * kBlockM);
          tma_load_2d(s + kI8BoxBytes, &tmQl, bar, kb * kI8BlockK, m_blk * kBlockM);
          tma_load_2d(s + 2 * kI8BoxBytes, &tmX, bar, kb * kI8BlockK, n_blk * kI8BlockN);
          ring.advance();
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ------------------------------ consumers: wgmma + filter ------------------------------
    const int et = static_cast<int>(threadIdx.x) - kGemmProducerThreads;  // 0 .. 255
    const int wg = et >> 7;                                               // queries [64 wg, +64) of the tile's 128
    const int q4 = lane & 3;
    const int frow = 64 * wg + 16 * (warp & 3) + (lane >> 2);             // fragment rows frow, frow + 8
    Ring<kI8Stages> ring;
    FragFilter<32, ALLOW> filter{stash + et, cand, count, overflow, C, row_base, lane, allow};
    auto release = [&](uint32_t s) {
      if (lane == 0) mbar_arrive(&empty_bar[s]);
    };

    for (int tile = static_cast<int>(blockIdx.x); tile < num_tiles; tile += static_cast<int>(gridDim.x)) {
      const int m_blk = tile % qgroups, n_blk = tile / qgroups;
      const int row0 = m_blk * kBlockM + frow, row1 = row0 + 8;
      const int col0 = n_blk * kI8BlockN;
      // issued before the mainloop, first read after it: the loads' latency hides behind the MMAs
      const float inf = __int_as_float(0x7f800000);
      const float2 g0 = row0 < nq ? qsig[row0] : make_float2(0.f, 0.f), g1 = row1 < nq ? qsig[row1] : make_float2(0.f, 0.f);
      float t0 = inf, t1 = inf;
      if constexpr (!DENSE) {
        t0 = row0 < nq ? thr[row0] : inf;
        t1 = row1 < nq ? thr[row1] : inf;
      }
      float sc[32];  // scales of this thread's columns col0 + 8 (i >> 1) + 2 q4 + (i & 1)
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int c = col0 + 8 * (i >> 1) + 2 * q4 + (i & 1);
        sc[i] = c < n_cols ? __ldg(reinterpret_cast<const float*>(xrows + static_cast<size_t>(c) * pitch + dpad)) : 0.f;
      }

      int32_t ah[64], al[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) ah[i] = al[i] = 0;
      ring_consume(
          full_bar, ring, 0, num_k, 41,
          [&](uint32_t stage, uint32_t accumulate) {
            const uint32_t qh = smem_u32(smem + stage * kI8StageBytes) + wg * (64 * kI8BlockK);
            const uint32_t ql = qh + kI8BoxBytes;
            const uint32_t xb = smem_u32(smem + stage * kI8StageBytes + 2 * kI8BoxBytes);
#pragma unroll
            for (int k = 0; k < kI8BlockK / 32; ++k) {
              const uint64_t db = wgmma_desc(xb + k * 32, kDescKMajorSW128);
              const uint32_t acc = (accumulate | k) != 0 ? 1u : 0u;
              wgmma_m64n128k32_s8(ah, wgmma_desc(qh + k * 32, kDescKMajorSW128), db, acc);
              wgmma_m64n128k32_s8(al, wgmma_desc(ql + k * 32, kDescKMajorSW128), db, acc);
            }
          },
          release);
      wgmma_fence_regs(ah);
      wgmma_fence_regs(al);

      // combined scores in accumulator fragment order: v[4 j + 2 H + b] is fragment row frow + 8 H, column 8 j + 2 q4 + b
      float v[64];
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const int i = 2 * j + b;
          v[4 * j + b] = __fmul_rn(sc[i], __fmaf_rn(g0.x, static_cast<float>(ah[4 * j + b]), __fmul_rn(g0.y, static_cast<float>(al[4 * j + b]))));
          v[4 * j + 2 + b] = __fmul_rn(sc[i], __fmaf_rn(g1.x, static_cast<float>(ah[4 * j + 2 + b]), __fmul_rn(g1.y, static_cast<float>(al[4 * j + 2 + b]))));
        }

      if constexpr (DENSE) {  // first round: every score at position = column
#pragma unroll 1
        for (int h = 0; h < 2; ++h) {
          const int row = h ? row1 : row0;
          if (row >= nq) continue;
          unsigned long long* mine = cand + static_cast<size_t>(row) * C;
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int c = col0 + 8 * (i >> 1) + 2 * q4 + (i & 1);
            const int r = 4 * (i >> 1) + (i & 1);
            if (c < n_cols) mine[c] = make_key(h ? v[r + 2] : v[r], row_base + static_cast<uint32_t>(c));
          }
        }
        continue;
      }
      filter.tile(v, t0, t1, row0, col0, n_cols);
    }
    filter.drain();
  }

  __syncthreads();
}

// Host launcher.  Qh, Ql: [nq, K] int8 query splits, row pitch ldq bytes; qsig [nq] (sig_hi, sig_lo); X: the corpus rows of
// the round, [n_cols] rows of pitch `pitch` bytes with the scale at byte dpad.  dense: every score goes to
// cand[q * C + column], and allow is not read; otherwise survivors (score > thr[q]) are appended as
// make_key(score, row_base + column) and a list that would grow beyond C sets *overflow.  allow: nullptr, or the
// allowed-row bitmap of a filtered search (indexed by row_base + column), which survivors must also pass.  Returns
// cudaSuccess / a CUDA error (tensor-map failures: cudaErrorInvalidValue).
static inline cudaError_t launch_scan_i8(bool dense, const uint32_t* allow, const int8_t* Qh, const int8_t* Ql, int64_t ldq,
                                         const float2* qsig, const int8_t* X, int64_t pitch, int dpad, int nq, int n_cols,
                                         int K, const float* thr, unsigned long long* cand, int* count, int* overflow, int C,
                                         uint32_t row_base, int num_sms, cudaStream_t stream) {
  if (nq <= 0 || n_cols <= 0 || K <= 0) return cudaSuccess;
  CUtensorMap tmQh, tmQl, tmX;
  if (make_tmap_2d(&tmQh, Qh, 1, (uint64_t)K, (uint64_t)nq, (uint64_t)ldq, kI8BlockK, kBlockM, 128) != 0 ||
      make_tmap_2d(&tmQl, Ql, 1, (uint64_t)K, (uint64_t)nq, (uint64_t)ldq, kI8BlockK, kBlockM, 128) != 0 ||
      make_tmap_2d(&tmX, X, 1, (uint64_t)K, (uint64_t)n_cols, (uint64_t)pitch, kI8BlockK, kI8BlockN, 128) != 0)
    return cudaErrorInvalidValue;
  const int64_t num_tiles =
      static_cast<int64_t>((nq + kBlockM - 1) / kBlockM) * ((n_cols + kI8BlockN - 1) / kI8BlockN);
  const int grid = static_cast<int>(num_tiles < num_sms ? num_tiles : num_sms);
  auto launch = [&](auto dense_c, auto allow_c) {
    constexpr bool DENSE = decltype(dense_c)::value, ALLOW = decltype(allow_c)::value;
    static bool attr_set = false;  // per instantiation
    if (!attr_set) {
      cudaError_t e =
          cudaFuncSetAttribute(scan_i8_kernel<DENSE, ALLOW>, cudaFuncAttributeMaxDynamicSharedMemorySize, kI8SmemBytes);
      if (e != cudaSuccess) return e;
      attr_set = true;
    }
    scan_i8_kernel<DENSE, ALLOW><<<grid, kGemmProducerThreads + kI8Consumers, kI8SmemBytes, stream>>>(
        tmQh, tmQl, tmX, K, X, pitch, dpad, qsig, thr, cand, count, overflow, nq, n_cols, C, row_base,
        ALLOW ? allow : nullptr);
    return cudaGetLastError();
  };
  // a dense round stores every score, so the filter variant exists for threshold rounds only
  if (dense) return launch(std::true_type{}, std::false_type{});
  if (allow) return launch(std::false_type{}, std::true_type{});
  return launch(std::false_type{}, std::false_type{});
}

}  // namespace om
