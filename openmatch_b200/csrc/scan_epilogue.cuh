// Fused top-k filter epilogue of the search scan GEMM + candidate key encoding.
#pragma once
#include <string.h>

#include "gemm.cuh"

namespace om {

// ---------------------------------------------------------------------------------------------------
// candidate keys: descending unsigned order == (score descending, row ascending)
// ---------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t f32_orderable(float s) {
  s = s + 0.0f;  // -0 -> +0
#ifdef __CUDA_ARCH__
  uint32_t u = __float_as_uint(s);
#else
  uint32_t u;
  memcpy(&u, &s, 4);
#endif
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float f32_from_orderable(uint32_t u) {
  u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float s;
  memcpy(&s, &u, 4);
  return s;
#endif
}
__host__ __device__ __forceinline__ unsigned long long make_key(float s, uint32_t row) {
  return (static_cast<unsigned long long>(f32_orderable(s)) << 32) | static_cast<unsigned long long>(0xffffffffu - row);
}
__host__ __device__ __forceinline__ uint32_t key_row(unsigned long long k) {
  return 0xffffffffu - static_cast<uint32_t>(k & 0xffffffffull);
}
__host__ __device__ __forceinline__ float key_score(unsigned long long k) {
  return f32_from_orderable(static_cast<uint32_t>(k >> 32));
}

// ---------------------------------------------------------------------------------------------------
// fused scan epilogue
// ---------------------------------------------------------------------------------------------------
// Filter shape: one 32-column max (3-input max tree), then a 32-bit mask and a 31-SEL select tree per survivor.
template <bool DENSE, int EPI_THREADS = 256>
struct EpiScan {
  const float* thr;          // [nq] strict lower bound per query
  unsigned long long* cand;  // [nq, C]
  int* count;                // [nq]
  int* overflow;             // single flag
  int nq, n_cols, C;
  uint32_t row_base;  // corpus row of column 0 of this round
  // DENSE: first round, every score is stored at position = column (no threshold yet)
  // Pass 0: a thread compares its 32-column chunks against its query's threshold and parks the rare
  // survivors (up to kStash per tile) in a private shared-memory stash.  The accumulator buffer is then
  // released to the MMA warp, and end() ISSUES one atomicAdd that reserves the survivors' slots in the
  // query's candidate list; the atomic's result is consumed only at the end of the thread's NEXT tile
  // (double-buffered stash), so its L2 round trip is hidden behind a whole tile of work.
  // Overflow path (dense early rounds): if some lane of the warp found more than kStash survivors, the warp
  // sweeps the tile a second time (pass 1) and those lanes append the excess synchronously.
  // Everything is force-inlined and State never has its address taken, so it lives in registers.
  static constexpr int kPasses = 2;
  static constexpr bool kPrefetch = false;
  static constexpr int kStash = 8;                      // survivors a thread can park per tile
  static constexpr int kEpiThreads = EPI_THREADS;       // 8 epilogue warps in the product
  __host__ __device__ static constexpr int smem_bytes(int) { return DENSE ? 0 : 2 * kStash * kEpiThreads * 8; }
  struct State {
    float t;
    int k, n, skip, pos2, tid, buf;
    unsigned long long* stash;     // [2][kStash][kEpiThreads], this thread owns column `tid` of buffer `buf`
    int p_n, p_pos, p_row, p_buf;  // reservation in flight: p_n keys of buffer p_buf go to row p_row at p_pos
  };
  __device__ __forceinline__ void bind(State& s, uint8_t* smem, int epi_tid) const {
    s.stash = reinterpret_cast<unsigned long long*>(smem);
    s.tid = epi_tid;
    s.buf = 0;
    s.p_n = 0;
  }
  __device__ __forceinline__ void finish(State& s) const { drain(s); }
  __device__ __forceinline__ void begin(State& s, int row, int, int) const {
    s.t = (row < nq && !DENSE) ? thr[row] : __int_as_float(0x7f800000);
    s.k = 0;
    s.n = 0;
    if constexpr (DENSE) {  // no stash / reservation in the dense round
      s.p_n = 0;
      s.buf = 0;
    }
  }
  __device__ __forceinline__ unsigned long long* slot(const State& s, int buf, int j) const {
    return s.stash + (static_cast<size_t>(buf) * kStash + j) * kEpiThreads + s.tid;
  }
  __device__ __forceinline__ void drain(State& s) const {
    if (s.p_n > 0) {
      unsigned long long* mine = cand + static_cast<size_t>(s.p_row) * C;
      for (int j = 0; j < s.p_n; ++j)
        if (s.p_pos + j < C) mine[s.p_pos + j] = *slot(s, s.p_buf, j);
      if (s.p_pos + s.p_n > C) *overflow = 1;
      s.p_n = 0;
    }
  }
  __device__ __forceinline__ bool need_pass(const State& s, int) const {
    if constexpr (DENSE) return false;
    return __any_sync(0xffffffffu, s.n > kStash);
  }
  __device__ __forceinline__ void between(State& s, int row) const {
    s.skip = kStash;
    s.pos2 = C;
    if (s.n > kStash) {
      s.pos2 = atomicAdd(count + row, s.n - kStash);
      if (s.pos2 + (s.n - kStash) > C) *overflow = 1;
    }
  }
  __device__ __forceinline__ void end(State& s, int row) const {
    if constexpr (DENSE) return;
    drain(s);  // last tile's survivors: their atomic was issued a whole tile ago
    if (s.k > 0) {
      s.p_pos = atomicAdd(count + row, s.k);  // result first used by the next drain()
      s.p_n = s.k;
      s.p_row = row;
      s.p_buf = s.buf;
      s.buf ^= 1;
    }
  }
  __device__ __forceinline__ void chunk(State& s, int row, int col0, const float (&v)[32], int pass) const {
    if (row >= nq || col0 >= n_cols) return;
    unsigned long long* mine = cand + static_cast<size_t>(row) * C;
    if constexpr (DENSE) {
      if (col0 + 32 <= n_cols) {
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          ulonglong2 kk;
          kk.x = make_key(v[i], row_base + col0 + i);
          kk.y = make_key(v[i + 1], row_base + col0 + i + 1);
          *reinterpret_cast<ulonglong2*>(mine + col0 + i) = kk;
        }
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (col0 + i < n_cols) mine[col0 + i] = make_key(v[i], row_base + col0 + i);
      }
      return;
    }
    const float t = s.t;
    const int lim = n_cols - col0;  // columns >= lim are out of range (only in the last tile)
    if (pass == 1 && s.n <= kStash) return;
    float mx = v[0];
#pragma unroll
    for (int i = 1; i < 32; ++i) mx = fmaxf(mx, v[i]);
    if (!(mx > t)) return;  // common case: nothing in this chunk beats the threshold
    // Survivor path.  Kept deliberately COMPACT (a bit mask + a short loop with a select tree instead of 32
    // unrolled predicated blocks): it is executed rarely per warp, so its instructions are cold in the
    // instruction cache and every extra cache line costs hundreds of cycles (~1000 cycles per
    // survivor with the unrolled form).
    uint32_t mask = 0;
#pragma unroll
    for (int i = 0; i < 32; ++i) mask |= (v[i] > t ? 1u : 0u) << i;
    if (lim < 32) mask &= (1u << lim) - 1u;
#pragma unroll 1
    while (mask) {
      const int i = __ffs(mask) - 1;
      mask &= mask - 1;
      const unsigned long long key = make_key(pick32(v, i), row_base + col0 + i);
      if (pass == 0) {
        if (s.k < kStash) {
          *slot(s, s.buf, s.k) = key;
          ++s.k;
        }
        ++s.n;
      } else if (s.skip > 0) {
        --s.skip;
      } else {
        if (s.pos2 < C) mine[s.pos2] = key;
        ++s.pos2;
      }
    }
  }
  // v[i] for a run-time i without local memory: 5-level select tree (31 SEL)
  __device__ __forceinline__ static float pick32(const float (&v)[32], int i) {
    float a[16], b[8], c[4], d[2];
#pragma unroll
    for (int j = 0; j < 16; ++j) a[j] = (i & 1) ? v[2 * j + 1] : v[2 * j];
#pragma unroll
    for (int j = 0; j < 8; ++j) b[j] = (i & 2) ? a[2 * j + 1] : a[2 * j];
#pragma unroll
    for (int j = 0; j < 4; ++j) c[j] = (i & 4) ? b[2 * j + 1] : b[2 * j];
#pragma unroll
    for (int j = 0; j < 2; ++j) d[j] = (i & 8) ? c[2 * j + 1] : c[2 * j];
    return (i & 16) ? d[1] : d[0];
  }
};

}  // namespace om
