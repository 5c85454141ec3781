// Candidate key encoding and the top-k filter of the search scans: the survivor protocol, the fragment filter of the
// wide and int8 scans and the fused epilogue of the GEMM core and its launcher.
#pragma once
#include <cuda_fp16.h>
#include <string.h>

#include <type_traits>

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
// the survivor protocol of every scan filter
// ---------------------------------------------------------------------------------------------------
// A score survives a round when it beats its query's strict threshold.  A survivor is parked in a per-thread stash in
// shared memory (slot j of thread t at stash[j * kStashThreads + t]); at the end of a tile ONE atomicAdd reserves the
// parked keys' slots in the query's candidate list, and its result is consumed a tile later (double-buffered stash), when
// drain_stash() copies them, so the atomic's L2 round trip hides behind a whole tile of work.  Survivors beyond the stash
// (dense early rounds) are reserved by a synchronous atomicAdd and stored at once.  A list that would grow beyond C sets
// *overflow, which voids the round's certificate.
//
// The survivor path is kept deliberately COMPACT (a bit mask + a short loop with a select tree instead of unrolled
// predicated blocks): it runs rarely per warp, so its instructions are cold in the instruction cache and every extra
// cache line costs hundreds of cycles (~1000 cycles per survivor with a 32-way unrolled form).
constexpr int kStashThreads = 32 * kGemmEpiWarps;  // filter threads of every scan CTA: two consumer warpgroups

template <int N>
using SurvivorMask = std::conditional_t<N == 64, unsigned long long, uint32_t>;
__device__ __forceinline__ int mask_popc(uint32_t m) { return __popc(m); }
__device__ __forceinline__ int mask_popc(unsigned long long m) { return __popcll(m); }
__device__ __forceinline__ int mask_ffs(uint32_t m) { return __ffs(m); }
__device__ __forceinline__ int mask_ffs(unsigned long long m) { return __ffsll(static_cast<long long>(m)); }

// v[i] for a run-time i < N without local memory: a select tree of log2(N) levels (N - 1 SEL)
template <int N, int BIT = 1>
__device__ __forceinline__ float pick(const float (&v)[N], int i) {
  if constexpr (N == 1) {
    return v[0];
  } else {
    float a[N / 2];
#pragma unroll
    for (int j = 0; j < N / 2; ++j) a[j] = (i & BIT) ? v[2 * j + 1] : v[2 * j];
    return pick<N / 2, 2 * BIT>(a, i);
  }
}

// Bit i set where v[i] > t; decided by one N-value max, which rejects the values in the common case.  The max takes
// pairs, so its dependency chain is N / 2 long rather than N - 1 (a 63-deep chain per row made the C2 scan 2 % slower,
// H100 SXM at 700 W).
template <int N>
__device__ __forceinline__ SurvivorMask<N> survivors(const float (&v)[N], float t) {
  float mx = fmaxf(v[0], v[1]);
#pragma unroll
  for (int i = 2; i < N; i += 2) mx = fmaxf(mx, fmaxf(v[i], v[i + 1]));
  if (!(mx > t)) return 0;
  SurvivorMask<N> mask = 0;
#pragma unroll
  for (int w = 0; w < N / 32; ++w) {  // in 32-bit words: a 64-bit shift per bit would double the cold path
    uint32_t m = 0;
#pragma unroll
    for (int i = 0; i < 32; ++i) m |= (v[32 * w + i] > t ? 1u : 0u) << i;
    mask |= static_cast<SurvivorMask<N>>(m) << (32 * w);
  }
  return mask;
}

// Parks the survivors `mask` of v (bit i: corpus column col(i) of the round) in stash slots k, k + 1, ... < S of this
// thread (slot j at stash[j * kStashThreads]) and stores the excess into row's candidate list.  Returns the number of
// slots now filled.
template <int S, int N, class Col>
__device__ __forceinline__ int park(const float (&v)[N], SurvivorMask<N> mask, Col col, int k, unsigned long long* stash,
                                    int row, unsigned long long* cand, int* count, int* overflow, int C,
                                    uint32_t row_base) {
  const int n = mask_popc(mask);
  int pos = 0;
  if (k + n > S) {  // more than the stash holds: reserve the excess synchronously
    pos = atomicAdd(count + row, k + n - S);
    if (pos + (k + n - S) > C) *overflow = 1;
  }
  unsigned long long* mine = cand + static_cast<size_t>(row) * C;
  int idx = k;
#pragma unroll 1
  while (mask) {
    const int i = mask_ffs(mask) - 1;
    mask &= mask - 1;
    const unsigned long long key = make_key(pick(v, i), row_base + static_cast<uint32_t>(col(i)));
    if (idx < S)
      stash[idx * kStashThreads] = key;
    else if (pos + idx - S < C)
      mine[pos + idx - S] = key;
    ++idx;
  }
  return idx < S ? idx : S;
}

// Filtered search: the bits of mask whose corpus row row_base + col(i) the allowed-row bitmap keeps (bit r & 31 of word
// r >> 5 set = row r may be returned).  Called on the survivor path only, after the max test, so a round reads the bitmap
// for the few rows that beat their query's threshold; the rows of masked-out columns are never read.
template <int N, class Col>
__device__ __forceinline__ SurvivorMask<N> allowed(SurvivorMask<N> mask, const uint32_t* allow, uint32_t row_base, Col col) {
  SurvivorMask<N> keep = 0;
#pragma unroll 1
  while (mask) {
    const int i = mask_ffs(mask) - 1;
    const SurvivorMask<N> bit = static_cast<SurvivorMask<N>>(1) << i;
    mask &= ~bit;
    const uint32_t r = row_base + static_cast<uint32_t>(col(i));
    if ((__ldg(allow + (r >> 5)) >> (r & 31)) & 1u) keep |= bit;
  }
  return keep;
}

// Copies n parked keys (slot j at stash[j * kStashThreads]) to list[pos ...], whose slots an atomicAdd reserved.
__device__ __forceinline__ void drain_stash(const unsigned long long* stash, int n, unsigned long long* list, int pos,
                                            int C, int* overflow) {
  for (int j = 0; j < n; ++j)
    if (pos + j < C) list[pos + j] = stash[j * kStashThreads];
  if (n > 0 && pos + n > C) *overflow = 1;
}

// ---------------------------------------------------------------------------------------------------
// top-k filter on wgmma accumulator fragments (scan_wide_kernel: COLS = 64 of an m64n256 fp32 tile; scan_i8_kernel:
// COLS = 32 of its m64n128 combined scores)
// ---------------------------------------------------------------------------------------------------
// A thread owns fragment rows l/4 and l/4 + 8 (H = 0, 1) of its warp's 16 x COLS columns of the 4 COLS-column tile:
// bit i of a row's survivor mask is column 8 (i >> 1) + 2 (l % 4) + (i & 1) of the tile, value acc[4 (i >> 1) + 2 H + (i & 1)].
// The 4 lanes of a quad share both rows and reserve their parked survivors with one atomicAdd per row (shuffle prefix for
// the lane offsets).  Stash: [buffer][row half][slot][thread] keys.
constexpr int kFragStash = 4;  // survivors a thread parks per row and tile
constexpr int kFragStashBytes = 2 * 2 * kFragStash * kStashThreads * 8;

// ALLOW: filtered search, survivors are also masked by the allowed-row bitmap `allow` (see allowed()).
template <int COLS, bool ALLOW = false>
struct FragFilter {
  unsigned long long* stash;  // this thread's slot 0 of buffer 0, row half 0
  unsigned long long* cand;
  int* count;
  int* overflow;
  int C;
  uint32_t row_base;
  int lane;
  const uint32_t* allow = nullptr;
  int buf = 0;
  // reservation in flight: p_n[h] keys of stash buffer p_buf go to query p_row + 8 h at (quad leader's p_pos[h]) + p_excl[h]
  int p_n[2] = {0, 0}, p_excl[2] = {0, 0}, p_pos[2] = {0, 0}, p_row = 0, p_buf = 0;

  __device__ __forceinline__ int col(int i) const { return 8 * (i >> 1) + 2 * (lane & 3) + (i & 1); }

  // Filter of fragment row H: returns the number of survivors parked in the stash (<= kFragStash).
  template <int H>
  __device__ __forceinline__ int filter_row(const float (&acc)[2 * COLS], float t, int row, int col0, int lim,
                                            unsigned long long* sb) const {
    float v[COLS];
#pragma unroll
    for (int i = 0; i < COLS; ++i) v[i] = acc[4 * (i >> 1) + 2 * H + (i & 1)];
    SurvivorMask<COLS> mask = survivors(v, t);
    if (!mask) return 0;
    if (lim < 4 * COLS) {  // last corpus tile: columns >= lim are padding, and a zero can beat a negative threshold
#pragma unroll 1
      for (int i = 0; i < COLS; ++i)
        if (col(i) >= lim) mask &= ~(static_cast<SurvivorMask<COLS>>(1) << i);
    }
    if constexpr (ALLOW) mask = allowed<COLS>(mask, allow, row_base, [&](int i) { return col0 + col(i); });
    return park<kFragStash>(v, mask, [&](int i) { return col0 + col(i); }, 0, sb, row, cand, count, overflow, C,
                            row_base);
  }

  // The previous tile's survivors: their atomic was issued a whole tile ago.
  __device__ __forceinline__ void drain() {
    if (!__any_sync(0xffffffffu, (p_n[0] | p_n[1]) != 0)) return;
    const unsigned long long* s = stash + p_buf * (2 * kFragStash * kStashThreads);
#pragma unroll
    for (int h = 0; h < 2; ++h)
      drain_stash(s + h * kFragStash * kStashThreads, p_n[h], cand + static_cast<size_t>(p_row + 8 * h) * C,
                  __shfl_sync(0xffffffffu, p_pos[h], lane & ~3) + p_excl[h], C, overflow);
    p_n[0] = p_n[1] = 0;
  }

  // One tile: rows row0 and row0 + 8 (thresholds t0, t1) x the tile's columns from col0; columns >= n_cols are padding.
  __device__ __forceinline__ void tile(const float (&acc)[2 * COLS], float t0, float t1, int row0, int col0, int n_cols) {
    drain();
    const int lim = n_cols - col0;  // <= 0: the whole tile lies past n_cols and every column is masked
    unsigned long long* sb = stash + buf * (2 * kFragStash * kStashThreads);
    const int k[2] = {filter_row<0>(acc, t0, row0, col0, lim, sb),
                      filter_row<1>(acc, t1, row0 + 8, col0, lim, sb + kFragStash * kStashThreads)};
    if (!__any_sync(0xffffffffu, (k[0] | k[1]) != 0)) return;
    // exclusive prefix per lane over its quad, one atomic per quad and row, whose result the next drain() consumes
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int x = k[h];
      int y = __shfl_up_sync(0xffffffffu, x, 1, 4);
      if ((lane & 3) >= 1) x += y;
      y = __shfl_up_sync(0xffffffffu, x, 2, 4);
      if ((lane & 3) >= 2) x += y;
      const int n = __shfl_sync(0xffffffffu, x, lane | 3);
      if ((lane & 3) == 0 && n > 0) p_pos[h] = atomicAdd(count + row0 + 8 * h, n);
      p_n[h] = k[h];
      p_excl[h] = x - k[h];
    }
    p_row = row0;
    p_buf = buf;
    buf ^= 1;
  }
};

// ---------------------------------------------------------------------------------------------------
// fused scan epilogue of the GEMM core (gemm.cuh): one thread per query row, 32-column chunks
// ---------------------------------------------------------------------------------------------------
// DENSE: first round, every score is stored at position = column (no threshold yet).  Otherwise the survivor protocol
// above with a stash of kStash keys per thread and tile; the thread owns a whole row, so it reserves its own slots.
// Everything is force-inlined and State never has its address taken, so it lives in registers.
// ALLOW (threshold rounds only): filtered search, survivors are also masked by the allowed-row bitmap of the base.  The
// base is empty otherwise, so the functor's layout, and the kernel parameters behind it, stay those of the plain scan.
template <bool ALLOW>
struct ScanAllow {};
template <>
struct ScanAllow<true> {
  const uint32_t* allow;  // allowed-row bitmap over the rows of the index shard
};
template <bool DENSE, bool ALLOW = false>
struct EpiScan : ScanAllow<ALLOW> {
  static_assert(!(DENSE && ALLOW), "a filtered first round runs as a threshold round at -inf");
  const float* thr;          // [nq] strict lower bound per query
  unsigned long long* cand;  // [nq, C]
  int* count;                // [nq]
  int* overflow;             // single flag
  int nq, n_cols, C;
  uint32_t row_base;  // corpus row of column 0 of this round
  static constexpr bool kPrefetch = false;
  static constexpr int kStash = 8;  // survivors a thread can park per tile
  __host__ __device__ static constexpr int smem_bytes(int) { return DENSE ? 0 : 2 * kStash * kStashThreads * 8; }
  struct State {
    float t;
    int k, tid, buf;
    unsigned long long* stash;     // [2][kStash][kStashThreads], this thread owns column `tid` of buffer `buf`
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
    if constexpr (DENSE) {  // no stash / reservation in the dense round
      s.p_n = 0;
      s.buf = 0;
    }
  }
  __device__ __forceinline__ unsigned long long* slot0(const State& s, int buf) const {
    return s.stash + static_cast<size_t>(buf) * kStash * kStashThreads + s.tid;
  }
  __device__ __forceinline__ void drain(State& s) const {
    if (s.p_n > 0) {
      drain_stash(slot0(s, s.p_buf), s.p_n, cand + static_cast<size_t>(s.p_row) * C, s.p_pos, C, overflow);
      s.p_n = 0;
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
  __device__ __forceinline__ void chunk(State& s, int row, int col0, const float (&v)[32]) const {
    if (row >= nq || col0 >= n_cols) return;
    if constexpr (DENSE) {
      unsigned long long* mine = cand + static_cast<size_t>(row) * C;
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
    uint32_t mask = survivors(v, s.t);
    if (!mask) return;  // common case: nothing in this chunk beats the threshold
    const int lim = n_cols - col0;  // columns >= lim are out of range (only in the last tile)
    if (lim < 32) mask &= (1u << lim) - 1u;
    if constexpr (ALLOW) mask = allowed<32>(mask, this->allow, row_base + col0, [](int i) { return i; });
    s.k = park<kStash>(v, mask, [&](int i) { return col0 + i; }, s.k, slot0(s, s.buf), row, cand, count, overflow, C,
                       row_base);
  }
};

// Host launcher of the scan on the GEMM core (128-row corpus tiles from a dynamic tile queue).  Q: [nq, K] fp16 queries,
// row pitch ldq elements; X: [n_cols, K] fp16 corpus rows, row pitch ldx.  dense: every score goes to cand[q * C + column],
// and allow is not read; otherwise survivors (score > thr[q]) are appended as make_key(score, row_base + column).  allow:
// nullptr, or the allowed-row bitmap of a filtered search, which survivors must also pass.
static inline cudaError_t launch_scan_core(bool dense, const uint32_t* allow, const __half* Q, int64_t ldq, const __half* X,
                                           int64_t ldx, int nq, int n_cols, int K, const float* thr,
                                           unsigned long long* cand, int* count, int* overflow, int C, uint32_t row_base,
                                           int num_sms, cudaStream_t stream) {
  auto launch = [&](const auto& epi) {
    return launch_gemm<128, 3, true, std::decay_t<decltype(epi)>, true>(Q, ldq, X, ldx, nq, n_cols, K, epi, num_sms, stream,
                                                                       /*dynamic_sched=*/true);
  };
  if (dense) return launch(EpiScan<true>{{}, thr, cand, count, overflow, nq, n_cols, C, row_base});
  if (allow) return launch(EpiScan<false, true>{{allow}, thr, cand, count, overflow, nq, n_cols, C, row_base});
  return launch(EpiScan<false>{{}, thr, cand, count, overflow, nq, n_cols, C, row_base});
}

}  // namespace om
