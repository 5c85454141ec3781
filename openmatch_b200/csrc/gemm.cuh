// Persistent, warp-specialised wgmma GEMM core for sm_90a:   C[m, n] = sum_k A[m, k] * B[n, k]
// (both operands K-major bf16 — or IEEE half with F16 — fp32 accumulation).  It runs the encoder linear layers
// (A = activations [T, H], B = nn.Linear weight [out, in]) and the search scan rounds that the wide scan of
// scan_gemm.cuh does not take: the first round, query chunks of <= 128 queries and every round with pair_scan off
// (A = queries [nq, d], B = corpus rows [N, d]).  Its ring protocol (ring.cuh) is shared with the wide scan and the
// fused loss.
//
//   warp 0 (one lane)       TMA producer : global -> STAGES-deep smem ring (128B-swizzled boxes)
//   warps 1..3              idle (they pad the producer role to a whole warpgroup, so the consumers start at warp 4)
//   warps 4..11             two consumer warpgroups: warpgroup g issues wgmma m64 x BN x 16 for rows [64 g, 64 g + 64) of
//                           the 128-row tile, accumulating in registers; then both write their accumulators into a
//                           padded fp32 tile in shared memory and run the epilogue functor on it with the row-per-thread
//                           mapping of the functor contract below (thread <-> accumulator row, 32-column chunks)
//
// Pipelines: the STAGES-slot ring of ring.cuh (TMA <-> consumers, released one wgmma group late); the staged accumulator
// tile is handed over with two named barriers per tile.  Tile schedule: static (tile = blockIdx.x + i * gridDim.x) or
// dynamic (claimed from a global counter by the producer, published through a 4-deep smem ring).
#pragma once
#include <type_traits>

#include "ring.cuh"
#include "tmap.cuh"

namespace om {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;  // 64 bf16 = 128 B = one swizzle row
constexpr int kWgmmaK = 16;
constexpr int kGemmProducerThreads = 128;  // warpgroup 0: TMA producer + idle warps
constexpr int kGemmEpiWarps = 8;           // two consumer warpgroups

template <int BN, int STAGES>
struct GemmCfg {
  static_assert(BN == 128, "BN must be 128 (one wgmma m64n128 per consumer warpgroup)");
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kBBytes = BN * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kAccPitch = BN + 4;                    // floats per staged row: conflict-free row reads
  static constexpr int kAccOffset = STAGES * kStageBytes;     // staged fp32 accumulator tile [128][kAccPitch]
  static constexpr int kBarOffset = kAccOffset + kBlockM * kAccPitch * 4;
  static constexpr int kEpiOffset = kBarOffset + 1024;        // epilogue scratch starts 1024-B aligned (TMA store)
  static constexpr int kSmemBytes = kEpiOffset + 1024;        // + slack for 1024-B alignment of the base
  static_assert(kBarOffset % 1024 == 0, "barrier block must stay 1024-B aligned");
};

// Epilogue functor contract (all methods __device__, called by the 256 epilogue threads; thread <-> row (half)):
//   struct State;                                             per-thread, per-tile scratch
//   void begin(State&, int row, int m_blk, int n_blk) const;  once per tile, before the tile's mainloop
//   void chunk(State&, int row, int col0, const float (&v)[32]) const;   v = C[row, col0 .. col0+31]
//   void end(State&, int row) const;                           once per tile
//   static constexpr bool kPrefetch = false;                   true: prefetch(State&, row, col0) is called for the
//        thread's first chunk BEFORE the tile's mainloop, and chunk(..., int next_col0) receives the column of the
//        thread's next chunk (-1: none) so that global operands (residual) are always one chunk ahead of the math
//   __host__ __device__ static constexpr int smem_bytes(int epi_warps);            > 0: that much dynamic smem is reserved for the functor
//        and handed over through bind(State&, uint8_t* smem, int epilogue_thread_index) once per thread; the
//        State object persists across the thread's tiles and finish(State&) is called after the last one
//   end() runs right after the thread's last chunk: long-latency tails (atomics, global stores) placed there overlap the
//        next tile's mainloop
// Rows >= M and columns >= N contain zeros (TMA out-of-bounds fill) and must be masked by the functor.
// Named barrier 1 is the functors'; the core uses barrier 2.

template <int BN, bool F16>
__device__ __forceinline__ void wgmma_tile_k16(float (&acc)[BN / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (F16) wgmma_m64n128k16_f16<0, 0>(acc, da, db, accumulate);
  else wgmma_m64n128k16_bf16<0, 0>(acc, da, db, accumulate);
}

template <int BN, int STAGES, bool M_FASTEST, class Epi, bool F16>
__global__ void __launch_bounds__(kGemmProducerThreads + 32 * kGemmEpiWarps, 1)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N,
                    int K, const __grid_constant__ Epi epi, int* tile_counter) {
  using Cfg = GemmCfg<BN, STAGES>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* acc_tile = reinterpret_cast<float*>(smem + Cfg::kAccOffset);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;
  // dynamic tile scheduler (tile_counter != nullptr): the producer claims tile indices from a global
  // counter and publishes them to the consumer warps through a 4-deep smem ring
  constexpr int kSched = 4;
  uint64_t* sfull_bar = empty_bar + STAGES;
  uint64_t* sempty_bar = sfull_bar + kSched;
  volatile int* tile_ring = reinterpret_cast<volatile int*>(sempty_bar + kSched);
  uint8_t* epi_smem = smem + Cfg::kEpiOffset;  // Epi::smem_bytes() of scratch owned by the epilogue functor
  const bool dyn = tile_counter != nullptr;

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = static_cast<int>(threadIdx.x & 31);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  if (warp == 1 && lane == 0) {
    ring_init(full_bar, empty_bar, STAGES, kGemmEpiWarps);  // every consumer warp
    ring_init(sfull_bar, sempty_bar, kSched, kGemmEpiWarps);  // one lane per consumer warp
    fence_barrier_init();
  }
  __syncthreads();

  const int num_m = (M + kBlockM - 1) / kBlockM;
  const int num_n = (N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_k = (K + kBlockK - 1) / kBlockK;
  const int first_tile = static_cast<int>(blockIdx.x);
  const int tile_step = static_cast<int>(gridDim.x);

  if (warp == 0) {
    if (lane == 0) {
      // ------------------------------ TMA producer ------------------------------
      Ring<STAGES> ring;
      Ring<kSched> sched;
      int tile = first_tile;
      if (dyn) {
        tile = atomicAdd(tile_counter, 1);
        if (tile >= num_tiles) tile = -1;
      }
      while (true) {
        if (dyn) {  // publish (also the -1 sentinel) to the consumer warps
          ring_wait_free(sempty_bar, sched, 5);
          tile_ring[sched.stage] = tile;
          mbar_arrive(&sfull_bar[sched.stage]);
          sched.advance();
          if (tile < 0) break;
        } else if (tile >= num_tiles) {
          break;
        }
        // claim the next tile now; the atomic's round trip overlaps this tile's loads
        int next = dyn ? atomicAdd(tile_counter, 1) : tile + tile_step;
        const int m_blk = M_FASTEST ? tile % num_m : tile / num_n;
        const int n_blk = M_FASTEST ? tile / num_m : tile % num_n;
        for (int kb = 0; kb < num_k; ++kb) {
          uint64_t* bar = ring_acquire_tx(full_bar, empty_bar, ring, Cfg::kStageBytes, 1);
          uint8_t* sa = smem + ring.stage * Cfg::kStageBytes;
          tma_load_2d(sa, &tmA, bar, kb * kBlockK, m_blk * kBlockM);
          tma_load_2d(sa + Cfg::kABytes, &tmB, bar, kb * kBlockK, n_blk * BN);
          ring.advance();
        }
        tile = (dyn && next >= num_tiles) ? -1 : next;
      }
    }
  } else if (warp >= 4) {
    // ------------------------------ consumers: wgmma + epilogue ------------------------------
    const int et = static_cast<int>(threadIdx.x) - kGemmProducerThreads;  // 0 .. 255
    const int wg = et >> 7;                  // consumer warpgroup = rows [64 wg, +64) of the MMA tile
    const int ew = (warp - 4) & 3;           // epilogue: rows [32 ew, +32) of the tile
    const int half = (warp - 4) >> 2;        // epilogue: column group of the tile
    constexpr int kChunks = BN / 32 / 2;
    typename Epi::State st;  // lives across tiles: functors may keep work in flight from one tile to the next
    if constexpr (Epi::smem_bytes(kGemmEpiWarps) > 0) epi.bind(st, epi_smem, et);
    Ring<kSched> sched;
    Ring<STAGES> ring;
    // staging coordinates of this thread's accumulator fragment
    const int frow = 64 * wg + 16 * (warp & 3) + (lane >> 2), fcol = 2 * (lane & 3);
    for (int tile = first_tile;; tile += tile_step) {
      if (dyn) {
        mbar_wait_warp(&sfull_bar[sched.stage], sched.phase, 7);
        tile = tile_ring[sched.stage];
        __syncwarp();
        if (lane == 0) mbar_arrive(&sempty_bar[sched.stage]);
        sched.advance();
        if (tile < 0) break;
      } else if (tile >= num_tiles) {
        break;
      }
      const int m_blk = M_FASTEST ? tile % num_m : tile / num_n;
      const int n_blk = M_FASTEST ? tile / num_m : tile % num_n;
      const int row = m_blk * kBlockM + ew * 32 + lane;
      epi.begin(st, row, m_blk, n_blk);
      if constexpr (Epi::kPrefetch) epi.prefetch(st, row, n_blk * BN + half * kChunks * 32);

      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      ring_consume(
          full_bar, ring, 0, num_k, 3,
          [&](uint32_t stage, uint32_t accumulate) {
            const uint32_t a_addr = smem_u32(smem + stage * Cfg::kStageBytes) + wg * (64 * 128);
            const uint32_t b_addr = smem_u32(smem + stage * Cfg::kStageBytes + Cfg::kABytes);
#pragma unroll
            for (int k = 0; k < kBlockK / kWgmmaK; ++k)
              wgmma_tile_k16<BN, F16>(acc, wgmma_desc(a_addr + k * 32, kDescKMajorSW128),
                                      wgmma_desc(b_addr + k * 32, kDescKMajorSW128), (accumulate | k) != 0 ? 1u : 0u);
          },
          [&](uint32_t stage) {
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
          });
      wgmma_fence_regs(acc);

      // stage the accumulators: every epilogue thread has finished reading the previous tile
      named_bar_sync(2, 32 * kGemmEpiWarps);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        *reinterpret_cast<float2*>(acc_tile + frow * Cfg::kAccPitch + 8 * j + fcol) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(acc_tile + (frow + 8) * Cfg::kAccPitch + 8 * j + fcol) =
            make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
      named_bar_sync(2, 32 * kGemmEpiWarps);

      const float* my_row = acc_tile + (ew * 32 + lane) * Cfg::kAccPitch;
      const int c0 = half * kChunks;
#pragma unroll 1
      for (int c = c0; c < c0 + kChunks; ++c) {
        float v[32];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 t = *reinterpret_cast<const float4*>(my_row + c * 32 + 4 * i);
          v[4 * i] = t.x, v[4 * i + 1] = t.y, v[4 * i + 2] = t.z, v[4 * i + 3] = t.w;
        }
        const bool has_next = c + 1 < c0 + kChunks;
        if constexpr (Epi::kPrefetch)
          epi.chunk(st, row, n_blk * BN + c * 32, v, has_next ? n_blk * BN + (c + 1) * 32 : -1);
        else
          epi.chunk(st, row, n_blk * BN + c * 32, v);
      }
      epi.end(st, row);
    }
    if constexpr (Epi::smem_bytes(kGemmEpiWarps) > 0) epi.finish(st);  // drain whatever the functor still has in flight
  }

  __syncthreads();
}

// Pool of tile counters for the dynamic scheduler: launch i uses counter i % 64 (zeroed on the launching stream
// just before the kernel), so up to 64 dynamically scheduled GEMMs may be in flight.
static inline int* next_tile_counter(cudaStream_t stream) {
  static int* pool = nullptr;
  static unsigned next = 0;
  if (!pool && cudaMalloc(&pool, 64 * sizeof(int)) != cudaSuccess) return nullptr;
  int* c = pool + (next++ & 63u);
  if (cudaMemsetAsync(c, 0, sizeof(int), stream) != cudaSuccess) return nullptr;
  return c;
}

// Host launcher.  A: [M, K] row pitch lda elements; B: [N, K] row pitch ldb elements (bf16, or IEEE half with F16).
// Returns cudaSuccess / a CUDA error; tensor-map failures map to cudaErrorInvalidValue.
// dynamic_sched: claim tiles from a global counter instead of the static blockIdx + i * gridDim order, which keeps all
// CTAs on neighbouring tiles (with the static order CTAs drift apart over thousands of tiles and stop sharing operand
// tiles in L2).
template <int BN, int STAGES, bool M_FASTEST, class Epi, bool F16 = false>
static inline cudaError_t launch_gemm(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K,
                                      const Epi& epi, int num_sms, cudaStream_t stream, bool dynamic_sched = false) {
  using Cfg = GemmCfg<BN, STAGES>;
  if (M <= 0 || N <= 0 || K <= 0) return cudaSuccess;
  CUtensorMap tmA, tmB;
  if (make_tmap_bf16_2d(&tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, kBlockK, kBlockM) != 0)
    return cudaErrorInvalidValue;
  if (make_tmap_bf16_2d(&tmB, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb * 2, kBlockK, BN) != 0)
    return cudaErrorInvalidValue;
  auto kern = gemm_bf16_tn_kernel<BN, STAGES, M_FASTEST, Epi, F16>;
  const int smem_bytes = Cfg::kSmemBytes + Epi::smem_bytes(kGemmEpiWarps);
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const int num_tiles = ((M + kBlockM - 1) / kBlockM) * ((N + BN - 1) / BN);
  const int threads = kGemmProducerThreads + 32 * kGemmEpiWarps;
  const int grid = num_tiles < num_sms ? num_tiles : num_sms;
  int* counter = nullptr;
  if (dynamic_sched) {
    counter = next_tile_counter(stream);
    if (!counter) return cudaErrorMemoryAllocation;
  }
  kern<<<grid, threads, smem_bytes, stream>>>(tmA, tmB, M, N, K, epi, counter);
  return cudaGetLastError();
}

}  // namespace om
