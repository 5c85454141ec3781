// In-batch-negatives contrastive loss, forward + backward, as ONE persistent wgmma kernel, replacing
//   logits = x @ y.T ; F.cross_entropy(logits, target)          src/openmatch/loss.py:7-15
//   scores = q_reps @ p_reps.T ; CrossEntropyLoss(mean)          src/openmatch/modeling/dense_retrieval_model.py:113-122
// and their autograd backward (~8 PyTorch launches forward, as many backward).
//
// loss_fused_kernel: cooperative grid (<= 1 CTA per SM), phases separated by grid barriers; every GEMM runs on the
// ring of ring.cuh (TMA -> 4-stage smem ring -> one consumer warpgroup issuing wgmma 2 x (64x128x16), fp32
// accumulators in registers -> stores), with the ring position carried from phase to phase:
//   PREP    fp32 (or unaligned) inputs only: Q, P -> bf16 row-major copies.  Aligned bf16 inputs are read in place.
//   LOGITS  S = Q P^T, fp32 [nq, np]                      (A = Q, B = P, both K-major)
//   SOFTMAX one warp per query row, the row in registers: log-sum-exp (fp32), loss_i = lse_i - s_i,t_i,
//           G = w (softmax - onehot) -> bf16 [nq, np]; after the barrier the last CTA reduces the row losses in a
//           fixed order (deterministic)
//   GRADS   dQ = G P   (A = G K-major,            B = P as stored = MN-major, K = np split into slices)
//           dP = G^T Q (A = G as stored = MN-major, B = Q as stored = MN-major)
// The backward GEMMs read their operands through MN-major shared-memory descriptors, so no transposed copy of Q, P
// or G is ever written.
#include <algorithm>
#include <cstdlib>
#include <type_traits>

#include "common.h"
#include "gemm.cuh"

namespace om {

constexpr int kLossBN = 128, kLossStages = 4, kLossThreads = 256;
struct LossCfg {
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kLossBN * kBlockK * 2;
  static constexpr int kBarOffset = kLossStages * kStageBytes;
  static constexpr int kSmemBytes = kBarOffset + 1024 + 1024;  // barriers + slack for 1024-B alignment of the base
};

// [0] logits (Q, P)   [1] dQ (G, P)   [2] dP (G, Q); 128-B swizzle; K-major operands: boxes {64 k, 128 rows},
// MN-major operands: boxes {64 mn, 64 k} (two per stage)
struct LossMaps {
  CUtensorMap a[3], b[3];
};

struct LossArgs {
  const void* Q;
  const void* P;
  int is_bf16;
  int nq, np, d, dpad, npp;
  int direct;  // Q / P are bf16, 16-byte aligned rows: no PREP phase, the tensor maps point at them
  const int64_t* target;
  float w, loss_scale;
  __nv_bfloat16 *qb, *pb, *G;
  float *S, *row_loss, *loss_out, *dQ, *dP;
  int* bad_target;
  unsigned* grid_bar;
  // split-K of the dQ GEMM (its K = np is the long dimension and it has only nq/128 x d/128 output tiles)
  int dq_split;          // number of K slices per dQ tile (1 = off)
  float* dq_part;        // [dq_split, nq, d] partial tiles
  unsigned* dq_sem;      // [tiles, 4] arrival counters (self-resetting)
  int sm_fast;           // SOFTMAX keeps a row in registers (np % 4 == 0, np <= kSoftmaxMaxCols)
  unsigned long long* ts;  // [8] phase timestamps (globaltimer) of the last call, diagnostics
};

constexpr int kSoftmaxMaxCols = 4096;

#ifdef OM_LOSS_TRACE  // measurement builds only: per-CTA event times of the gradient GEMMs
__device__ unsigned long long om_loss_trace[160][64];
#define OM_TRACE(slot) \
  do { if (static_cast<unsigned>(slot) < 64u) om_loss_trace[blockIdx.x][(slot)] = global_timer_ns(); } while (0)
#else
#define OM_TRACE(slot) do { } while (0)
#endif

__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Self-resetting grid barrier (the cooperative-groups scheme): CTA 0 adds 0x80000000 - (G - 1), the others 1, so
// the top bit flips exactly when all G have arrived and the low bits return to zero.  Bounded spin: a lost CTA
// raises the fault word instead of hanging the GPU.
__device__ __forceinline__ void grid_sync(unsigned* bar) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned inc = blockIdx.x == 0 ? 0x80000000u - (gridDim.x - 1u) : 1u;
    __threadfence();
    const unsigned old = atomicAdd(bar, inc);
    const long long t0 = clock64();
    while (((old ^ *reinterpret_cast<volatile unsigned*>(bar)) & 0x80000000u) == 0u) {
      if (clock64() - t0 > OM_WAIT_TIMEOUT_CYCLES) {
        atomicCAS(&om_dev_fault, 0u, 0x80ee0000u | (blockIdx.x & 0xffffu));
        break;
      }
    }
    __threadfence();
  }
  __syncthreads();
}

constexpr int kLossSmemBytes = LossCfg::kSmemBytes;

struct LossSmem {
  uint8_t* ring;
  uint64_t *full_bar, *empty_bar;
};
using LossRing = Ring<kLossStages>;  // per-thread ring position, carried across the GEMM phases

// MN-major operand tile in shared memory: two TMA boxes {64 mn, 64 k} back to back.  Inside a box the 64 mn elements
// of one k are a 128-byte row, 8 such rows form a 1024-byte swizzle atom (stride between 8-k groups, SBO = 1024 B);
// the second 64 mn elements live in the second box (LBO = 8192 B).  One wgmma (K = 16) consumes two 8-k groups, so the
// descriptor start address advances by 2048 B per instruction.
constexpr uint32_t kMnBoxBytes = 64 * kBlockK * 2;
constexpr int kMaxSplit = 4;  // K slices per output tile of the split GEMM
constexpr uint64_t kDescMNMajorSW128 = wgmma_desc_base(kMnBoxBytes, 1024);

// 64 x 128 x 16 step of the 64-row half `h` of the tile; A_MN / B_MN: operand stored MN-major
template <bool A_MN, bool B_MN>
__device__ __forceinline__ void loss_mma_k16(float (&acc)[64], uint32_t a_addr, uint32_t b_addr, int h, int k,
                                             uint32_t accumulate) {
  // K-major: the half is 64 rows further (8 KB), a K step 32 B; MN-major: the half is the second box (8 KB), a K step 2 KB
  const uint64_t da = wgmma_desc(a_addr + h * 8192 + k * (A_MN ? 2048 : 32), A_MN ? kDescMNMajorSW128 : kDescKMajorSW128);
  const uint64_t db = wgmma_desc(b_addr + k * (B_MN ? 2048 : 32), B_MN ? kDescMNMajorSW128 : kDescKMajorSW128);
  wgmma_m64n128k16_bf16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, accumulate);
}

// One GEMM of the kernel: C[M, N] fp32 (row pitch ldc) = A B^T with A [M, K], B [N, K]; a_mn / b_mn say that the
// operand is stored [K, M] / [K, N] (MN-major) instead of K-major.  S > 1 splits K into S slices (see gemm_phase).
struct GemmDesc {
  const CUtensorMap *tmA, *tmB;
  int M, N, K;
  float* C;
  int ldc;
  bool a_mn, b_mn;
  int S;
  float* part;
  unsigned* sem;
  int tb;  // first trace slot (measurement builds), negative: not traced
};

// This CTA's share of the work items of one GEMM; `rot` rotates the item -> CTA assignment so that back-to-back
// GEMMs start on different CTAs.  An item is a 128 x 128 tile, or with S > 1 one of S K-slices of a tile: every slice
// stores its partial tile to part[s], and the slice that arrives last at the tile's counter (per epilogue warp:
// 32 rows) adds the S partials in the fixed order s = 0 .. S-1 into C, so the result does not depend on which slice
// finished last.
__device__ __forceinline__ void gemm_phase(const GemmDesc& g, int rot, const LossSmem& sm, LossRing& ring, int warp,
                                           int lane) {
  const int M = g.M, N = g.N, S = g.S, ldc = g.ldc;
  const int num_n = (N + kLossBN - 1) / kLossBN;
  const int num_k = (g.K + kBlockK - 1) / kBlockK;
  const int kper = (num_k + S - 1) / S;  // the host chose S such that (S - 1) * kper < num_k
  const int num_items = ((M + kBlockM - 1) / kBlockM) * num_n * S;
  const int G = static_cast<int>(gridDim.x);
  const int first = (static_cast<int>(blockIdx.x) + G - rot % G) % G;
  if (warp == 0) {
    if (lane == 0) {  // TMA producer
      fence_proxy_async_global();  // operands were written with ordinary stores by other CTAs before the barrier
      int tslot = g.tb;
      for (int item = first; item < num_items; item += G, tslot += 8) {
        const int tile = item / S, ks = item - tile * S;
        const int m0 = (tile / num_n) * kBlockM, n0 = (tile % num_n) * kLossBN;
        const int kb_end = min(num_k, (ks + 1) * kper);
        OM_TRACE(tslot);
        for (int kb = ks * kper; kb < kb_end; ++kb) {
          uint64_t* bar = ring_acquire_tx(sm.full_bar, sm.empty_bar, ring, LossCfg::kStageBytes, 1);
          uint8_t* sa = sm.ring + ring.stage * LossCfg::kStageBytes;
          uint8_t* sb = sa + LossCfg::kABytes;
          if (!g.a_mn) {
            tma_load_2d(sa, g.tmA, bar, kb * kBlockK, m0);
          } else {
            tma_load_2d(sa, g.tmA, bar, m0, kb * kBlockK);
            tma_load_2d(sa + kMnBoxBytes, g.tmA, bar, m0 + 64, kb * kBlockK);
          }
          if (!g.b_mn) {
            tma_load_2d(sb, g.tmB, bar, kb * kBlockK, n0);
          } else {
            tma_load_2d(sb, g.tmB, bar, n0, kb * kBlockK);
            tma_load_2d(sb + kMnBoxBytes, g.tmB, bar, n0 + 64, kb * kBlockK);
          }
          ring.advance();
        }
      }
    }
  } else if (warp >= 4) {  // consumer warpgroup: wgmma for both 64-row halves of the tile, then stores
    const int ew = warp & 3;
    int tslot = (ew == 0 && lane == 0) ? g.tb : -1000;
    for (int item = first; item < num_items; item += G, tslot += 8) {
      const int tile = item / S, ks = item - tile * S;
      const int m_blk = tile / num_n, n_blk = tile % num_n;
      const int kb_begin = ks * kper, kb_end = min(num_k, kb_begin + kper);
      float* Cw = S > 1 ? g.part + static_cast<int64_t>(ks) * M * ldc : g.C;
      float acc[2][64];
      ring_consume(
          sm.full_bar, ring, kb_begin, kb_end, 3,
          [&](uint32_t stage, uint32_t accumulate) {
            if (!accumulate) OM_TRACE(tslot + 1);
            const uint32_t a_addr = smem_u32(sm.ring + stage * LossCfg::kStageBytes);
            const uint32_t b_addr = a_addr + LossCfg::kABytes;
            // operand majors are immediates of the instruction: one fully unrolled k block per layout
            auto mma = [&](auto a_mn, auto b_mn) {
#pragma unroll
              for (int k = 0; k < kBlockK / kWgmmaK; ++k) {
#pragma unroll
                for (int h = 0; h < 2; ++h)
                  loss_mma_k16<decltype(a_mn)::value, decltype(b_mn)::value>(acc[h], a_addr, b_addr, h, k,
                                                                             (accumulate | k) != 0 ? 1u : 0u);
              }
            };
            if (!g.a_mn && !g.b_mn) mma(std::false_type{}, std::false_type{});
            else if (!g.a_mn) mma(std::false_type{}, std::true_type{});
            else if (g.b_mn) mma(std::true_type{}, std::true_type{});
            else mma(std::true_type{}, std::false_type{});
          },
          [&](uint32_t stage) {
            if (lane == 0) mbar_arrive(&sm.empty_bar[stage]);
          });
      wgmma_fence_regs(acc[0]);
      wgmma_fence_regs(acc[1]);
      OM_TRACE(tslot + 3);
      // fragments -> global: every quad of lanes writes 32 consecutive bytes of a row (whole sectors)
      const bool vec = (ldc & 1) == 0 && (reinterpret_cast<uintptr_t>(Cw) & 7) == 0;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int rw = m_blk * kBlockM + h * 64 + ew * 16 + (lane >> 2) + 8 * u;
          if (rw >= M) continue;
          float* out = Cw + static_cast<int64_t>(rw) * ldc;
#pragma unroll
          for (int j = 0; j < kLossBN / 8; ++j) {
            const int col = n_blk * kLossBN + 8 * j + 2 * (lane & 3);
            const float v0 = acc[h][4 * j + 2 * u], v1 = acc[h][4 * j + 2 * u + 1];
            if (vec && col + 2 <= N) {
              *reinterpret_cast<float2*>(out + col) = make_float2(v0, v1);
            } else {
              if (col < N) out[col] = v0;
              if (col + 1 < N) out[col + 1] = v1;
            }
          }
        }
      OM_TRACE(tslot + 4);
      if (S > 1) {
        // all S slices of a tile run at the same time on different CTAs: each waits for the others and then adds
        // the S partials of ITS share of the warp's 32 rows, in slice order
        __threadfence();  // this lane's partial rows are visible before the counter moves
        named_bar_sync(5, 128);  // ... and those of the whole warpgroup (a warp stored rows of other warps' shares)
        unsigned* arrive = &g.sem[(tile * 4 + ew) * 2];
        if (lane == 0) {
          atomicAdd(arrive, 1u);
          const long long t0 = clock64();
          while (*reinterpret_cast<volatile unsigned*>(arrive) < static_cast<unsigned>(S)) {
            if (clock64() - t0 > OM_WAIT_TIMEOUT_CYCLES) {
              atomicCAS(&om_dev_fault, 0u, 0x80ef0000u | (blockIdx.x & 0xffffu));
              break;
            }
          }
          __threadfence();
        }
        __syncwarp();
        OM_TRACE(tslot + 5);
        const int rps = (32 + S - 1) / S, rb = ks * rps, re = min(32, rb + rps);
        const int r0 = m_blk * kBlockM + ew * 32, c = n_blk * kLossBN + lane * 4;
        const int64_t slice = static_cast<int64_t>(M) * ldc;
        if ((ldc & 3) == 0 && c + 4 <= N) {  // lane <-> 4 consecutive columns: one 512-byte row per load instruction
#pragma unroll 1
          for (int h = rb; h < re; h += 8) {
            float4 v[kMaxSplit][8];
#pragma unroll
            for (int sl = 0; sl < kMaxSplit; ++sl)
#pragma unroll
              for (int r = 0; r < 8; ++r) {
                const bool ok = sl < S && h + r < re && r0 + h + r < M;
                v[sl][r] = ok ? __ldcg(reinterpret_cast<const float4*>(g.part + sl * slice + static_cast<int64_t>(r0 + h + r) * ldc + c))
                              : make_float4(0.f, 0.f, 0.f, 0.f);
              }
#pragma unroll
            for (int r = 0; r < 8; ++r) {
              float4 acc = v[0][r];
#pragma unroll
              for (int sl = 1; sl < kMaxSplit; ++sl)
                acc.x += v[sl][r].x, acc.y += v[sl][r].y, acc.z += v[sl][r].z, acc.w += v[sl][r].w;
              if (h + r < re && r0 + h + r < M) *reinterpret_cast<float4*>(g.C + static_cast<int64_t>(r0 + h + r) * ldc + c) = acc;
            }
          }
        } else {
          for (int r = rb; r < re && r0 + r < M; ++r)
            for (int i = 0; i < 4 && c + i < N; ++i) {
              const float* src = g.part + static_cast<int64_t>(r0 + r) * ldc + c + i;
              float acc = __ldcg(src);
              for (int sl = 1; sl < S; ++sl) acc += __ldcg(src + sl * slice);
              g.C[static_cast<int64_t>(r0 + r) * ldc + c + i] = acc;
            }
        }
        OM_TRACE(tslot + 6);
        __syncwarp();
        if (lane == 0 && atomicAdd(arrive + 1, 1u) == static_cast<unsigned>(S - 1)) {  // last one out resets both
          arrive[0] = 0u;
          arrive[1] = 0u;
        }
      }
    }
  }
}

// src [rows, cols] (fp32 or bf16, dense) -> dst bf16 [rows, ldd]; grid-strided over 8-element row segments
// (pads untouched: TMA never reads beyond the logical extent)
template <typename T>
__device__ __forceinline__ void to_bf16_rows(const T* __restrict__ src, int rows, int cols, __nv_bfloat16* dst, int ldd,
                                             int t_begin, int t_step) {
  const int segs = (cols + 7) / 8;
  const int64_t total = static_cast<int64_t>(rows) * segs;
  const bool vec = (cols & 7) == 0 && (reinterpret_cast<uintptr_t>(src) & 31) == 0;
#pragma unroll 4
  for (int64_t i = t_begin; i < total; i += t_step) {
    const int r = static_cast<int>(i / segs), c = static_cast<int>(i % segs) * 8;
    const T* in = src + static_cast<int64_t>(r) * cols + c;
    __nv_bfloat16* out = dst + static_cast<int64_t>(r) * ldd + c;
    if (vec) {
      uint4 o;
      if constexpr (sizeof(T) == 4) {
        const float4 lo = *reinterpret_cast<const float4*>(in), hi = *reinterpret_cast<const float4*>(in + 4);
        o = make_uint4(pack_bf16x2(lo.x, lo.y), pack_bf16x2(lo.z, lo.w), pack_bf16x2(hi.x, hi.y), pack_bf16x2(hi.z, hi.w));
      } else {
        o = *reinterpret_cast<const uint4*>(in);
      }
      *reinterpret_cast<uint4*>(out) = o;
    } else {
      for (int j = 0; j < 8 && c + j < cols; ++j) out[j] = __float2bfloat16(static_cast<float>(in[j]));
    }
  }
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(kLossThreads, 1)
loss_fused_kernel(const __grid_constant__ LossMaps maps, const __grid_constant__ LossArgs a) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ double red[kLossThreads];
  __shared__ float xch[kLossThreads / 32][2];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  LossSmem sm;
  sm.ring = smem;
  sm.full_bar = reinterpret_cast<uint64_t*>(smem + LossCfg::kBarOffset);
  sm.empty_bar = sm.full_bar + kLossStages;
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = static_cast<int>(threadIdx.x & 31);
  const int G = static_cast<int>(gridDim.x);

  if (warp == 0 && lane == 0) {
    for (int i = 0; i < 3; ++i) {
      tma_prefetch_desc(&maps.a[i]);
      tma_prefetch_desc(&maps.b[i]);
    }
  }
  if (warp == 1 && lane == 0) {
    ring_init(sm.full_bar, sm.empty_bar, kLossStages, 4);  // one arrive per consumer warp
    fence_barrier_init();
  }
  __syncthreads();
  LossRing ring;

  // ------------------------------ PREP ------------------------------
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    *a.bad_target = 0;
    a.ts[4] = 0ull;
    a.ts[0] = global_timer_ns();
  }
  if (!a.direct) {
    const int t0 = static_cast<int>(blockIdx.x) * kLossThreads + static_cast<int>(threadIdx.x), tn = G * kLossThreads;
    if (a.is_bf16) {
      to_bf16_rows(static_cast<const __nv_bfloat16*>(a.P), a.np, a.d, a.pb, a.dpad, t0, tn);
      to_bf16_rows(static_cast<const __nv_bfloat16*>(a.Q), a.nq, a.d, a.qb, a.dpad, t0, tn);
    } else {
      to_bf16_rows(static_cast<const float*>(a.P), a.np, a.d, a.pb, a.dpad, t0, tn);
      to_bf16_rows(static_cast<const float*>(a.Q), a.nq, a.d, a.qb, a.dpad, t0, tn);
    }
    fence_proxy_async_global();
    grid_sync(a.grid_bar);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) a.ts[1] = global_timer_ns();

  // ------------------------------ LOGITS ------------------------------
  {
    const GemmDesc g{&maps.a[0], &maps.b[0], a.nq, a.np, a.d, a.S, a.np, false, false, 1, nullptr, nullptr, -1000};
    gemm_phase(g, 0, sm, ring, warp, lane);
  }
  grid_sync(a.grid_bar);
  if (blockIdx.x == 0 && threadIdx.x == 0) a.ts[2] = global_timer_ns();

  // ------------------------------ SOFTMAX + GRAD OF THE LOGITS ------------------------------
  {
    const int tpq = a.np / a.nq;
    const float wl = a.w * a.loss_scale;
    const bool want_grads = a.dQ || a.dP;
    if (a.sm_fast) {
      // two warps per query row (alternating 128-column chunks), the row in registers: one trip to L2, one exp per
      // element; the pair exchanges its partial max / sum through shared memory
      constexpr int kV = kSoftmaxMaxCols / 256;  // float4 per lane
      const int pair = warp >> 1, half = warp & 1;
      for (int q = pair * G + static_cast<int>(blockIdx.x); q < a.nq; q += (kLossThreads / 64) * G) {
        const float* s = a.S + static_cast<int64_t>(q) * a.np;
        __nv_bfloat16* grow = a.G + static_cast<int64_t>(q) * a.npp;
        int64_t t = a.target ? a.target[q] : static_cast<int64_t>(q) * tpq;
        if (t < 0 || t >= a.np) {
          if (lane == 0) *a.bad_target = 1;
          t = 0;
        }
        float4 v[kV];
#pragma unroll
        for (int i = 0; i < kV; ++i) {
          const int col = (2 * i + half) * 128 + lane * 4;
          v[i] = col < a.np ? __ldcg(reinterpret_cast<const float4*>(s + col))
                            : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        }
        float m = -INFINITY;
#pragma unroll
        for (int i = 0; i < kV; ++i) m = fmaxf(m, fmaxf(fmaxf(v[i].x, v[i].y), fmaxf(v[i].z, v[i].w)));
        m = warp_max(m);
        if (lane == 0) xch[warp][0] = m;
        named_bar_sync(1 + pair, 64);
        m = fmaxf(m, xch[warp ^ 1][0]);
        float z = 0.f;
#pragma unroll
        for (int i = 0; i < kV; ++i) {
          if ((2 * i + half) * 128 < a.np) {
            v[i].x = expf(v[i].x - m), v[i].y = expf(v[i].y - m), v[i].z = expf(v[i].z - m), v[i].w = expf(v[i].w - m);
            z += (v[i].x + v[i].y) + (v[i].z + v[i].w);
          }
        }
        z = warp_sum(z);
        if (lane == 0) xch[warp][1] = z;
        named_bar_sync(1 + pair, 64);
        z += xch[warp ^ 1][1];
        if (half == 0 && lane == 0) a.row_loss[q] = (m + logf(z)) - __ldcg(s + t);
        if (want_grads) {
          const float sc = wl / z;
          const int tc = static_cast<int>(t);
#pragma unroll
          for (int i = 0; i < kV; ++i) {
            const int col = (2 * i + half) * 128 + lane * 4;
            if (col < a.np) {
              float g0 = v[i].x * sc, g1 = v[i].y * sc, g2 = v[i].z * sc, g3 = v[i].w * sc;
              if (static_cast<unsigned>(tc - col) < 4u) {
                const int k = tc - col;
                g0 -= k == 0 ? wl : 0.f, g1 -= k == 1 ? wl : 0.f, g2 -= k == 2 ? wl : 0.f, g3 -= k == 3 ? wl : 0.f;
              }
              *reinterpret_cast<uint2*>(grow + col) = make_uint2(pack_bf16x2(g0, g1), pack_bf16x2(g2, g3));
            }
          }
        }
      }
    } else {  // any width / alignment: one warp per row, three passes over it
      for (int q = warp * G + static_cast<int>(blockIdx.x); q < a.nq; q += (kLossThreads / 32) * G) {
        const float* s = a.S + static_cast<int64_t>(q) * a.np;
        __nv_bfloat16* grow = a.G + static_cast<int64_t>(q) * a.npp;
        int64_t t = a.target ? a.target[q] : static_cast<int64_t>(q) * tpq;
        if (t < 0 || t >= a.np) {
          if (lane == 0) *a.bad_target = 1;
          t = 0;
        }
        float m = -INFINITY;
        for (int j = lane; j < a.np; j += 32) m = fmaxf(m, __ldcg(s + j));
        m = warp_max(m);
        float z = 0.f;
        for (int j = lane; j < a.np; j += 32) z += expf(__ldcg(s + j) - m);
        z = warp_sum(z);
        if (lane == 0) a.row_loss[q] = (m + logf(z)) - __ldcg(s + t);
        if (want_grads) {
          const float sc = wl / z;
          for (int j = lane; j < a.np; j += 32) {
            float gv = expf(__ldcg(s + j) - m) * sc;
            if (j == t) gv -= wl;
            grow[j] = __float2bfloat16(gv);
          }
        }
      }
    }
  }
  fence_proxy_async_global();
  grid_sync(a.grid_bar);
  if (blockIdx.x == 0 && threadIdx.x == 0) a.ts[3] = global_timer_ns();

  // ------------------------------ LOSS (last CTA, fixed summation order) ------------------------------
  if (static_cast<int>(blockIdx.x) == G - 1) {
    double acc = 0.0;
    for (int i = threadIdx.x; i < a.nq; i += kLossThreads) acc += a.row_loss[i];
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int s = kLossThreads / 2; s > 0; s >>= 1) {
      if (static_cast<int>(threadIdx.x) < s) red[threadIdx.x] += red[threadIdx.x + s];
      __syncthreads();
    }
    // out-of-range targets (PyTorch would device-assert) poison the loss with NaN instead of being ignored
    if (threadIdx.x == 0)
      *a.loss_out = *a.bad_target ? __int_as_float(0x7fc00000) : static_cast<float>(red[0] * a.w * a.loss_scale);
  }

  // ------------------------------ GRADS ------------------------------
  if (threadIdx.x == 0) OM_TRACE(60);
  int rot = 0;
  if (a.dQ) {  // first: the slice reduction of its last arrivers overlaps the dP tiles of everybody else
    const GemmDesc g{&maps.a[1], &maps.b[1], a.nq, a.d, a.np, a.dQ, a.d, false, true, a.dq_split, a.dq_part, a.dq_sem, 0};
    gemm_phase(g, rot, sm, ring, warp, lane);
    rot = ((a.nq + kBlockM - 1) / kBlockM) * ((a.d + kLossBN - 1) / kLossBN) * a.dq_split;
  }
  if (a.dP) {
    const GemmDesc g{&maps.a[2], &maps.b[2], a.np, a.d, a.nq, a.dP, a.d, true, true, 1, nullptr, nullptr, 16};
    gemm_phase(g, rot, sm, ring, warp, lane);
  }
  if (warp >= 4 && lane == 0) atomicMax(&a.ts[4], global_timer_ns());
  if (warp == 4 && lane == 0) OM_TRACE(61);
}

struct LossWs {
  void* p = nullptr;
  size_t bytes = 0;
  unsigned* grid_bar = nullptr;  // persistent (self-resetting), zeroed once: [0] grid barrier, [64..] split-K counters,
                                 // last 64 bytes: phase timestamps
  // tensor maps are rebuilt only when an address or an extent they encode changes.  G's offset in the workspace
  // depends on whether the caller keeps the logits (scores_out), so it is part of the key.
  LossMaps maps;
  const void* maps_base = nullptr;
  const void *maps_q = nullptr, *maps_p = nullptr, *maps_g = nullptr;
  int maps_nq = 0, maps_np = 0, maps_d = 0;
};
constexpr int kLossBarBytes = 65536, kLossSemSlots = (kLossBarBytes - 256 - 64) / 4;
static LossWs g_loss_ws;

// Measurement switches (read once): OM_LOSS_COPY_INPUTS = always convert / copy the inputs (no in-place TMA reads),
// OM_LOSS_SPLITK = n overrides the K slices of dQ, OM_LOSS_LOOPED_SOFTMAX = three-pass softmax rows.
struct LossKnobs {
  bool copy_inputs, looped_softmax;
  int splitk;  // 0 = automatic
  LossKnobs() {
    copy_inputs = getenv("OM_LOSS_COPY_INPUTS") != nullptr;
    looped_softmax = getenv("OM_LOSS_LOOPED_SOFTMAX") != nullptr;
    const char* e = getenv("OM_LOSS_SPLITK");
    splitk = e ? std::max(1, atoi(e)) : 0;
  }
};
static const LossKnobs& loss_knobs() {
  static const LossKnobs k;
  return k;
}  // grown on demand; one process drives one GPU (see header)

}  // namespace om

using namespace om;

extern "C" int om_contrastive_loss_fwd_bwd(const void* Q, const void* P, om_dtype dtype, int nq, int np, int d,
                                           const int64_t* target, int reduction, float loss_scale, float* loss_out,
                                           float* dQ, float* dP, float* scores_out, void* stream) {
  if (!Q || !P || !loss_out || nq <= 0 || np <= 0 || d <= 0)
    return fail(OM_EINVAL, "om_contrastive_loss_fwd_bwd: bad arguments (nq=%d np=%d d=%d)", nq, np, d);
  if (dtype != OM_F32 && dtype != OM_BF16) return fail(OM_EINVAL, "loss: dtype must be f32 or bf16");
  if (reduction != OM_REDUCE_MEAN && reduction != OM_REDUCE_SUM) return fail(OM_EINVAL, "loss: bad reduction");
  if (!target && np < nq) return fail(OM_EINVAL, "loss: default target needs np >= nq");
  const int sms = device_sm_count();
  if (sms < 0) return sms;
  NvtxRange nvtx("om.loss");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  LossWs& ws = g_loss_ws;
  const int dpad = (int)round_up(d, 8), npp = (int)round_up(np, 8);
  // aligned bf16 inputs are read in place by TMA (row pitch = d elements must be a multiple of 16 bytes)
  const bool direct = dtype == OM_BF16 && d % 8 == 0 && ((reinterpret_cast<uintptr_t>(Q) | reinterpret_cast<uintptr_t>(P)) & 15) == 0 &&
                      !loss_knobs().copy_inputs;
  Layout lay;
  const size_t o_qb = lay.add(direct ? 0 : (size_t)nq * dpad * 2), o_pb = lay.add(direct ? 0 : (size_t)np * dpad * 2);
  const size_t o_s = lay.add(scores_out ? 0 : (size_t)nq * np * 4);
  const size_t o_g = lay.add((size_t)nq * npp * 2);
  const size_t o_rl = lay.add((size_t)nq * 4), o_flag = lay.add(256);
  // split-K of dQ: enough slices to spread its few tiles over the grid, >= 8 k-blocks per slice, at most 4 slices
  // (OM_LOSS_SPLITK overrides, for measurements)
  int dq_split = 1;
  const int dq_tiles = ((nq + kBlockM - 1) / kBlockM) * ((d + kLossBN - 1) / kLossBN);
  if (dQ) {
    const int num_k = (np + kBlockK - 1) / kBlockK;
    int want = std::min(std::min(sms / std::max(1, dq_tiles), num_k / 8), kMaxSplit);
    if (loss_knobs().splitk) want = std::min(std::min(loss_knobs().splitk, num_k), std::min(kMaxSplit, sms / std::max(1, dq_tiles)));
    if (dq_tiles * 8 > kLossSemSlots) want = 1;
    if (want > 1) {
      const int kper = (num_k + want - 1) / want;
      dq_split = (num_k + kper - 1) / kper;  // no empty slice
    }
  }
  const size_t o_part = lay.add(dq_split > 1 ? (size_t)dq_split * nq * d * 4 : 0);
  const size_t off = lay.bytes;
  if (off > ws.bytes) {
    if (ws.p) {
      // the workspace is process-global: the call that last used it may have run on another stream
      OM_CUDA(cudaDeviceSynchronize());
      cudaFree(ws.p);
    }
    ws.p = nullptr;
    ws.bytes = 0;
    ws.maps_base = nullptr;
    OM_CUDA(dev_malloc(&ws.p, off));
    ws.bytes = off;
  }
  if (!ws.grid_bar) {
    OM_CUDA(cudaMalloc(&ws.grid_bar, kLossBarBytes));
    // on `st`, ahead of the launch below: a legacy-stream memset is not ordered before a launch on a non-blocking stream
    OM_CUDA(cudaMemsetAsync(ws.grid_bar, 0, kLossBarBytes, st));
  }
  LossArgs a;
  a.Q = Q;
  a.P = P;
  a.is_bf16 = dtype == OM_BF16;
  a.nq = nq;
  a.np = np;
  a.d = d;
  a.dpad = dpad;
  a.direct = direct ? 1 : 0;
  a.npp = npp;
  a.target = target;
  a.w = reduction == OM_REDUCE_MEAN ? 1.0f / nq : 1.0f;
  a.loss_scale = loss_scale;
  a.qb = region<__nv_bfloat16>(ws.p, o_qb);
  a.pb = region<__nv_bfloat16>(ws.p, o_pb);
  a.G = region<__nv_bfloat16>(ws.p, o_g);
  a.S = scores_out ? scores_out : region<float>(ws.p, o_s);
  a.row_loss = region<float>(ws.p, o_rl);
  a.loss_out = loss_out;
  a.dQ = dQ;
  a.dP = dP;
  a.bad_target = region<int>(ws.p, o_flag);
  a.grid_bar = ws.grid_bar;
  a.dq_split = dq_split;
  a.dq_part = region<float>(ws.p, o_part);
  a.dq_sem = ws.grid_bar + 64;
  a.ts = reinterpret_cast<unsigned long long*>(reinterpret_cast<uint8_t*>(ws.grid_bar) + kLossBarBytes - 64);
  a.sm_fast = (np % 4 == 0 && np <= kSoftmaxMaxCols && (reinterpret_cast<uintptr_t>(a.S) & 15) == 0 &&
               !loss_knobs().looped_softmax)
                  ? 1
                  : 0;

  const void* q_src = direct ? Q : static_cast<const void*>(a.qb);
  const void* p_src = direct ? P : static_cast<const void*>(a.pb);
  const uint64_t in_pitch = direct ? (uint64_t)d * 2 : (uint64_t)dpad * 2;
  if (ws.maps_base != ws.p || ws.maps_q != q_src || ws.maps_p != p_src || ws.maps_g != a.G || ws.maps_nq != nq ||
      ws.maps_np != np || ws.maps_d != d) {
    const uint64_t un = (uint64_t)np, uq = (uint64_t)nq, ud = (uint64_t)d;
    int rc = 0;
    // K-major operands: box {64 k, 128 rows}; MN-major operands (the matrix as stored, K = its rows): box {64, 64}
    rc |= make_tmap_bf16_2d(&ws.maps.a[0], q_src, ud, uq, in_pitch, kBlockK, kBlockM);            // Q   [nq, d]
    rc |= make_tmap_bf16_2d(&ws.maps.b[0], p_src, ud, un, in_pitch, kBlockK, kLossBN);            // P   [np, d]
    rc |= make_tmap_bf16_2d(&ws.maps.a[1], a.G, un, uq, (uint64_t)npp * 2, kBlockK, kBlockM);     // G   [nq, np], K = np
    rc |= make_tmap_bf16_2d(&ws.maps.b[1], p_src, ud, un, in_pitch, 64, kBlockK);                 // P   as [K = np, N = d]
    rc |= make_tmap_bf16_2d(&ws.maps.a[2], a.G, un, uq, (uint64_t)npp * 2, 64, kBlockK);          // G   as [K = nq, M = np]
    rc |= make_tmap_bf16_2d(&ws.maps.b[2], q_src, ud, uq, in_pitch, 64, kBlockK);                 // Q   as [K = nq, N = d]
    if (rc != 0) return fail(OM_ECUDA, "loss: tensor-map encode failed (%d)", rc);
    ws.maps_base = ws.p;
    ws.maps_q = q_src;
    ws.maps_p = p_src;
    ws.maps_g = a.G;
    ws.maps_nq = nq;
    ws.maps_np = np;
    ws.maps_d = d;
  }

  static int max_ctas = 0;
  if (!max_ctas) {
    OM_CUDA(cudaFuncSetAttribute(loss_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kLossSmemBytes));
    int per_sm = 0;
    OM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, loss_fused_kernel, kLossThreads, kLossSmemBytes));
    if (per_sm < 1) return fail(OM_ECUDA, "loss: fused kernel does not fit on an SM");
    max_ctas = sms;  // one CTA per SM: the whole grid is co-resident (required by the grid barrier)
  }
  auto tiles = [](int m, int n) { return ((m + kBlockM - 1) / kBlockM) * ((n + kLossBN - 1) / kLossBN); };
  const int gemm_tiles = std::max(tiles(nq, np), (dQ ? tiles(nq, d) * dq_split : 0) + (dP ? tiles(np, d) : 0));
  const int prep_ctas = direct ? 0 : (int)std::min<int64_t>(sms, ((int64_t)(nq + np) * dpad / 8 + kLossThreads - 1) / kLossThreads);
  int grid = std::max(std::max(gemm_tiles, (nq + 7) / 8), prep_ctas);
  grid = std::max(1, std::min(grid, max_ctas));
  void* params[] = {const_cast<LossMaps*>(&ws.maps), &a};
  OM_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(loss_fused_kernel), dim3(grid), dim3(kLossThreads), params,
                                      kLossSmemBytes, st));
  return 0;
}

extern "C" int om_debug_loss_phase_ns(uint64_t out[4]) {
  if (!out) return fail(OM_EINVAL, "om_debug_loss_phase_ns: null output");
  if (!g_loss_ws.grid_bar) return fail(OM_ESTATE, "om_debug_loss_phase_ns: no loss call yet");
  unsigned long long ts[5];
  OM_CUDA(cudaDeviceSynchronize());  // the last loss call may have run on any stream
  OM_CUDA(cudaMemcpy(ts, reinterpret_cast<uint8_t*>(g_loss_ws.grid_bar) + kLossBarBytes - 64, sizeof(ts), cudaMemcpyDeviceToHost));
  for (int i = 0; i < 4; ++i) out[i] = ts[i + 1] - ts[i];
  return 0;
}

#ifdef OM_LOSS_TRACE
extern "C" int om_debug_loss_trace(unsigned long long* out, int ctas) {
  OM_CUDA(cudaMemcpyFromSymbol(out, om_loss_trace, sizeof(unsigned long long) * 64 * std::min(ctas, 160)));
  return 0;
}
#endif
