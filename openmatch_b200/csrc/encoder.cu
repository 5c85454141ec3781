// H100-native encoder forward behind DRModel.encode (src/openmatch/modeling/dense_retrieval_model.py:133-155):
// HF BertModel (post-LN, GELU-erf) or T5EncoderModel (pre-RMSNorm, ReLU, shared relative position bias)
// -> 'first' / 'mean' pooling (:145-150, src/openmatch/utils.py:233-235) -> bias-free LinearHead
// (src/openmatch/modeling/linear.py:19,22-23) -> F.normalize (:153-154).
//
// Per layer (T = B*L tokens, H hidden, I = heads * head width (64; BERT also 32) attention width, F ffn).  LayerNorm /
// RMSNorm never runs as a kernel of its own: the residual stream is kept UN-normalised (s, fp32 + a bf16 copy) together
// with per-row (sum, sum of squares); the normalisation is folded algebraically into the GEMM that consumes it,
//        LN(s) W^T = rstd * (s Wf^T) + (W beta + b),   Wf = W diag(gamma) with every row centred (sum_i Wf[j, i] = 0,
//        which makes the "- rstd * mean * rowsum" term vanish; RMSNorm has no mean, rows stay as they are),
// and into the residual read of the GEMM that produces the next s:
//   QKV    wgmma GEMM [T,H]x[3I,H]^T on bf16(s) and the folded weights; epilogue: rstd[row] * acc + folded bias
//          -> bf16 Q|K [T,2I] and V transposed [I, T]
//   ATTN   one CTA per (128-row tile, 64 columns of Q|K = one 64-wide head or two 32-wide heads), one warpgroup, 64
//          query rows and one head at a time: S = Q K^T (wgmma, registers) -> masked softmax on the accumulator
//          fragments -> P (bf16, registers) -> O = P V (wgmma) -> ctx bf16 [T,I]
//   OPROJ  wgmma GEMM [T,I]x[H,I]^T, epilogue (EpiResidNorm): s' = acc + bias + LN(s) (BERT) / + s (T5), written in
//          place as fp32 (TMA load + TMA store of the residual tile) and as bf16, row statistics of s' accumulated
//   FFN1   wgmma GEMM [T,H]x[F,H]^T on bf16(s') and folded weights; epilogue: rstd[row] * acc + folded bias, GELU(erf) /
//          ReLU -> bf16 [T,F]
//   FFN2   wgmma GEMM [T,F]x[H,F]^T, epilogue (EpiResidNorm) like OPROJ -> next layer's s
// One norm kernel runs after the last layer (last_hidden_state for pooling).  Activations feeding tensor cores are
// bf16; the residual stream, normalisation statistics, softmax, pooling, head and L2-normalisation are fp32.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <new>
#include <set>
#include <string>
#include <vector>

#include "common.h"
#include "gemm.cuh"
#include "quant_i8.cuh"

namespace om {

constexpr int kAttnCols = 64;    // columns of Q, K and V^T an attention work item loads: one 64-wide or two 32-wide heads
constexpr int kMaxL = 128;       // one attention tile; sequences of at most kMaxL tokens take attn_kernel
constexpr int kMaxLongL = 512;   // longest padded om_encode sequence (a multiple of 128 tokens above kMaxL) and T5
                                 // sequence; longer sequences take attn_stream_kernel
constexpr float kLog2e = 1.4426950408889634f;

// ===================================================================================================
// GEMM epilogues
// ===================================================================================================
// GELU(x) = x/2 (1 + erf(x / sqrt 2)) for an element pair: the FFN1 epilogue is issue-bound, so erf is the cheapest
// approximation that is invisible after bf16 rounding of the output:
// z P(z^2) / Q(z^2) on [-4, 4], P cubic, Q cubic with Q >= 1, fitted against math.erf: max |err| 2.1e-5
// (bf16 output rounding is 2e-3 relative); 6 FFMA + 1 MUFU.RCP per element.
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float2 gelu_erf2(float2 x) {
  float2 z = mul2(x, splat2(0.70710678118654752440f));
  z.x = fminf(fmaxf(z.x, -4.f), 4.f);
  z.y = fminf(fmaxf(z.y, -4.f), 4.f);
  const float2 z2 = mul2(z, z);
  float2 p = fma2(splat2(0.0006061712047085166f), z2, splat2(0.041214898228645325f));
  p = fma2(p, z2, splat2(0.1745881289243698f));
  p = fma2(p, z2, splat2(1.1282498836517334f));
  float2 q = fma2(splat2(0.008151348680257797f), z2, splat2(0.10013707727193832f));
  q = fma2(q, z2, splat2(0.48736122250556946f));
  q = fma2(q, z2, splat2(1.0f));
  const float2 erf = mul2(mul2(p, z), make_float2(rcp_approx(q.x), rcp_approx(q.y)));
  const float2 hx = mul2(x, splat2(0.5f));
  return fma2(hx, erf, hx);
}

enum { ACT_NONE = 0, ACT_GELU = 1, ACT_RELU = 2 };

// Normalisation of one row of the residual stream from its (sum, sum of squares): rstd and rstd * mean.
// The statistics arrive as kStatParts partial (sum, sumsq) pairs per row — one per (column tile, epilogue column group)
// of the GEMM that produced the row, summed here in a fixed order (deterministic, no atomics); unused slots hold zeros.
// LayerNorm: var = E[x^2] - mean^2 (fp32; clamped at 0), RMSNorm: mean = 0.  stats == nullptr: identity (rstd 1, rm 0).
constexpr int kStatParts = 16;
struct RowNorm {
  const float* stats;  // [T, kStatParts, 2] or nullptr
  float inv_h, eps;
  int rms;
  __device__ __forceinline__ void get(int row, int M, float& rstd, float& rm) const {
    rstd = 1.f;
    rm = 0.f;
    if (stats && row < M) {
      const float4* p = reinterpret_cast<const float4*>(stats + static_cast<int64_t>(row) * (2 * kStatParts));
      float sum = 0.f, sq = 0.f;
#pragma unroll
      for (int j = 0; j < kStatParts / 2; ++j) {
        const float4 t = __ldg(p + j);
        sum += t.x;
        sq += t.y;
        sum += t.z;
        sq += t.w;
      }
      const float mean = rms ? 0.f : sum * inv_h;
      const float var = fmaxf(sq * inv_h - mean * mean, 0.f);
      rstd = rsqrtf(var + eps);
      rm = rstd * mean;
    }
  }
};

// Coalescing stage for bf16 epilogue outputs.  A thread owns one accumulator ROW, so a direct 16-byte store
// per lane touches 32 different cache lines per warp instruction and the SM's load/store unit — not the tensor
// core — bounds the GEMM.  Instead two
// consecutive 32-column chunks (= 128 bytes per row) are written into a warp-private 4 KB shared-memory tile
// in the TMA SWIZZLE_128B layout (16-byte pieces XOR-ed with row & 7) and ONE lane issues a TMA store of the
// 32-row x 64-column box: no LSU work for the global write, rows beyond M are clipped by the tensor map.
struct StagedBf16 {
  static constexpr int kBytesPerWarp = 4096;
  uint32_t held[16];  // first chunk of the pair, packed bf16x2
  int have, held_col, in_flight;
  uint8_t* tile;
  __device__ __forceinline__ void bind(uint8_t* smem, int epi_tid) {
    tile = smem + (epi_tid >> 5) * kBytesPerWarp;  // 1024-byte aligned (swizzle atom)
    have = 0;
    in_flight = 0;
  }
  // direct (uncoalesced) store of one 32-column chunk: tail of an odd chunk count
  __device__ __forceinline__ static void store_direct(const uint32_t (&pk)[16], __nv_bfloat16* out, int64_t ldo, int row,
                                                      int col0, int M) {
    if (row >= M) return;
    uint4* dst = reinterpret_cast<uint4*>(out + static_cast<int64_t>(row) * ldo + col0);
#pragma unroll
    for (int i = 0; i < 4; ++i) dst[i] = make_uint4(pk[4 * i], pk[4 * i + 1], pk[4 * i + 2], pk[4 * i + 3]);
  }
  // pk = packed chunk [col0, col0+32) of this lane's row; every lane of the warp must call this
  __device__ __forceinline__ void push(const uint32_t (&pk)[16], const CUtensorMap* tm_out, int row, int col0) {
    if (!have) {
#pragma unroll
      for (int i = 0; i < 16; ++i) held[i] = pk[i];
      have = 1;
      held_col = col0;
      return;
    }
    have = 0;
    const int lane = threadIdx.x & 31;
    if (in_flight) {  // the previous TMA store must have finished reading the tile
      if (lane == 0) bulk_wait_group_read0();
      __syncwarp();
    }
    uint8_t* mine = tile + lane * 128;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      *reinterpret_cast<uint4*>(mine + ((p ^ (lane & 7)) << 4)) =
          make_uint4(held[4 * p], held[4 * p + 1], held[4 * p + 2], held[4 * p + 3]);
      *reinterpret_cast<uint4*>(mine + (((p + 4) ^ (lane & 7)) << 4)) =
          make_uint4(pk[4 * p], pk[4 * p + 1], pk[4 * p + 2], pk[4 * p + 3]);
    }
    fence_proxy_async_smem();  // generic-proxy writes -> visible to the TMA (async proxy)
    __syncwarp();
    if (lane == 0) {
      tma_store_2d(tm_out, tile, held_col, row);  // lane 0's row is the first row of the warp's 32-row slab
      bulk_commit_group();
    }
    in_flight = 1;
  }
  __device__ __forceinline__ void flush_tail(__nv_bfloat16* out, int64_t ldo, int row, int M) {
    if (have) {
      store_direct(held, out, ldo, row, held_col, M);
      have = 0;
    }
  }
  __device__ __forceinline__ void finish() {
    if (in_flight && (threadIdx.x & 31) == 0) bulk_wait_group0();
  }
};

// out bf16 [M, ldo] = act(rstd[row] * acc + bias[col])   (norm.stats == nullptr: rstd = 1, plain act(acc + bias)).
// The mean term of a folded LayerNorm needs no work here: the folded weight rows are centred (fold_norm_kernel), so
// sum_i s_i W''[j, i] already equals sum_i (s_i - mean) W'[j, i].
template <int ACT>
struct EpiBiasActBf16 {
  CUtensorMap tm_out;  // box {64 cols, 32 rows} over out, SWIZZLE_128B (TMA store)
  __nv_bfloat16* out;
  int64_t ldo;
  const float* bias;  // nullable (folded bias W beta + b when the input is normalised)
  int M, N;
  RowNorm norm;
  static constexpr bool kPrefetch = false;
  __host__ __device__ static constexpr int smem_bytes(int epi_warps) { return epi_warps * StagedBf16::kBytesPerWarp; }
  struct State {
    StagedBf16 stage;
    float rstd, rm;
  };
  __device__ __forceinline__ void bind(State& s, uint8_t* smem, int epi_tid) const { s.stage.bind(smem, epi_tid); }
  __device__ __forceinline__ void finish(State& s) const { s.stage.finish(); }
  __device__ __forceinline__ void begin(State& s, int row, int, int) const {
    s.stage.have = 0;
    norm.get(row, M, s.rstd, s.rm);
  }
  __device__ __forceinline__ void end(State& s, int row) const { s.stage.flush_tail(out, ldo, row, M); }
  __device__ __forceinline__ void chunk(State& s, int row, int col0, const float (&v)[32]) const {
    if (col0 >= N) return;  // warp-uniform; N is a multiple of 32 for every encoder GEMM (checked on the host)
    uint32_t packed[16];
    float bv[32];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 t = bias ? __ldg(reinterpret_cast<const float4*>(bias + col0) + j) : make_float4(0.f, 0.f, 0.f, 0.f);
      bv[4 * j] = t.x, bv[4 * j + 1] = t.y, bv[4 * j + 2] = t.z, bv[4 * j + 3] = t.w;
    }
    const float2 rs = splat2(s.rstd);
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      float2 ab = fma2(rs, make_float2(v[i], v[i + 1]), make_float2(bv[i], bv[i + 1]));
      if (ACT == ACT_GELU) {
        ab = gelu_erf2(ab);
      } else if (ACT == ACT_RELU) {
        ab.x = fmaxf(ab.x, 0.f);
        ab.y = fmaxf(ab.y, 0.f);
      }
      packed[i >> 1] = pack_bf16x2(ab.x, ab.y);
    }
    s.stage.push(packed, &tm_out, row, col0);
  }
};

// QKV projection: columns [0, 2I) -> qk bf16 [T, 2I]; columns [2I, 3I) -> vt bf16 [I, ldv], V transposed
// (the P*V GEMM wants V^T K-major, i.e. token-contiguous) in the attention kernel's tile-local column order:
// token m of attention tile m / valid_rows sits at column tile * 128 + m % valid_rows, so every tile's
// V^T box starts at a 256-byte aligned column.
struct EpiQKV {
  CUtensorMap tm_qk;  // box {64 cols, 32 rows} over qk, SWIZZLE_128B (TMA store)
  __nv_bfloat16* qk;
  __nv_bfloat16* vt;
  int64_t ldv;
  const float* bias;  // nullable, [3I] (folded: W beta + b)
  int M, I2;          // I2 = 2*I
  int valid_rows;     // tokens per attention tile (spt * L)
  RowNorm norm;       // normalisation of the input rows, applied here (see the file header)
  static constexpr bool kPrefetch = false;
  __host__ __device__ static constexpr int smem_bytes(int epi_warps) { return epi_warps * StagedBf16::kBytesPerWarp; }
  struct State {
    int vcol;
    StagedBf16 stage;
    float rstd, rm;
  };
  __device__ __forceinline__ void bind(State& s, uint8_t* smem, int epi_tid) const { s.stage.bind(smem, epi_tid); }
  __device__ __forceinline__ void finish(State& s) const { s.stage.finish(); }
  __device__ __forceinline__ void begin(State& s, int row, int, int) const {
    s.vcol = (row / valid_rows) * 128 + row % valid_rows;
    s.stage.have = 0;
    norm.get(row, M, s.rstd, s.rm);
  }
  __device__ __forceinline__ void end(State& s, int row) const { s.stage.flush_tail(qk, I2, row, M); }
  __device__ __forceinline__ void chunk(State& s, int row, int col0, const float (&v)[32]) const {
    if (col0 >= I2 + (I2 >> 1)) return;  // warp-uniform
    float bv[32];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 t = bias ? __ldg(reinterpret_cast<const float4*>(bias + col0) + j) : make_float4(0.f, 0.f, 0.f, 0.f);
      bv[4 * j] = t.x, bv[4 * j + 1] = t.y, bv[4 * j + 2] = t.z, bv[4 * j + 3] = t.w;
    }
    const float rstd = s.rstd;
    if (col0 < I2) {
      uint32_t packed[16];
#pragma unroll
      for (int i = 0; i < 32; i += 2)
        packed[i >> 1] = pack_bf16x2(fmaf(rstd, v[i], bv[i]), fmaf(rstd, v[i + 1], bv[i + 1]));
      s.stage.push(packed, &tm_qk, row, col0);
    } else if (row < M) {
      __nv_bfloat16* dst = vt + static_cast<int64_t>(col0 - I2) * ldv + s.vcol;
#pragma unroll
      for (int i = 0; i < 32; ++i)
        dst[static_cast<int64_t>(i) * ldv] = __float2bfloat16(fmaf(rstd, v[i], bv[i]));  // lanes = consecutive tokens
    }
  }
};

// Residual epilogue of the O-proj and FFN2 GEMMs:   s'[m, n] = acc + bias[n] + R(s[m, n])
//   R = LayerNorm of the residual stream with the producer's (gamma, beta) and the row's (mean, rstd)   (BERT, post-LN)
//   R = identity                                                                                        (T5, pre-norm)
// s lives in fp32 [T, H] and is updated IN PLACE; bf16(s') goes to xb (the next GEMM's A operand) and every (thread, tile)
// writes its partial (sum, sum of squares) of s' into its own slot of stats_out for whoever normalises s' next.
// A thread owns an accumulator ROW, so touching global memory directly would cost one cache line per lane and
// instruction; instead each warp moves its 32-row x 32-column chunks through shared memory with TMA:
//   TMA load  s[32 rows, 32 cols] fp32 -> 4 KB tile (SWIZZLE_128B; the first chunk of a tile is requested before the
//             tile's mainloop, the residual of the NEXT tile is pulled into L2 a tile ahead; one tile per warp: the
//             shared memory a second one would take is what the mainloop's ring and the staged accumulator need)
//   in place  thread r rewrites row r of the tile (16-byte pieces XOR-ed with r & 7: conflict-free) and writes bf16(s')
//             into a 2 KB tile (SWIZZLE_64B: 64-byte rows, also conflict-free)
//   TMA store both tiles; rows >= M are clipped by the tensor maps.
struct EpiResidNorm {
  CUtensorMap tm_s;   // fp32 s [T, H], box {32 cols, 32 rows}, SWIZZLE_128B (load and store)
  CUtensorMap tm_xb;  // bf16 xb [T, H], box {32 cols, 32 rows}, SWIZZLE_64B (store)
  const float* bias;  // nullable [N]
  RowNorm norm;       // statistics of s (norm.stats == nullptr: R = identity)
  const float* gamma;  // [N] LayerNorm weight / bias applied to the residual (BERT); unused when norm.stats == nullptr
  const float* beta;
  float* stats_out;  // [T, kStatParts, 2]: slot n_blk * parts + column group <- this thread's (sum, sumsq) of s'
  int parts;         // column groups per tile (epilogue warps / 4); (N / BN) * parts <= kStatParts
  int M, N;
  int bn;            // tile width (BN of the GEMM): geometry of the static tile schedule, for the L2 prefetch below
  static constexpr bool kPrefetch = true;
  static constexpr int kF32Tile = 4096, kBf16Tile = 2048, kPerWarp = kF32Tile + kBf16Tile;
  static constexpr int kMaxN = 1024;     // per-column constants staged in shared memory: 2 * kMaxN floats
  __host__ __device__ static constexpr int smem_bytes(int epi_warps) { return epi_warps * kPerWarp + 1024 + 2 * kMaxN * 4; }
  struct State {
    uint8_t* f32tile;   // [4096]
    uint8_t* bf16tile;  // [2048]
    uint64_t* bars;     // [1]
    const float* gsm;   // [N] gamma of the residual's LayerNorm (1 when there is none)
    const float* bsm;   // [N] bias + beta
    uint32_t parity;    // phase parity of bars[0]
    int slot;           // statistics slot of this (tile, column group)
    int group;          // column group of this warp
    float rstd, rm, rsum, rsq;
  };
  __device__ __forceinline__ void bind(State& s, uint8_t* smem, int epi_tid) const {
    const int w = epi_tid >> 5, nw = blockDim.x / 32 - kGemmProducerThreads / 32;
    s.f32tile = smem + w * kF32Tile;                        // 1024-byte aligned (swizzle atoms)
    s.bf16tile = smem + nw * kF32Tile + w * kBf16Tile;       // 512-byte aligned is enough for SWIZZLE_64B
    s.bars = reinterpret_cast<uint64_t*>(smem + nw * kPerWarp) + w;
    s.parity = 0;
    s.group = w >> 2;
    if ((epi_tid & 31) == 0) {
      mbar_init(&s.bars[0], 1);
      fence_barrier_init();
    }
    // per-column constants, once per CTA: every lane of a chunk reads the same column's gamma / (bias + beta), so they
    // come from shared memory as broadcasts instead of 24 dependent global loads per chunk and thread
    float* gs = reinterpret_cast<float*>(smem + nw * kPerWarp + 1024);
    float* bs = gs + kMaxN;
    const bool ln = norm.stats != nullptr;
    for (int c = epi_tid; c < N; c += nw * 32) {
      gs[c] = ln ? gamma[c] : 1.f;
      bs[c] = (bias ? bias[c] : 0.f) + (ln ? beta[c] : 0.f);
    }
    s.gsm = gs;
    s.bsm = bs;
    named_bar_sync(1, nw * 32);  // the epilogue warps only (the producer / MMA warps never join barrier 1)
  }
  __device__ __forceinline__ void finish(State&) const {
    if ((threadIdx.x & 31) == 0) bulk_wait_group0();
  }
  __device__ __forceinline__ void begin(State& s, int row, int m_blk, int n_blk) const {
    norm.get(row, M, s.rstd, s.rm);
    s.rsum = 0.f;
    s.rsq = 0.f;
    s.slot = n_blk * parts + s.group;
    // The residual of the tile this CTA processes NEXT (static schedule: tile + gridDim.x, n fastest) is pulled into L2
    // now, a whole tile ahead: its TMA loads then cost an L2 hit instead of an exposed HBM round trip per chunk.
    if (bn > 0 && (threadIdx.x & 31) == 0) {  // bn == 0: no look-ahead
      const int num_n = (N + bn - 1) / bn, num_m = (M + kBlockM - 1) / kBlockM;
      const int next = m_blk * num_n + n_blk + static_cast<int>(gridDim.x);
      if (next < num_m * num_n) {
        const int nm = next / num_n, nn = next - nm * num_n;
        const int row0 = row + (nm - m_blk) * kBlockM;  // lane 0's row = first row of the warp's slab
        const int cols = bn / parts;                     // columns per column group
#pragma unroll 1
        for (int c = 0; c < cols; c += 32) tma_prefetch_l2_2d(&tm_s, nn * bn + s.group * cols + c, row0);
      }
    }
  }
  // request the residual of chunk [row0 .. row0+32) x [col0 .. col0+32) into tile `b` (lane 0; the tile's last TMA store
  // must have finished READING it: the caller waits for that)
  __device__ __forceinline__ void request(State& s, int row0, int col0) const {
    bulk_wait_group_read0();  // the tile's last TMA store has finished reading it
    mbar_arrive_expect_tx(&s.bars[0], kF32Tile);
    tma_load_2d(s.f32tile, &tm_s, &s.bars[0], col0, row0);
  }
  __device__ __forceinline__ void prefetch(State& s, int row, int col0) const {
    if (col0 >= N) return;  // warp-uniform
    if ((threadIdx.x & 31) == 0) request(s, row, col0);  // lane 0's row = first row of the warp's 32-row slab
  }
  __device__ __forceinline__ void end(State& s, int row) const {
    if (row < M)
      *reinterpret_cast<float2*>(stats_out + (static_cast<int64_t>(row) * kStatParts + s.slot) * 2) = make_float2(s.rsum, s.rsq);
  }
  __device__ __forceinline__ void chunk(State& s, int row, int col0, const float (&v)[32], int next_col0) const {
    if (col0 >= N) return;  // warp-uniform
    const int lane = threadIdx.x & 31;
    mbar_wait_warp(&s.bars[0], s.parity, 20);
    s.parity ^= 1u;
    uint8_t* mine = s.f32tile + lane * 128;
    uint8_t* mineb = s.bf16tile + lane * 64;
    // R = (s - mean) * rstd * gamma + beta = s * (rstd * gamma) + (beta - rstd * mean * gamma); without a LayerNorm on the
    // residual (T5) gamma = 1, rstd = 1, mean = 0:  s' = acc + s * (rstd g) + ((bias + beta) - rstd mean g)
    const float rstd = s.rstd, nrm = -s.rm;
    const float4* gp = reinterpret_cast<const float4*>(s.gsm + col0);
    const float4* bp = reinterpret_cast<const float4*>(s.bsm + col0);
    float rsum = 0.f, rsq = 0.f;
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      float4* slot = reinterpret_cast<float4*>(mine + ((p ^ (lane & 7)) << 4));
      const float4 r = *slot;
      const float4 g = gp[p], bb = bp[p];
      float4 o;
      o.x = fmaf(r.x, rstd * g.x, fmaf(nrm, g.x, bb.x)) + v[4 * p];
      o.y = fmaf(r.y, rstd * g.y, fmaf(nrm, g.y, bb.y)) + v[4 * p + 1];
      o.z = fmaf(r.z, rstd * g.z, fmaf(nrm, g.z, bb.z)) + v[4 * p + 2];
      o.w = fmaf(r.w, rstd * g.w, fmaf(nrm, g.w, bb.w)) + v[4 * p + 3];
      *slot = o;
      rsum += (o.x + o.y) + (o.z + o.w);
      rsq = fmaf(o.x, o.x, fmaf(o.y, o.y, fmaf(o.z, o.z, fmaf(o.w, o.w, rsq))));
      // bf16 tile: 64-byte rows, 16-byte piece (p >> 1) XOR-ed with (row >> 1) & 3 (SWIZZLE_64B)
      uint2* hb = reinterpret_cast<uint2*>(mineb + ((((p >> 1) ^ ((lane >> 1) & 3)) << 4) | ((p & 1) << 3)));
      *hb = make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
    }
    if (row < M) {  // rows beyond M hold zero-filled residuals + garbage-free accumulators, but must not count
      s.rsum += rsum;
      s.rsq += rsq;
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      tma_store_2d(&tm_s, s.f32tile, col0, row);
      tma_store_2d(&tm_xb, s.bf16tile, col0, row);
      bulk_commit_group();
      if (next_col0 >= 0 && next_col0 < N) request(s, row, next_col0);  // waits for the stores above to release the tile
    }
  }
};

// ===================================================================================================
// row-wise kernels: one warp per token row, H % 128 == 0, H <= 1024
// ===================================================================================================
constexpr int kMaxVec = 8;  // float4 per lane: 8 * 4 * 32 = 1024 columns

template <bool RMS>
__device__ __forceinline__ void norm_row(float4 (&v)[kMaxVec], int nvec, int H, float eps) {
  float s = 0.f;
  if (!RMS) {
#pragma unroll
    for (int j = 0; j < kMaxVec; ++j)
      if (j < nvec) s += (v[j].x + v[j].y) + (v[j].z + v[j].w);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  }
  const float mean = RMS ? 0.f : s / H;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < kMaxVec; ++j)
    if (j < nvec) {
      const float a = v[j].x - mean, b = v[j].y - mean, c = v[j].z - mean, d = v[j].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / H + eps);
#pragma unroll
  for (int j = 0; j < kMaxVec; ++j)
    if (j < nvec) {
      v[j].x = (v[j].x - mean) * rstd;
      v[j].y = (v[j].y - mean) * rstd;
      v[j].z = (v[j].z - mean) * rstd;
      v[j].w = (v[j].w - mean) * rstd;
    }
}

__device__ __forceinline__ void affine_store(const float4 (&v)[kMaxVec], int nvec, int lane, const float* gamma,
                                             const float* beta, float* out) {
#pragma unroll
  for (int j = 0; j < kMaxVec; ++j)
    if (j < nvec) {
      const int c = (j * 32 + lane) * 4;
      const float4 g = *reinterpret_cast<const float4*>(gamma + c);
      float4 y = make_float4(v[j].x * g.x, v[j].y * g.y, v[j].z * g.z, v[j].w * g.w);
      if (beta) {
        const float4 b = *reinterpret_cast<const float4*>(beta + c);
        y.x += b.x, y.y += b.y, y.z += b.z, y.w += b.w;
      }
      *reinterpret_cast<float4*>(out + c) = y;
    }
}

// out = Norm(h) * gamma (+ beta), fp32; out may alias h.
template <bool RMS>
__global__ void __launch_bounds__(128) norm_kernel(const float* h, const float* gamma, const float* beta, float eps,
                                                   int T, int H, float* out) {
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= T) return;
  const int nvec = H >> 7;
  float4 v[kMaxVec];
  const float* src = h + static_cast<int64_t>(row) * H;
#pragma unroll
  for (int j = 0; j < kMaxVec; ++j)
    if (j < nvec) v[j] = *reinterpret_cast<const float4*>(src + (j * 32 + lane) * 4);
  norm_row<RMS>(v, nvec, H, eps);
  affine_store(v, nvec, lane, gamma, beta, out + static_cast<int64_t>(row) * H);
}

// Row statistics of a freshly embedded row: slot 0 of the row's kStatParts partials holds (sum, sum of squares), the
// other slots zeros (the GEMM epilogues that normalise the row sum all slots, see RowNorm).
__device__ __forceinline__ void store_row_stats(const float4 (&v)[kMaxVec], int nvec, int lane, float* stats_row) {
  float s = 0.f, q = 0.f;
#pragma unroll
  for (int j = 0; j < kMaxVec; ++j)
    if (j < nvec) {
      s += (v[j].x + v[j].y) + (v[j].z + v[j].w);
      q = fmaf(v[j].x, v[j].x, fmaf(v[j].y, v[j].y, fmaf(v[j].z, v[j].z, fmaf(v[j].w, v[j].w, q))));
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if (lane < kStatParts) reinterpret_cast<float2*>(stats_row)[lane] = lane == 0 ? make_float2(s, q) : make_float2(0.f, 0.f);
}

__device__ __forceinline__ void raw_store(const float4 (&v)[kMaxVec], int nvec, int lane, float* out_f32,
                                          __nv_bfloat16* out_bf16) {
#pragma unroll
  for (int j = 0; j < kMaxVec; ++j)
    if (j < nvec) {
      const int c = (j * 32 + lane) * 4;
      *reinterpret_cast<float4*>(out_f32 + c) = v[j];
      *reinterpret_cast<uint2*>(out_bf16 + c) = make_uint2(pack_bf16x2(v[j].x, v[j].y), pack_bf16x2(v[j].z, v[j].w));
    }
}

// ---------------------------------------------------------------------------------------------------
// packed (variable-length) layout, om_encode_packed: sequences of <= 128 tokens are bin-packed whole into 128-row tiles,
// longer ones start on a tile boundary and take ceil(l / 128) tiles; the rows in between are padding.
// ---------------------------------------------------------------------------------------------------
struct PackedSeq {  // one sequence of a packed call, in layout order (ascending row0)
  int row0;         // first layout row, relative to the row group being encoded
  int len;          // tokens
  int out;          // output row of its representation (relative to the call's chunk of sequences)
  int pad_;
  int64_t tok0;     // offset of its first token in the caller's packed token array
};

// rowmap[r] = (slot of the sequence that holds layout row r, position inside it), (-1, -1) for a padding row; kmask[r] =
// 0 for a real row, -inf for padding (padding rows are never attended to).  One thread per row: binary search of the
// (row0-sorted) sequence table.
__global__ void packed_rowmap_kernel(const PackedSeq* seqs, int nseq, int T, int2* rowmap, float* kmask) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= T) return;
  int lo = 0, hi = nseq;  // the last sequence with row0 <= r lies in [lo, hi)
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (seqs[mid].row0 <= r) lo = mid;
    else hi = mid;
  }
  const int pos = r - seqs[lo].row0;
  const bool real = pos >= 0 && pos < seqs[lo].len;
  rowmap[r] = real ? make_int2(lo, pos) : make_int2(-1, -1);
  kmask[r] = real ? 0.f : __int_as_float(0xff800000);
}

// padding row of the packed layout: zeros (fp32, bf16) and zero statistics, so that everything computed from it stays
// finite (a NaN there would reach real rows through P V, where masked keys are multiplied by 0)
__device__ __forceinline__ void zero_row(int nvec, int lane, float* out_f32, __nv_bfloat16* out_bf16, float* stats_row) {
  float4 v[kMaxVec];
#pragma unroll
  for (int j = 0; j < kMaxVec; ++j) v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  raw_store(v, nvec, lane, out_f32, out_bf16);
  if (lane < kStatParts) reinterpret_cast<float2*>(stats_row)[lane] = make_float2(0.f, 0.f);
}

// RoBERTa position ids (modeling_roberta.py create_position_ids_from_input_ids, padding_idx = kRobertaPad): a token with
// id != 1 at index t of its sequence gets 1 + #{t' <= t : id[t'] != 1}, a token with id 1 gets position 1.  They come
// from the ids alone, not from the attention mask, so a pad id inside a sequence's content takes position 1 and does not
// advance the count.  pos_ids[layout row] for every token of the nseq sequences: seqs == nullptr, sequence b is the
// padded row ids[b * L, (b + 1) * L) at layout rows b * L + t; else sequence k is ids[seqs[k].tok0 + t] at layout row
// seqs[k].row0 + t, t < seqs[k].len.  One warp per sequence: an inclusive warp scan of (id != 1) per 32-token chunk and
// a running carry.
constexpr int kRobertaPad = 1;

__global__ void __launch_bounds__(128) roberta_pos_kernel(const int64_t* ids, int nseq, int L, const PackedSeq* seqs,
                                                          int32_t* pos_ids) {
  const int s = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (s >= nseq) return;
  int64_t tok0 = static_cast<int64_t>(s) * L, row0 = tok0;
  int len = L;
  if (seqs) {
    tok0 = seqs[s].tok0;
    row0 = seqs[s].row0;
    len = seqs[s].len;
  }
  int carry = 0;
  for (int c = 0; c < len; c += 32) {
    const int t = c + lane;
    const int real = t < len && ids[tok0 + t] != kRobertaPad ? 1 : 0;
    int incl = real;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (t < len) pos_ids[row0 + t] = real ? kRobertaPad + carry + incl : kRobertaPad;
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
}

// BERT embeddings (modeling_bert.py:53-112): s = word[id] + type[tt] + pos[l], UN-normalised (fp32 + bf16) with its row
// statistics; the embedding LayerNorm is applied by the first layer's QKV / O-proj epilogues like every other LayerNorm.
// s is stored minus its row mean: only the embedding LayerNorm reads it, which is shift-invariant.  A common offset in
// the embedding tables otherwise leaves rows whose mean is tens of times their standard deviation, and the bf16 copy that
// the QKV GEMM reads (and the folded weights' rounding residue, scaled by mean / std) would bury the row's information.
// rowmap != nullptr (packed layout): token and position come from the row map, padding rows are zeroed; a real token's
// row is bitwise the row the padded layout gives it.  kPosIds (RoBERTa): the position is pos_ids[row] (roberta_pos_kernel)
// instead of the token's index in its sequence; everything else is shared.
template <bool kPosIds>
__global__ void __launch_bounds__(128) bert_embed_kernel(const int64_t* ids, const int64_t* tts, const float* word,
                                                         const float* type, const float* pos, int T, int L, int H, int vocab,
                                                         int type_vocab, float* out_f32, __nv_bfloat16* out_bf16,
                                                         float* stats, const int2* rowmap, const PackedSeq* seqs,
                                                         const int32_t* pos_ids) {
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= T) return;
  const int nvec = H >> 7;
  int64_t tok = row;
  int l = row % L;
  if (rowmap) {
    const int2 m = rowmap[row];
    if (m.x < 0) {
      zero_row(nvec, lane, out_f32 + static_cast<int64_t>(row) * H, out_bf16 + static_cast<int64_t>(row) * H,
               stats + static_cast<int64_t>(row) * (2 * kStatParts));
      return;
    }
    tok = seqs[m.x].tok0 + m.y;
    l = m.y;
  }
  if (kPosIds) l = pos_ids[row];
  int64_t id = ids[tok];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  int64_t tt = tts ? tts[tok] : 0;
  tt = tt < 0 ? 0 : (tt >= type_vocab ? type_vocab - 1 : tt);
  float4 v[kMaxVec];
#pragma unroll
  for (int j = 0; j < kMaxVec; ++j)
    if (j < nvec) {
      const int c = (j * 32 + lane) * 4;
      const float4 a = *reinterpret_cast<const float4*>(word + id * H + c);
      const float4 b = *reinterpret_cast<const float4*>(type + tt * H + c);
      const float4 p = *reinterpret_cast<const float4*>(pos + static_cast<int64_t>(l) * H + c);
      v[j] = make_float4((a.x + b.x) + p.x, (a.y + b.y) + p.y, (a.z + b.z) + p.z, (a.w + b.w) + p.w);
    }
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < kMaxVec; ++j)
    if (j < nvec) sum += (v[j].x + v[j].y) + (v[j].z + v[j].w);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / H;
#pragma unroll
  for (int j = 0; j < kMaxVec; ++j)
    if (j < nvec) v[j].x -= mean, v[j].y -= mean, v[j].z -= mean, v[j].w -= mean;
  raw_store(v, nvec, lane, out_f32 + static_cast<int64_t>(row) * H, out_bf16 + static_cast<int64_t>(row) * H);
  store_row_stats(v, nvec, lane, stats + static_cast<int64_t>(row) * (2 * kStatParts));
}

// T5: h = embed_tokens[id] (no position embedding, no scaling; modeling_t5.py:682,734), fp32 + bf16 + row statistics
// (rowmap: packed layout, as in bert_embed_kernel)
__global__ void __launch_bounds__(128) t5_embed_kernel(const int64_t* ids, const float* emb, int T, int H, int vocab,
                                                       float* out_f32, __nv_bfloat16* out_bf16, float* stats,
                                                       const int2* rowmap, const PackedSeq* seqs) {
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= T) return;
  const int nvec = H >> 7;
  int64_t tok = row;
  if (rowmap) {
    const int2 m = rowmap[row];
    if (m.x < 0) {
      zero_row(nvec, lane, out_f32 + static_cast<int64_t>(row) * H, out_bf16 + static_cast<int64_t>(row) * H,
               stats + static_cast<int64_t>(row) * (2 * kStatParts));
      return;
    }
    tok = seqs[m.x].tok0 + m.y;
  }
  int64_t id = ids[tok];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  float4 v[kMaxVec];
#pragma unroll
  for (int j = 0; j < kMaxVec; ++j)
    if (j < nvec) v[j] = *reinterpret_cast<const float4*>(emb + id * H + (j * 32 + lane) * 4);
  raw_store(v, nvec, lane, out_f32 + static_cast<int64_t>(row) * H, out_bf16 + static_cast<int64_t>(row) * H);
  store_row_stats(v, nvec, lane, stats + static_cast<int64_t>(row) * (2 * kStatParts));
}

// Weight folding (once, at om_encoder_finalize):  Wf[j, i] = bf16(W[j, i] * gamma[i] - centre * mean_i(W[j, i] * gamma[i]))
// and bfold[j] = b[j] + sum_i W[j, i] * beta[i] (fp32, un-centred W).  With centred rows (LayerNorm) the mean term of the
// folded normalisation vanishes identically:  sum_i s_i Wf[j, i] = sum_i (s_i - mean(s)) W[j, i] gamma[i]  (up to the bf16
// rounding of Wf, ~1e-3 of a weight, multiplied by mean(s) / std(s): below the bf16 rounding of the GEMM's output while
// the rows of s are no further from zero mean than LN(s), which the centred embedding rows ensure, see bert_embed_kernel).
// RMSNorm (T5): centre = 0, beta = none.
// One warp per output row j.
__global__ void __launch_bounds__(256) fold_norm_kernel(const float* __restrict__ W, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, const float* __restrict__ bias,
                                                        int N, int K, int centre, __nv_bfloat16* __restrict__ Wf,
                                                        float* bfold) {
  const int j = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (j >= N) return;
  const float* w = W + static_cast<int64_t>(j) * K;
  float c = 0.f, b = 0.f;
  for (int i = lane; i < K; i += 32) {
    const float wi = w[i];
    c = fmaf(wi, gamma[i], c);
    if (beta) b = fmaf(wi, beta[i], b);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    c += __shfl_xor_sync(0xffffffffu, c, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const float shift = centre ? c / static_cast<float>(K) : 0.f;
  for (int i = lane; i < K; i += 32) Wf[static_cast<int64_t>(j) * K + i] = __float2bfloat16(fmaf(w[i], gamma[i], -shift));
  if (lane == 0 && bfold) bfold[j] = b + (bias ? bias[j] : 0.f);
}

__global__ void keymask_kernel(const int64_t* attn_mask, float* kmask, int T) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < T) kmask[i] = attn_mask[i] != 0 ? 0.f : __int_as_float(0xff800000);
}

// ===================================================================================================
// attention: one CTA per (tile of 128 token rows = spt whole sequences, head)
// ===================================================================================================
struct AttnParams {
  int T, L, spt, I, Tvalid_rows;  // Tvalid_rows = spt * L: rows of the tile that belong to it
  float scale_log2;               // softmax scale * log2(e)
  const float* kmask;             // [T] 0 / -inf
  const float* relbias_log2;      // nullable [heads, 2*kMaxL-1] (attn_kernel) / [heads, 2*kMaxLongL-1]
                                  // (attn_stream_kernel), already multiplied by log2(e)
  __nv_bfloat16* ctx;             // [T, I]
  // packed layout (om_encode_packed; nullptr for om_encode): a row's sequence and position come from rowmap [T], its
  // length from seqs; attn_kernel starts at tile tile0 (the long sequences' tiles come first)
  const int2* rowmap;
  const PackedSeq* seqs;
  int tile0;
};

// Q, K and V^T of a tile in shared memory (48 KB, TMA, 128B-swizzled); S, P and O never leave registers.
constexpr int kAttnSmemQ = 0, kAttnSmemK = 16384, kAttnSmemV = 32768;
constexpr int kAttnSmemMisc = 49152;  // kb[4] u32, rel[256] f32, barrier
constexpr int kAttnSmemBytes = kAttnSmemMisc + 16 + 1024 + 64 + 1024;
constexpr int kAttnCtasPerSm = 3;

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// S = Q_h K^T for the 64 query rows [64 h, +64) of the tile: DH / 16 wgmma m64n128k16 (K = head width DH); qa / ka
// address the head's first column inside the 64-column Q / K boxes (a 32-wide head takes k-steps 0-1 or 2-3 of them)
template <int DH>
__device__ __forceinline__ void attn_scores(float (&s)[64], uint32_t qa, uint32_t ka) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < DH / 16; ++k)
    wgmma_m64n128k16_bf16<0, 0>(s, wgmma_desc(qa + k * 32, kDescKMajorSW128), wgmma_desc(ka + k * 32, kDescKMajorSW128),
                                k != 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(s);
}
// O (+)= P V for the same 64 rows: P from registers (the probabilities in s, packed to bf16 as the A fragment of each
// 16-key step), V^T [DH dims, 128 keys] as two K-major boxes of 64 keys; va addresses the head's first row in the first
// box (the second 32-wide head of a box starts 32 rows = 4 whole 1024-byte swizzle atoms in)
template <int DH>
__device__ __forceinline__ void attn_pv(float (&o)[DH / 2], const float (&s)[64], uint32_t va, uint32_t accumulate) {
  uint32_t a[8][4];
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    a[kk][0] = pack_bf16x2(s[8 * kk + 0], s[8 * kk + 1]);
    a[kk][1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
    a[kk][2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]);
    a[kk][3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
  }
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    const uint64_t vd = wgmma_desc(va + (kk >> 2) * 8192 + (kk & 3) * 32, kDescKMajorSW128);
    if constexpr (DH == 64)
      wgmma_m64n64k16_bf16_rs(o, a[kk], vd, (accumulate | kk) != 0 ? 1u : 0u);
    else
      wgmma_m64n32k16_bf16_rs(o, a[kk], vd, (accumulate | kk) != 0 ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(o);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Fragment coordinates (see ptx.cuh): element 4 j + e of a thread's accumulator is row rr[e >> 1], column 8 j + 2 (lane % 4)
// + (e & 1) of the 64-row block.
// DH = head width (64, or 32 for BERT).  A work item is a (tile, unit of kAttnCols columns) pair: the unit holds
// 64 / DH whole heads, so the boxes, the shared-memory layout and the work per item are those of one 64-wide head.
// The relative position bias (T5, MPNet) exists for 64-wide heads only.
template <int DH>
__global__ void __launch_bounds__(128, kAttnCtasPerSm)
attn_kernel(const __grid_constant__ CUtensorMap tmQK, const __grid_constant__ CUtensorMap tmVt, AttnParams p, int n_tiles,
            int n_units) {
  constexpr int NH = kAttnCols / DH;  // heads per unit
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint32_t* s_kb = reinterpret_cast<uint32_t*>(smem + kAttnSmemMisc);
  float* s_rel = reinterpret_cast<float*>(s_kb + 4);
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_rel + 256);  // [0] loads

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    tma_prefetch_desc(&tmQK);
    tma_prefetch_desc(&tmVt);
    mbar_init(&bars[0], 1);
    fence_barrier_init();
  }
  __syncthreads();
  // Persistent CTA: work items are (tile, unit) pairs taken unit-fastest, so that the CTAs running at the same time read
  // the same token rows of qk (neighbouring 128-byte slices of one DRAM page instead of one slice from each of many pages).
  const int n_items = n_tiles * n_units;
  const bool has_rel = DH == 64 && p.relbias_log2 != nullptr;
  const uint32_t qa = smem_u32(smem + kAttnSmemQ), ka = smem_u32(smem + kAttnSmemK), va = smem_u32(smem + kAttnSmemV);
  uint32_t par = 0;
#pragma unroll 1
  for (int item = blockIdx.x; item < n_items; item += gridDim.x, par ^= 1u) {
    const int t = item / n_units, unit = item - t * n_units;
    const int tile = p.tile0 + t;
    const int row0 = tile * p.Tvalid_rows;  // first token of this tile
    if (tid == 0) {  // shared memory of the previous item is free (trailing barrier): loads go out first
      mbar_arrive_expect_tx(&bars[0], 3 * 16384);
      tma_load_2d(smem + kAttnSmemQ, &tmQK, &bars[0], unit * kAttnCols, row0);
      tma_load_2d(smem + kAttnSmemK, &tmQK, &bars[0], p.I + unit * kAttnCols, row0);
      tma_load_2d(smem + kAttnSmemV, &tmVt, &bars[0], tile * 128, unit * kAttnCols);
      tma_load_2d(smem + kAttnSmemV + 8192, &tmVt, &bars[0], tile * 128 + 64, unit * kAttnCols);
    }
    {
      const int tok = row0 + tid;
      // key validity as 4 x 32-bit words (bit c%32 of word c/32): one ballot per warp
      const bool key_ok = (tid < p.Tvalid_rows && tok < p.T) && p.kmask[tok] == 0.f;
      const unsigned bits = __ballot_sync(0xffffffffu, key_ok);
      if (lane == 0) s_kb[warp] = bits;
      if (has_rel) {
        for (int i = tid; i < 2 * kMaxL - 1; i += 128) s_rel[i] = p.relbias_log2[unit * (2 * kMaxL - 1) + i];
      }
    }
    __syncthreads();  // key bits / relative bias of this item are in place
    mbar_wait_warp(&bars[0], par, 10);

#pragma unroll 1
    for (int hh = 0; hh < 2 * NH; ++hh) {
      const int h = hh / NH, hd = hh % NH;  // 64-row half of the tile, head of the unit
      float sc[64];
      attn_scores<DH>(sc, qa + h * 8192 + hd * DH * 2, ka + hd * DH * 2);
      // ---- softmax on the fragments: this thread holds columns 8 j + 2 (lane % 4) + {0, 1} of two query rows ----
      int rr[2], c_lo[2], c_hi[2];
      bool valid[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        rr[u] = h * 64 + 16 * warp + (lane >> 2) + 8 * u;
        valid[u] = rr[u] < p.Tvalid_rows && row0 + rr[u] < p.T;
        // this row may attend key c iff the key is valid AND belongs to the row's own sequence [c_lo, c_hi)
        if (p.rowmap) {  // packed: the sequence of the row map (contiguous inside the tile); a padding row attends none
          const int2 mp = valid[u] ? p.rowmap[row0 + rr[u]] : make_int2(-1, -1);
          c_lo[u] = mp.x >= 0 ? rr[u] - mp.y : 0;
          c_hi[u] = mp.x >= 0 ? c_lo[u] + p.seqs[mp.x].len : 0;
        } else {
          c_lo[u] = valid[u] ? (rr[u] / p.L) * p.L : 0;
          c_hi[u] = valid[u] ? c_lo[u] + p.L : 0;
        }
      }
      float m[2] = {__int_as_float(0xff800000), __int_as_float(0xff800000)};
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int u = e >> 1, c = 8 * j + 2 * (lane & 3) + (e & 1);
          float v = sc[4 * j + e] * p.scale_log2;
          if (has_rel) v += s_rel[c - rr[u] + (kMaxL - 1)];
          const bool ok = c >= c_lo[u] && c < c_hi[u] && ((s_kb[c >> 5] >> (c & 31)) & 1u);
          v = ok ? v : __int_as_float(0xff800000);
          sc[4 * j + e] = v;
          m[u] = fmaxf(m[u], v);
        }
      float sum[2] = {0.f, 0.f};
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        m[u] = quad_max(m[u]);
        if (!(m[u] > __int_as_float(0xff800000))) m[u] = 0.f;  // every key masked (padding row): all p = 0
      }
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float pv = ex2_approx(sc[4 * j + e] - m[e >> 1]);  // ex2(-inf) = 0 for masked keys
          sc[4 * j + e] = pv;
          sum[e >> 1] += pv;
        }
      float o[DH / 2];
      attn_pv<DH>(o, sc, va + hd * DH * 128, 0u);
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const float tot = quad_sum(sum[u]);
        const float inv = tot > 0.f ? 1.0f / tot : 0.f;
        if (valid[u]) {
          __nv_bfloat16* dst =
              p.ctx + static_cast<int64_t>(row0 + rr[u]) * p.I + unit * kAttnCols + hd * DH + 2 * (lane & 3);
#pragma unroll
          for (int j = 0; j < DH / 8; ++j)
            *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(o[4 * j + 2 * u] * inv, o[4 * j + 2 * u + 1] * inv);
        }
      }
    }
    // the next item's TMA loads overwrite Q / K / V: every warp must be done with its wgmma reads
    __syncthreads();
  }  // item loop
}

// ---------------------------------------------------------------------------------------------------
// Sequences of kMaxL + 1 .. kMaxStreamL tokens, padded (L = 256 / 384 / 512) or packed: one CTA of three warpgroups per
// (128-row query tile, unit) loops over the sequence's 128-key tiles with an online softmax.  At these lengths attention
// is a large share of a layer (4 L^2 I FLOP against 24 L H^2 for the GEMMs), and at head width 64 the exponentials take
// about as long as the MMAs, so the loads must run ahead of the compute and the two halves of the query tile must not
// wait for each other:
//   producer  warp 0: Q once, then the sequence's 128-key tiles (K, V^T: 32 KB, and the tile's key-validity bits,
//             one ballot of kmask per 32 keys) into a ring of kAttnStreamStages slots with full / empty mbarriers
//             (ring.cuh); warps 1-3 only hand their registers over (setmaxnreg)
//   consumers warpgroups 1 and 2 own query rows [0, 64) and [64, 128) of the tile and walk the ring independently,
//             S_j = Q K_j^T (wgmma) -> running max / sum -> P_j (bf16, registers) -> O = O alpha + P_j V_j (wgmma), and
//             release a slot once both of its MMAs have completed; while one warpgroup is in its softmax the other's
//             wgmma run.
// The key-validity bits come per key tile, so the length is bounded by nothing the kernel sizes.  Keys of a tile that
// are all valid (every tile but a sequence's last) skip the masking.  Padding rows after a sequence's last token attend
// like its tokens (finite values nobody reads).  REL (T5, MPNet: 64-wide heads, at most kMaxLongL tokens) adds the relative
// position bias, a [2 kMaxLongL - 1] row per head held in shared memory.
// ---------------------------------------------------------------------------------------------------
constexpr int kMaxStreamL = 8192;
constexpr int kAttnStreamStages = 4;
constexpr int kAttnStreamThreads = 384;
constexpr int kAttnStreamStageBytes = 32768;  // K [128 keys, 64 cols] + V^T as two [64 cols, 64 keys] boxes
constexpr int kAttnStreamSmemRing = 16384;    // after Q [128 rows, 64 cols]
constexpr int kAttnStreamSmemMisc = kAttnStreamSmemRing + kAttnStreamStages * kAttnStreamStageBytes;
// misc: key bits [stages][4] u32, full[stages], empty[stages], Q barrier; then the relative bias row (REL)
constexpr int kAttnStreamSmemRel = kAttnStreamSmemMisc + 256;
static_assert(kAttnStreamStages * 16 + (2 * kAttnStreamStages + 1) * 8 <= 256, "stream kernel: misc overlaps rel");
constexpr int kAttnStreamSmemBytes = kAttnStreamSmemRel + (2 * kMaxLongL - 1) * 4 + 1024;

template <int DH, bool REL>
__global__ void __launch_bounds__(kAttnStreamThreads, 1)
attn_stream_kernel(const __grid_constant__ CUtensorMap tmQK, const __grid_constant__ CUtensorMap tmVt, AttnParams p) {
  constexpr int NH = kAttnCols / DH;  // heads per unit
  constexpr int S = kAttnStreamStages;
  static_assert(!REL || DH == 64, "the relative position bias exists for 64-wide heads only");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint32_t* s_kb = reinterpret_cast<uint32_t*>(smem + kAttnStreamSmemMisc);  // [S][4]: key bits of each slot
  uint64_t* full = reinterpret_cast<uint64_t*>(s_kb + 4 * S);
  uint64_t* empty = full + S;
  uint64_t* qbar = empty + S;
  float* s_rel = reinterpret_cast<float*>(smem + kAttnStreamSmemRel);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int qt = blockIdx.x, unit = blockIdx.y;
  const int row0 = qt * 128;  // first row of this query tile
  // the sequence's length and the position of the tile's first query in it: padded, every sequence takes L / 128 tiles;
  // packed, it starts on a tile boundary and the tile's first row is one of its tokens (place_packed)
  int len = p.L, qpos0 = qt % (p.L / 128) * 128;
  if (p.rowmap) {
    const int2 mp = p.rowmap[row0];
    len = p.seqs[mp.x].len;
    qpos0 = mp.y;
  }
  const int nk = (len + 127) / 128;  // key tiles of the sequence
  const int kt0 = qt - qpos0 / 128;  // its first tile

  if (tid == 0) {
    tma_prefetch_desc(&tmQK);
    tma_prefetch_desc(&tmVt);
    ring_init(full, empty, S, 8);  // a slot is released by each of the 8 consumer warps
    mbar_init(qbar, 1);
    fence_barrier_init();
  }
  if constexpr (REL) {
    for (int i = tid; i < 2 * kMaxLongL - 1; i += kAttnStreamThreads)
      s_rel[i] = p.relbias_log2[unit * (2 * kMaxLongL - 1) + i];
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------ producer warpgroup ------------------------------
    setmaxnreg_dec<40>();
    if (warp != 0) return;
    if (lane == 0) {
      mbar_arrive_expect_tx(qbar, 16384);
      tma_load_2d(smem, &tmQK, qbar, unit * kAttnCols, row0);
    }
    Ring<S> ring;
#pragma unroll 1
    for (int j = 0; j < nk; ++j, ring.advance()) {
      const int k0 = (kt0 + j) * 128;
      unsigned bits[4];
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const int tok = k0 + 32 * w + lane;
        bits[w] = __ballot_sync(0xffffffffu, tok < p.T && p.kmask[tok] == 0.f);
      }
      if (lane == 0) {
        ring_wait_free(empty, ring, 14);
        uint32_t* kb = s_kb + 4 * ring.stage;
#pragma unroll
        for (int w = 0; w < 4; ++w) kb[w] = bits[w];
        // the arrive releases the bit stores above to every consumer that sees the slot's phase complete
        mbar_arrive_expect_tx(&full[ring.stage], kAttnStreamStageBytes);
        uint8_t* slot = smem + kAttnStreamSmemRing + ring.stage * kAttnStreamStageBytes;
        tma_load_2d(slot, &tmQK, &full[ring.stage], p.I + unit * kAttnCols, k0);
        tma_load_2d(slot + 16384, &tmVt, &full[ring.stage], k0, unit * kAttnCols);
        tma_load_2d(slot + 16384 + 8192, &tmVt, &full[ring.stage], k0 + 64, unit * kAttnCols);
      }
      __syncwarp();
    }
    return;
  }

  // ------------------------------ consumer warpgroups ------------------------------
  setmaxnreg_inc<232>();
  const int wg = (warp >> 2) - 1;  // 64-row half of the tile
  const uint32_t qa = smem_u32(smem) + wg * 8192, ring_a = smem_u32(smem + kAttnStreamSmemRing);
  const float scale = p.scale_log2;
  // m_run: running maximum of the raw (unscaled) scores, or under REL of the scaled and biased logits (the bias breaks
  // "the maximum of the scaled scores is the scaled maximum"); ms scales m_run and the scores in the softmax below
  const float ms = REL ? 1.f : scale;
  int rr[2];
  float m_run[NH][2], sum[NH][2], o[NH][DH / 2];
#pragma unroll
  for (int u = 0; u < 2; ++u) rr[u] = wg * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * u;
#pragma unroll
  for (int hd = 0; hd < NH; ++hd) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      m_run[hd][u] = __int_as_float(0xff800000);
      sum[hd][u] = 0.f;
    }
#pragma unroll
    for (int i = 0; i < DH / 2; ++i) o[hd][i] = 0.f;
  }
  mbar_wait_warp(qbar, 0, 15);
  Ring<S> ring;
#pragma unroll 1
  for (int j = 0; j < nk; ++j, ring.advance()) {
    mbar_wait_warp(&full[ring.stage], ring.phase, 16);
    const uint32_t ka = ring_a + ring.stage * kAttnStreamStageBytes, va = ka + 16384;
    const uint32_t* kb = s_kb + 4 * ring.stage;
    const bool all_keys = (kb[0] & kb[1] & kb[2] & kb[3]) == 0xffffffffu;
#pragma unroll
    for (int hd = 0; hd < NH; ++hd) {
      float sc[64];
      attn_scores<DH>(sc, qa + hd * DH * 2, ka + hd * DH * 2);
      if (!all_keys) {
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int c = 8 * jj + 2 * (lane & 3) + (e & 1);
            if (!((kb[c >> 5] >> (c & 31)) & 1u)) sc[4 * jj + e] = __int_as_float(0xff800000);
          }
      }
      if constexpr (REL) {  // scaled logit + bias of the relative position (key - query); a masked key stays -inf
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int c = 8 * jj + 2 * (lane & 3) + (e & 1);
            sc[4 * jj + e] = fmaf(sc[4 * jj + e], scale, s_rel[(kMaxLongL - 1) - (qpos0 + rr[e >> 1]) + 128 * j + c]);
          }
      }
      float m_j[2] = {__int_as_float(0xff800000), __int_as_float(0xff800000)};
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
#pragma unroll
        for (int e = 0; e < 4; ++e) m_j[e >> 1] = fmaxf(m_j[e >> 1], sc[4 * jj + e]);
      // softmax in the log2 domain: p = 2^(s * scale - m * scale), one FFMA and one ex2 per score (scale > 0, so the
      // maximum of the scaled scores is the scaled maximum); under REL p = 2^(v - m) on the biased logits v
      float alpha[2], mm[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const float m_new = fmaxf(m_run[hd][u], quad_max(m_j[u]));
        mm[u] = (m_new > __int_as_float(0xff800000)) ? m_new * ms : 0.f;  // no allowed key seen so far: all p = 0
        alpha[u] = (m_run[hd][u] > __int_as_float(0xff800000)) ? ex2_approx(fmaf(m_run[hd][u], ms, -mm[u])) : 0.f;
        m_run[hd][u] = m_new;
        sum[hd][u] *= alpha[u];
      }
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float pv = ex2_approx(fmaf(sc[4 * jj + e], ms, -mm[e >> 1]));  // ex2(-inf) = 0 for masked keys
          sc[4 * jj + e] = pv;
          sum[hd][e >> 1] += pv;
        }
#pragma unroll
      for (int i = 0; i < DH / 2; ++i) o[hd][i] *= alpha[(i >> 1) & 1];
      attn_pv<DH>(o[hd], sc, va + hd * DH * 128, 1u);
    }
    // both MMAs of every head have completed (attn_pv waits for its group): the slot may be refilled
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[ring.stage]);
  }

#pragma unroll
  for (int hd = 0; hd < NH; ++hd)
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const float tot = quad_sum(sum[hd][u]);
      const float inv = tot > 0.f ? 1.0f / tot : 0.f;
      if (row0 + rr[u] < p.T) {
        __nv_bfloat16* dst = p.ctx + static_cast<int64_t>(row0 + rr[u]) * p.I + unit * kAttnCols + hd * DH + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < DH / 8; ++jj)
          *reinterpret_cast<uint32_t*>(dst + 8 * jj) =
              pack_bf16x2(o[hd][4 * jj + 2 * u] * inv, o[hd][4 * jj + 2 * u + 1] * inv);
      }
    }
}

// ===================================================================================================
// pooling / head / normalise (fp32)
// ===================================================================================================
// pooled[b, :] = hidden[b, 0, :]  or  sum_l hidden[b,l,:] m[b,l] / clamp(sum_l m[b,l], 1e-9)
__global__ void pool_kernel(const float* hidden, const int64_t* mask, int L, int H, int mean, float* pooled) {
  const int b = blockIdx.x;
  const float* src = hidden + static_cast<int64_t>(b) * L * H;
  if (!mean) {
    for (int c = threadIdx.x; c < H; c += blockDim.x) pooled[static_cast<int64_t>(b) * H + c] = src[c];
    return;
  }
  __shared__ float sm[kMaxLongL];
  for (int l = threadIdx.x; l < L; l += blockDim.x) sm[l] = mask[static_cast<int64_t>(b) * L + l] != 0 ? 1.f : 0.f;
  __syncthreads();
  float cnt = 0.f;
  for (int l = 0; l < L; ++l) cnt += sm[l];
  const float denom = fmaxf(cnt, 1e-9f);
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    float acc = 0.f;
    for (int l = 0; l < L; ++l) acc += src[static_cast<int64_t>(l) * H + c] * sm[l];
    pooled[static_cast<int64_t>(b) * H + c] = acc / denom;
  }
}

// packed layout: pooled[out, :] = hidden[row0, :]  or  the mean of the sequence's len rows.  One block per sequence.
__global__ void pool_packed_kernel(const float* hidden, const PackedSeq* seqs, int H, int mean, float* pooled) {
  const PackedSeq s = seqs[blockIdx.x];
  const float* src = hidden + static_cast<int64_t>(s.row0) * H;
  float* dst = pooled + static_cast<int64_t>(s.out) * H;
  if (!mean) {
    for (int c = threadIdx.x; c < H; c += blockDim.x) dst[c] = src[c];
    return;
  }
  const float denom = static_cast<float>(s.len);
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    float acc = 0.f;
    for (int l = 0; l < s.len; ++l) acc += src[static_cast<int64_t>(l) * H + c];
    dst[c] = acc / denom;
  }
}

// packed layout: out[tok0 + pos, :] = hidden[row, :] for every real row (padding rows are dropped).  One warp per row.
__global__ void __launch_bounds__(128) gather_packed_rows_kernel(const float* hidden, const int2* rowmap,
                                                                 const PackedSeq* seqs, int T, int H, float* out) {
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= T) return;
  const int2 m = rowmap[row];
  if (m.x < 0) return;
  const float* src = hidden + static_cast<int64_t>(row) * H;
  float* dst = out + (seqs[m.x].tok0 + m.y) * H;  // the caller's buffer: 4-byte alignment is all it promises
  for (int c = lane; c < H; c += 32) dst[c] = src[c];
}

// cross-encoder pairs (om_encode_pairs): the two token spans of one sequence, in the order of the sequence table
struct PairSpan {
  int64_t a0, b0;  // first token in the a / b store
  int a_len, b_len;
};
struct PairSpecials {  // prefix / suffix ids, passed by value
  int32_t prefix[4], suffix[4];
  int n_prefix, n_suffix;
};

__device__ __forceinline__ int32_t special_id(const int32_t (&ids)[4], int k) {
  int32_t id = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) id = j == k ? ids[j] : id;  // no dynamic indexing: the array stays in registers
  return id;
}

// tokens[s.row0 + pos] = (prefix ++ a[a0, a0 + a_len) ++ b[b0, b0 + b_len) ++ suffix)[pos] for every sequence s of one row
// group: the group's token stream in layout order, read by the packed embedding kernels through tok0 = row0.  One block
// per sequence.
__global__ void pair_tokens_kernel(const int32_t* a, const int32_t* b, const PackedSeq* seqs, const PairSpan* spans,
                                   PairSpecials sp, int64_t* tokens) {
  const PackedSeq s = seqs[blockIdx.x];
  const PairSpan p = spans[blockIdx.x];
  for (int pos = threadIdx.x; pos < s.len; pos += blockDim.x) {
    int k = pos;
    int32_t id;
    if (k < sp.n_prefix) id = special_id(sp.prefix, k);
    else if ((k -= sp.n_prefix) < p.a_len) id = a[p.a0 + k];
    else if ((k -= p.a_len) < p.b_len) id = b[p.b0 + k];
    else id = special_id(sp.suffix, k - p.b_len);
    tokens[s.row0 + pos] = id;
  }
}

// out[b, o] = sum_i in[b, i] * W[o, i]  (bias-free LinearHead).  One warp per (o, group of 8 rows).
__global__ void __launch_bounds__(256) head_kernel(const float* in, const float* W, int B, int Hin, int Hout, float* out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int groups = (B + 7) / 8;
  if (warp >= Hout * groups) return;
  const int o = warp % Hout, g = warp / Hout;
  const float* w = W + static_cast<int64_t>(o) * Hin;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = lane; i < Hin; i += 32) {
    const float wv = __ldg(w + i);
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int b = g * 8 + u;
      if (b < B) acc[u] = fmaf(in[static_cast<int64_t>(b) * Hin + i], wv, acc[u]);
    }
  }
#pragma unroll
  for (int u = 0; u < 8; ++u) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) acc[u] += __shfl_xor_sync(0xffffffffu, acc[u], s);
    const int b = g * 8 + u;
    if (lane == 0 && b < B) out[static_cast<int64_t>(b) * Hout + o] = acc[u];
  }
}

// F.normalize(x, dim=1) = x / max(||x||_2, 1e-12) (optional) and store as fp32 / bf16 / fp16 (round to nearest even from
// the fp32 value, so an fp16 output is bitwise the rounding of the fp32 output of the same call) with a row pitch
template <typename OutT>
__global__ void finish_reps_kernel(const float* in, int B, int D, int normalize, OutT* out, int64_t pitch) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  const float* src = in + static_cast<int64_t>(b) * D;
  float scale = 1.f;
  if (normalize) {
    float q = 0.f;
    for (int i = lane; i < D; i += 32) q = fmaf(src[i], src[i], q);
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) q += __shfl_xor_sync(0xffffffffu, q, s);
    scale = 1.0f / fmaxf(sqrtf(q), 1e-12f);
  }
  for (int i = lane; i < D; i += 32) out[static_cast<int64_t>(b) * pitch + i] = static_cast<OutT>(src[i] * scale);
}

// OM_I8 output: the values finish_reps_kernel<float> stores, quantised into int8 index rows (quant_i8.cuh), one warp per row
__global__ void finish_reps_i8_kernel(const float* in, int B, int D, int normalize, int8_t* out, int64_t pitch) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  const float* src = in + static_cast<int64_t>(b) * D;
  float scale = 1.f;
  if (normalize) {
    float q = 0.f;
    for (int i = lane; i < D; i += 32) q = fmaf(src[i], src[i], q);
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) q += __shfl_xor_sync(0xffffffffu, q, s);
    scale = 1.0f / fmaxf(sqrtf(q), 1e-12f);
  }
  quantize_row_i8([&](int i) { return __fmul_rn(src[i], scale); }, D, i8_dpad(D), out + static_cast<int64_t>(b) * pitch, lane);
}

__global__ void f32_to_bf16_kernel(const float* src, __nv_bfloat16* dst, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] = __float2bfloat16(src[i]);
}

// T5 relative-position bucket (bidirectional), same fp32 arithmetic as modeling_t5.py:188-234
static int t5_bucket(int rel, int num_buckets, int max_distance) {
  const int nb = num_buckets / 2;
  const int out = rel > 0 ? nb : 0;
  const int n = rel < 0 ? -rel : rel;
  const int max_exact = nb / 2;
  if (n < max_exact) return out + n;
  const float v = logf(static_cast<float>(n) / static_cast<float>(max_exact)) /
                  static_cast<float>(log(static_cast<double>(max_distance) / static_cast<double>(max_exact))) *
                  static_cast<float>(nb - max_exact);
  int large = max_exact + static_cast<int>(v);
  if (large > nb - 1) large = nb - 1;
  return out + large;
}

}  // namespace om

using namespace om;

// ===================================================================================================
// host side
// ===================================================================================================
struct LayerW {
  __nv_bfloat16 *wqkv = nullptr, *wo = nullptr, *w1 = nullptr, *w2 = nullptr;  // [3I,H] [H,I] [F,H] [H,F]
  float *bqkv = nullptr, *bo = nullptr, *b1 = nullptr, *b2 = nullptr;          // BERT only
  float *ln1_g = nullptr, *ln1_b = nullptr, *ln2_g = nullptr, *ln2_b = nullptr;  // BERT: post-attn / post-ffn LN
                                                                                 // T5  : pre-attn / pre-ffn RMS (g only)
  // normalisation folded into the consuming GEMM (om_encoder_finalize): wqkv / w1 hold W diag(gamma) in bf16 (rows
  // centred for LayerNorm), b*_fold = W beta + b (BERT); fp32 staging freed after folding
  float *wqkv_f32 = nullptr, *w1_f32 = nullptr;
  float *bqkv_fold = nullptr, *b1_fold = nullptr;
};

// One parameter a handle takes (om_encoder_set_weight): its canonical HF name, its shape ([rows] when cols < 0), where
// it lands (fp32 and / or bf16; bf16 only is converted through a temporary fp32 copy) and whether it has been set.
struct Param {
  std::string name;
  int64_t rows, cols;
  float* f32;
  __nv_bfloat16* bf16;
  bool set;
  size_t count() const { return static_cast<size_t>(rows) * (cols < 0 ? 1 : cols); }
};

struct om_encoder {
  om_encoder_desc d;
  int dh = 0;  // head width: 64, or 32 (BERT)
  int I = 0;   // heads * dh
  std::vector<LayerW> layers;
  float *word = nullptr, *pos = nullptr, *type = nullptr, *emb_g = nullptr, *emb_b = nullptr;  // BERT embeddings
  float* final_g = nullptr;                                                                    // T5 final RMSNorm
  float* rel_w = nullptr;         // T5, MPNet [buckets, heads]
  float* relbias_log2 = nullptr;  // [heads, 255]
  float* relbias_long_log2 = nullptr;  // [heads, 1023] (sequences longer than one tile)
  float* head_w = nullptr;        // [head_out, H]
  std::vector<Param> params;      // in the order om_encoder_finalize lists missing ones: embeddings, layers, head
  bool finalized = false;         // the weights are folded: no more om_encoder_set_weight
  // workspace
  int Tmax = 0, Tld = 0;
  float *h = nullptr, *kmask = nullptr, *pooled = nullptr, *headed = nullptr;
  __nv_bfloat16 *xb = nullptr, *qk = nullptr, *vt = nullptr, *ctx = nullptr, *inter = nullptr;
  float* stats[2] = {nullptr, nullptr};  // [Tmax, kStatParts, 2] row statistics of the residual stream (ping-pong)
  // packed calls: the sequence table of one chunk (device, and its pinned staging copy) and the row map of one row group
  PackedSeq* pk_seqs = nullptr;     // [Tmax]
  PackedSeq* pk_host = nullptr;     // [Tmax], pinned host memory
  cudaEvent_t pk_copied = nullptr;  // recorded after the last upload from pk_host
  int2* rowmap = nullptr;           // [Tmax]
  // pair calls (om_encode_pairs), allocated on the first one: the span table of one chunk (device, and its pinned staging
  // copy, uploaded under pk_copied) and the token stream of one row group
  PairSpan* pr_spans = nullptr;  // [Tmax]
  PairSpan* pr_host = nullptr;   // [Tmax], pinned host memory
  int64_t* pr_tokens = nullptr;  // [Tmax]
  int32_t* pos_ids = nullptr;    // [Tmax] RoBERTa / MPNet position id per layout row (roberta_pos_kernel); their handles only
  std::vector<void*> allocs;
};

namespace {

// BERT's post-LN encoder: RoBERTa with position ids computed from the token ids (roberta_pos_kernel), MPNet with those
// position ids and a relative position bias, DistilBERT under other parameter names; MPNet and DistilBERT have no
// token-type embeddings
bool bert_like(int arch) {
  return arch == OM_ARCH_BERT || arch == OM_ARCH_ROBERTA || arch == OM_ARCH_MPNET || arch == OM_ARCH_DISTILBERT;
}
bool has_token_types(int arch) { return arch == OM_ARCH_BERT || arch == OM_ARCH_ROBERTA; }
bool ids_positions(int arch) { return arch == OM_ARCH_ROBERTA || arch == OM_ARCH_MPNET; }
// a relative position bias shared by all layers, added to the scaled logits (relbias_log2 / relbias_long_log2)
bool has_relbias(int arch) { return arch == OM_ARCH_T5ENC || arch == OM_ARCH_MPNET; }

// The longest sequence the architecture and its position table allow: 8192 tokens and max_position_embeddings (BERT,
// DistilBERT) / max_position_embeddings - 2 (RoBERTa: positions start at padding_idx + 1 = 2); 512 tokens for T5 and
// MPNet (their relative-bias tables cover 512; MPNet also within max_position_embeddings - 2).  seq_limit_name names
// these limits for error messages.
int max_seq_len(const om_encoder_desc& d) {
  if (d.arch == OM_ARCH_T5ENC) return kMaxLongL;
  if (d.arch == OM_ARCH_MPNET) return std::min(kMaxLongL, d.max_pos - 2);
  return std::min(kMaxStreamL, d.arch == OM_ARCH_ROBERTA ? d.max_pos - 2 : d.max_pos);
}

const char* seq_limit_name(int arch) {
  return arch == OM_ARCH_ROBERTA                                ? "8192 tokens, max_position_embeddings - 2"
         : arch == OM_ARCH_BERT || arch == OM_ARCH_DISTILBERT ? "8192 tokens, max_position_embeddings"
         : arch == OM_ARCH_MPNET                                ? "512 tokens, max_position_embeddings - 2 (MPNet)"
                                                                : "512 tokens (T5)";
}

template <typename T>
int dev_alloc(om_encoder* e, T** p, size_t count) {
  void* q = nullptr;
  OM_CUDA(dev_malloc(&q, std::max<size_t>(count, 1) * sizeof(T)));
  e->allocs.push_back(q);
  *p = static_cast<T*>(q);
  return 0;
}

// frees one of the handle's allocations before the handle itself
void dev_free(om_encoder* e, void* p) {
  e->allocs.erase(std::find(e->allocs.begin(), e->allocs.end(), p));
  cudaFree(p);
}

// copies a fp32 [rows, cols] block (host or device) into dst (+ optional bf16 conversion).  om_encoder_set_weight has no
// stream: device data may still be in flight on any of the caller's streams (e.g. an optimizer step on a non-blocking
// stream), so the copy runs after all work issued so far, and it has finished on return, when the caller may free or
// overwrite the source.
int upload(const void* data, om_memkind kind, size_t count, float* dst_f32, __nv_bfloat16* dst_bf16) {
  if (kind == OM_DEVICE) OM_CUDA(cudaDeviceSynchronize());
  float* staged = dst_f32;
  float* tmp = nullptr;
  if (!staged) {
    OM_CUDA(cudaMalloc(&tmp, count * sizeof(float)));
    staged = tmp;
  }
  cudaError_t err =
      cudaMemcpy(staged, data, count * sizeof(float), kind == OM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice);
  if (err == cudaSuccess && dst_bf16) {
    f32_to_bf16_kernel<<<static_cast<int>(std::min<size_t>((count + 255) / 256, 4096)), 256>>>(staged, dst_bf16,
                                                                                              (int64_t)count);
    err = cudaGetLastError();
  }
  if (err == cudaSuccess) err = cudaDeviceSynchronize();
  if (tmp) cudaFree(tmp);
  if (err != cudaSuccess) return fail(OM_ECUDA, "weight upload failed: %s", cudaGetErrorString(err));
  return 0;
}

// The attention kernels of one head width, each with the dynamic shared memory it runs with: attn_opt_in raises their
// shared-memory limits, attn_launch runs one layer's attention over the tiles encode_layers describes.
template <int DH>
cudaError_t attn_opt_in() {
  const auto smem = cudaFuncAttributeMaxDynamicSharedMemorySize;
  cudaError_t err = cudaFuncSetAttribute(attn_stream_kernel<DH, false>, smem, kAttnStreamSmemBytes);
  if (DH == 64 && err == cudaSuccess) err = cudaFuncSetAttribute(attn_stream_kernel<64, true>, smem, kAttnStreamSmemBytes);
  if (err == cudaSuccess) err = cudaFuncSetAttribute(attn_kernel<DH>, smem, kAttnSmemBytes);
  return err;
}

template <int DH>
void attn_launch(const CUtensorMap& tmQK, const CUtensorMap& tmVt, const AttnParams& ap_stream, int n_stream,
                 const AttnParams& ap_short, int n_short, int units, int sms, cudaStream_t st) {
  if (n_stream > 0)
    (DH == 64 && ap_stream.relbias_log2 ? attn_stream_kernel<64, true> : attn_stream_kernel<DH, false>)
        <<<dim3(n_stream, units), kAttnStreamThreads, kAttnStreamSmemBytes, st>>>(tmQK, tmVt, ap_stream);
  if (n_short > 0)
    attn_kernel<DH><<<std::min(n_short * units, sms * kAttnCtasPerSm), 128, kAttnSmemBytes, st>>>(tmQK, tmVt, ap_short,
                                                                                                 n_short, units);
}

// The layers and the final normalisation over T token rows whose embedding (e->h, e->xb, e->stats[0]) and key mask
// (e->kmask) are in place.  Attention: tiles [0, n_stream) run attn_stream_kernel with ap_stream, the next n_short
// tiles attn_kernel with ap_short (tile0 = n_stream); ap_short.Tvalid_rows is the tile-local V^T layout of EpiQKV.
int encode_layers(om_encoder* e, int T, const AttnParams& ap_stream, int n_stream, const AttnParams& ap_short,
                  int n_short, int sms, cudaStream_t st) {
  const om_encoder_desc& d = e->d;
  const int H = d.hidden, I = e->I, F = d.ffn;
  const bool bert = bert_like(d.arch);
  const int rows4 = (T + 3) / 4;
  const int n_tiles = n_stream + n_short;
  CUtensorMap tmQK, tmVt;
  if (make_tmap_bf16_2d(&tmQK, e->qk, (uint64_t)2 * I, (uint64_t)T, (uint64_t)2 * I * 2, 64, 128) != 0 ||
      make_tmap_bf16_2d(&tmVt, e->vt, (uint64_t)n_tiles * 128, (uint64_t)I, (uint64_t)e->Tld * 2, 64, 64) != 0)
    return fail(OM_ECUDA, "om_encode: tensor map creation failed");

  // TMA-store tensor maps of the bf16 GEMM outputs (box = 64 columns x 32 rows = one epilogue warp's chunk pair) and the
  // residual stream's maps (fp32 load + store, bf16 store; box = 32 columns x 32 rows = one chunk)
  CUtensorMap tmQKout, tmInter, tmS, tmXb;
  if (make_tmap_bf16_2d(&tmQKout, e->qk, (uint64_t)2 * I, (uint64_t)T, (uint64_t)2 * I * 2, 64, 32) != 0 ||
      make_tmap_bf16_2d(&tmInter, e->inter, (uint64_t)F, (uint64_t)T, (uint64_t)F * 2, 64, 32) != 0 ||
      make_tmap_2d(&tmS, e->h, 4, (uint64_t)H, (uint64_t)T, (uint64_t)H * 4, 32, 32, 128) != 0 ||
      make_tmap_2d(&tmXb, e->xb, 2, (uint64_t)H, (uint64_t)T, (uint64_t)H * 2, 32, 32, 64) != 0)
    return fail(OM_ECUDA, "om_encode: output tensor map creation failed");
  const float inv_h = 1.0f / static_cast<float>(H);
  const int rms = bert ? 0 : 1;
  const RowNorm normA{e->stats[0], inv_h, d.ln_eps, rms}, normB{e->stats[1], inv_h, d.ln_eps, rms};
  const RowNorm ident{nullptr, inv_h, d.ln_eps, rms};
  // 128 x 128 tiles, 3-stage ring: the staged fp32 accumulator tile (66 KB) and the functors' shared memory leave room for
  // three 32 KB stages within the 227 KB an H100 block may use.  8 epilogue warps = 2 column groups per tile ->
  // (H / 128) * 2 <= kStatParts statistics slots for the residual GEMMs.
  auto wide_gemm = [&](const __nv_bfloat16* A, int K, const __nv_bfloat16* W, int M, int N, const auto& epi) -> cudaError_t {
    return launch_gemm<128, 3, false>(A, K, W, K, M, N, K, epi, sms, st);
  };
  auto resid_gemm = [&](const __nv_bfloat16* A, int K, const __nv_bfloat16* W, const EpiResidNorm& epi) -> cudaError_t {
    return launch_gemm<128, 3, false>(A, K, W, K, T, H, K, epi, sms, st);
  };
  if (((H + 127) / 128) * 2 > kStatParts)
    return fail(OM_EINVAL, "om_encode: hidden=%d needs more statistics slots than kStatParts", H);
  for (int li = 0; li < d.layers; ++li) {
    const LayerW& w = e->layers[li];
    NvtxRange nvtx_layer("om.encode.layer");
    // LayerNorm that produced this layer's input (BERT; applied on the fly wherever the input is consumed)
    const float* g_in = bert ? (li == 0 ? e->emb_g : e->layers[li - 1].ln2_g) : nullptr;
    const float* b_in = bert ? (li == 0 ? e->emb_b : e->layers[li - 1].ln2_b) : nullptr;
    {
      EpiQKV epi{tmQKout, e->qk, e->vt, e->Tld, bert ? w.bqkv_fold : nullptr, T, 2 * I, ap_short.Tvalid_rows, normA};
      cudaError_t err = wide_gemm(e->xb, H, w.wqkv, T, 3 * I, epi);
      if (err != cudaSuccess) return fail(OM_ECUDA, "QKV GEMM launch failed: %s", cudaGetErrorString(err));
    }
    const int units = I / kAttnCols;  // work items per tile: one per 64-wide head or pair of 32-wide heads
    (e->dh == 64 ? attn_launch<64> : attn_launch<32>)(tmQK, tmVt, ap_stream, n_stream, ap_short, n_short, units, sms, st);
    OM_CUDA(cudaGetLastError());
    {
      // s <- ctx Wo^T + bo + LN_in(s) (BERT) / + s (T5); statistics of the new s -> stats[1]
      EpiResidNorm epi{tmS, tmXb, bert ? w.bo : nullptr, bert ? normA : ident, g_in, b_in, e->stats[1], 2, T, H, 128};
      cudaError_t err = resid_gemm(e->ctx, I, w.wo, epi);
      if (err != cudaSuccess) return fail(OM_ECUDA, "O-proj GEMM launch failed: %s", cudaGetErrorString(err));
    }
    {
      cudaError_t err;
      if (bert) {
        EpiBiasActBf16<ACT_GELU> epi{tmInter, e->inter, F, w.b1_fold, T, F, normB};
        err = wide_gemm(e->xb, H, w.w1, T, F, epi);
      } else {
        EpiBiasActBf16<ACT_RELU> epi{tmInter, e->inter, F, nullptr, T, F, normB};
        err = wide_gemm(e->xb, H, w.w1, T, F, epi);
      }
      if (err != cudaSuccess) return fail(OM_ECUDA, "FFN1 GEMM launch failed: %s", cudaGetErrorString(err));
    }
    {
      // s <- inter W2^T + b2 + LN_attn(s) (BERT) / + s (T5); statistics -> stats[0] (the next layer's input)
      EpiResidNorm epi{tmS, tmXb, bert ? w.b2 : nullptr, bert ? normB : ident, w.ln1_g, w.ln1_b, e->stats[0], 2, T, H, 128};
      cudaError_t err = resid_gemm(e->inter, F, w.w2, epi);
      if (err != cudaSuccess) return fail(OM_ECUDA, "FFN2 GEMM launch failed: %s", cudaGetErrorString(err));
    }
  }
  // the one normalisation that runs as a kernel: last_hidden_state = LN_out(s) (BERT: last layer's output.LayerNorm,
  // T5: final_layer_norm), in place in e->h, for pooling and the optional out_hidden copy
  if (bert)
    norm_kernel<false><<<rows4, 128, 0, st>>>(e->h, e->layers[d.layers - 1].ln2_g, e->layers[d.layers - 1].ln2_b,
                                              d.ln_eps, T, H, e->h);
  else
    norm_kernel<true><<<rows4, 128, 0, st>>>(e->h, e->final_g, nullptr, d.ln_eps, T, H, e->h);
  OM_CUDA(cudaGetLastError());
  return 0;
}

// Embeds T layout rows into e->h / e->xb / e->stats[0]: the padded rows of nseq sequences of L tokens (seqs == nullptr),
// or the rows of a packed group (its sequence table seqs, L = 0, and the row map e->rowmap).  RoBERTa and MPNet first
// compute the position ids from the token ids, as HF does per sequence.  MPNet and DistilBERT ignore token_type_ids:
// every row adds the zeroed single row of e->type.
int embed_rows(om_encoder* e, const int64_t* ids, const int64_t* tts, int T, int L, const PackedSeq* seqs, int nseq,
               cudaStream_t st) {
  const om_encoder_desc& d = e->d;
  const bool types = has_token_types(d.arch);
  const int H = d.hidden, rows4 = (T + 3) / 4, type_vocab = types ? std::max(d.type_vocab, 1) : 1;
  if (!types) tts = nullptr;
  const int2* rowmap = seqs ? e->rowmap : nullptr;
  const int Lrow = seqs ? kMaxL : L;  // packed rows take their positions from the row map
  if (ids_positions(d.arch)) {
    roberta_pos_kernel<<<(nseq + 3) / 4, 128, 0, st>>>(ids, nseq, L, seqs, e->pos_ids);
    bert_embed_kernel<true><<<rows4, 128, 0, st>>>(ids, tts, e->word, e->type, e->pos, T, Lrow, H, d.vocab, type_vocab,
                                                   e->h, e->xb, e->stats[0], rowmap, seqs, e->pos_ids);
  } else if (bert_like(d.arch)) {
    bert_embed_kernel<false><<<rows4, 128, 0, st>>>(ids, tts, e->word, e->type, e->pos, T, Lrow, H, d.vocab, type_vocab,
                                                    e->h, e->xb, e->stats[0], rowmap, seqs, nullptr);
  } else {
    t5_embed_kernel<<<rows4, 128, 0, st>>>(ids, e->word, T, H, d.vocab, e->h, e->xb, e->stats[0], rowmap, seqs);
  }
  OM_CUDA(cudaGetLastError());
  return 0;
}

// the output arguments of the om_encode* entry points (who: the entry point, for the messages)
int check_out(const om_encoder* e, const char* who, const void* out_reps, om_dtype out_dtype, int64_t out_row_stride) {
  if (!out_reps) return fail(OM_EINVAL, "%s: null argument", who);
  if (!e->finalized) return fail(OM_ESTATE, "%s: call om_encoder_finalize first", who);
  if (out_dtype != OM_F32 && out_dtype != OM_BF16 && out_dtype != OM_F16 && out_dtype != OM_I8)
    return fail(OM_EINVAL, "%s: out dtype must be f32, bf16, f16 or i8", who);
  if (out_row_stride < om_encoder_rep_dim(e)) return fail(OM_EINVAL, "%s: out_row_stride < rep_dim", who);
  if (out_dtype == OM_I8 && (out_row_stride < i8_dpad(om_encoder_rep_dim(e)) + 16 || out_row_stride % 4 != 0 ||
                             reinterpret_cast<uintptr_t>(out_reps) % 4 != 0))
    return fail(OM_EINVAL, "%s: int8 rows need a 4-byte aligned out_reps and an out_row_stride that is a multiple of 4 and "
                "at least %d bytes (rep_dim rounded up to 16, + 16 for the scale)", who, i8_dpad(om_encoder_rep_dim(e)) + 16);
  return 0;
}

// softmax scale * log2(e) of the attention logits: BERT divides them by sqrt(head width) (1/8 for 64, 1/sqrt(32) for 32,
// applied to the fp32 scores), T5 does not scale them
float attn_scale_log2(const om_encoder* e) {
  const float scale = bert_like(e->d.arch) ? static_cast<float>(1.0 / sqrt(static_cast<double>(e->dh))) : 1.0f;
  return scale * kLog2e;
}

// pooled [B, hidden] (e->pooled) -> optional head -> optional normalise -> out_reps rows [B, rep_dim] at out_row_stride
int finish_reps(om_encoder* e, int B, void* out_reps, om_dtype out_dtype, int64_t out_row_stride, cudaStream_t st) {
  const om_encoder_desc& d = e->d;
  const int H = d.hidden, rep_dim = om_encoder_rep_dim(e);
  const float* reps = e->pooled;
  if (d.has_head) {
    const int warps = d.head_out * ((B + 7) / 8);
    head_kernel<<<(warps * 32 + 255) / 256, 256, 0, st>>>(e->pooled, e->head_w, B, H, d.head_out, e->headed);
    reps = e->headed;
  }
  if (out_dtype == OM_F32)
    finish_reps_kernel<float><<<(B + 3) / 4, 128, 0, st>>>(reps, B, rep_dim, d.normalize, static_cast<float*>(out_reps),
                                                          out_row_stride);
  else if (out_dtype == OM_I8)
    finish_reps_i8_kernel<<<(B + 3) / 4, 128, 0, st>>>(reps, B, rep_dim, d.normalize, static_cast<int8_t*>(out_reps),
                                                       out_row_stride);
  else if (out_dtype == OM_BF16)
    finish_reps_kernel<__nv_bfloat16><<<(B + 3) / 4, 128, 0, st>>>(reps, B, rep_dim, d.normalize,
                                                                  static_cast<__nv_bfloat16*>(out_reps), out_row_stride);
  else
    finish_reps_kernel<__half><<<(B + 3) / 4, 128, 0, st>>>(reps, B, rep_dim, d.normalize, static_cast<__half*>(out_reps),
                                                           out_row_stride);
  OM_CUDA(cudaGetLastError());
  return 0;
}

// Placement of the n sequences of one packed chunk (lengths len[0..n), token offsets tok0[0..n), each length <= Tmax):
//   * a sequence of more than 128 tokens starts on a tile boundary and takes ceil(l / 128) tiles, in input order;
//   * the others are bin-packed whole into tiles of min(128, Tmax) rows, first-fit decreasing (ties by input index:
//     placement is a deterministic function of the lengths), each bin's sequences back to back in insertion order;
//   * layout = the tiles of the sequences of more than 128 tokens (attn_stream_kernel), then the bins (attn_kernel);
//     cut into row groups of at most Tmax rows at unit (sequence / bin) boundaries, each group encoded on its own (in
//     the same order).  The last unit of a group is counted up to its last token.
// seqs receives the table in layout order (row0 relative to its group, out = index in the chunk).
struct PackedGroup {
  int k0, k1;     // sequences [k0, k1) of the table
  int T;          // layout rows of the group
  int n_stream;   // tiles of sequences of more than kMaxL tokens (the first tiles of the group)
  int n_tiles;
};

void place_packed(const int32_t* len, const int64_t* tok0, int n, int Tmax, std::vector<PackedSeq>& seqs,
                  std::vector<PackedGroup>& groups) {
  seqs.clear();
  groups.clear();
  const int cap = std::min(kMaxL, Tmax);
  std::vector<int> streams, shorts;
  for (int i = 0; i < n; ++i) (len[i] > kMaxL ? streams : shorts).push_back(i);
  std::stable_sort(shorts.begin(), shorts.end(), [&](int a, int b) { return len[a] > len[b]; });
  std::vector<std::vector<int>> bins;
  std::vector<int> fill;
  std::vector<std::set<int>> by_room(cap + 1);  // open bins by free rows
  for (int i : shorts) {
    int best = -1;  // first fit: the lowest-numbered bin with room
    for (int r = len[i]; r <= cap; ++r)
      if (!by_room[r].empty() && (best < 0 || *by_room[r].begin() < best)) best = *by_room[r].begin();
    if (best < 0) {
      best = static_cast<int>(bins.size());
      bins.emplace_back();
      fill.push_back(0);
    } else {
      by_room[cap - fill[best]].erase(best);
    }
    bins[best].push_back(i);
    fill[best] += len[i];
    by_room[cap - fill[best]].insert(best);
  }
  PackedGroup g{0, 0, 0, 0, 0};
  int row = 0;  // group-local first row of the next unit (a tile boundary)
  auto unit = [&](const std::vector<int>& members, int tiles, int used, bool stream) {
    if (row > 0 && row + (tiles - 1) * 128 + used > Tmax) {
      g.k1 = static_cast<int>(seqs.size());
      groups.push_back(g);
      g = PackedGroup{g.k1, g.k1, 0, 0, 0};
      row = 0;
    }
    int off = 0;
    for (int i : members) {
      seqs.push_back(PackedSeq{row + off, len[i], i, 0, tok0[i]});
      off += len[i];
    }
    g.T = row + (tiles - 1) * 128 + used;
    g.n_stream += stream ? tiles : 0;
    g.n_tiles += tiles;
    row += tiles * 128;
  };
  for (int i : streams) {
    const int tiles = (len[i] + 127) / 128;
    unit(std::vector<int>{i}, tiles, len[i] - (tiles - 1) * 128, true);
  }
  for (size_t b = 0; b < bins.size(); ++b) unit(bins[b], 1, fill[b], false);
  g.k1 = static_cast<int>(seqs.size());
  if (g.k1 > g.k0) groups.push_back(g);
}

// pair input of one packed chunk (om_encode_pairs): the two token stores, the chunk's spans in layout order (host) and
// the special ids
struct PairChunk {
  const int32_t* a;
  const int32_t* b;
  const PairSpan* spans;
  PairSpecials sp;
};

// Encodes one chunk of a packed call (its n sequences placed by place_packed into seqs / groups) into out rows [0, n):
// uploads the sequence table, then per row group the row map, the embedding, the layers and the pooling; then the
// output tail.  pairs != nullptr: each row group's token stream is first assembled from the pair stores into pr_tokens
// (the table's tok0 = row0, tokens = token_type_ids = nullptr).
int encode_packed_chunk(om_encoder* e, const int64_t* tokens, const int64_t* token_type_ids,
                        const std::vector<PackedSeq>& seqs, const std::vector<PackedGroup>& groups, const PairChunk* pairs,
                        int n, void* out_reps, om_dtype out_dtype, int64_t out_row_stride, float* out_hidden, int sms,
                        cudaStream_t st) {
  const om_encoder_desc& d = e->d;
  const bool rel = has_relbias(d.arch);
  const int H = d.hidden;
  // upload the tables through the pinned staging buffers: wait (on the host) only until the previous upload from them
  // has been read
  OM_CUDA(cudaEventSynchronize(e->pk_copied));
  memcpy(e->pk_host, seqs.data(), seqs.size() * sizeof(PackedSeq));
  OM_CUDA(cudaMemcpyAsync(e->pk_seqs, e->pk_host, seqs.size() * sizeof(PackedSeq), cudaMemcpyHostToDevice, st));
  if (pairs) {
    memcpy(e->pr_host, pairs->spans, seqs.size() * sizeof(PairSpan));
    OM_CUDA(cudaMemcpyAsync(e->pr_spans, e->pr_host, seqs.size() * sizeof(PairSpan), cudaMemcpyHostToDevice, st));
    tokens = e->pr_tokens;
  }
  OM_CUDA(cudaEventRecord(e->pk_copied, st));
  AttnParams ap;
  ap.L = 128;  // unused: every row's key range comes from the row map
  ap.spt = 1;
  ap.I = e->I;
  ap.Tvalid_rows = 128;
  ap.scale_log2 = attn_scale_log2(e);
  ap.kmask = e->kmask;
  ap.ctx = e->ctx;
  ap.rowmap = e->rowmap;
  for (const PackedGroup& g : groups) {
    const PackedSeq* gs = e->pk_seqs + g.k0;
    const int ns = g.k1 - g.k0, T = g.T, rows4 = (T + 3) / 4;
    if (pairs)
      pair_tokens_kernel<<<ns, 128, 0, st>>>(pairs->a, pairs->b, gs, e->pr_spans + g.k0, pairs->sp, e->pr_tokens);
    packed_rowmap_kernel<<<(T + 255) / 256, 256, 0, st>>>(gs, ns, T, e->rowmap, e->kmask);
    // (for pairs, RoBERTa's and MPNet's positions come from the stream pair_tokens_kernel assembled)
    OM_TRY(embed_rows(e, tokens, token_type_ids, T, 0, gs, ns, st));
    ap.T = T;
    ap.seqs = gs;
    AttnParams ap_stream = ap, ap_short = ap;
    ap_stream.relbias_log2 = rel ? e->relbias_long_log2 : nullptr;
    ap_short.relbias_log2 = rel ? e->relbias_log2 : nullptr;
    ap_short.tile0 = g.n_stream;
    OM_TRY(encode_layers(e, T, ap_stream, g.n_stream, ap_short, g.n_tiles - g.n_stream, sms, st));
    if (out_hidden) gather_packed_rows_kernel<<<rows4, 128, 0, st>>>(e->h, e->rowmap, gs, T, H, out_hidden);
    pool_packed_kernel<<<ns, 256, 0, st>>>(e->h, gs, H, d.pooling == OM_POOL_MEAN ? 1 : 0, e->pooled);
    OM_CUDA(cudaGetLastError());
  }
  return finish_reps(e, n, out_reps, out_dtype, out_row_stride, st);
}

// the packed length limit: max_seq_len and max_batch_tokens
int packed_max_len(const om_encoder* e) { return std::min(max_seq_len(e->d), e->Tmax); }

}  // namespace

extern "C" {

int om_encoder_create(const om_encoder_desc* desc, om_encoder** out) {
  if (!desc || !out) return fail(OM_EINVAL, "om_encoder_create: null argument");
  OM_TRY(device_sm_count());
  const om_encoder_desc& d = *desc;
  if (!bert_like(d.arch) && d.arch != OM_ARCH_T5ENC) return fail(OM_EINVAL, "unknown arch %d", d.arch);
  if (ids_positions(d.arch) && d.max_pos < 3)
    return fail(OM_EINVAL, "%s max_position_embeddings=%d unsupported (at least 3: positions start at 2)",
                d.arch == OM_ARCH_MPNET ? "MPNet" : "RoBERTa", d.max_pos);
  if (d.hidden <= 0 || d.hidden % 128 != 0 || d.hidden > 1024)
    return fail(OM_EINVAL, "hidden=%d unsupported (multiple of 128, <= 1024)", d.hidden);
  if (d.heads <= 0) return fail(OM_EINVAL, "heads=%d must be positive", d.heads);
  // head width: BERT's is hidden / heads, 32 or 64; T5's (d_kv) is 64
  if (bert_like(d.arch) && d.hidden % d.heads != 0)
    return fail(OM_EINVAL, "BERT requires hidden to be a multiple of heads (got hidden=%d heads=%d)", d.hidden, d.heads);
  const int dh = bert_like(d.arch) ? d.hidden / d.heads : 64;
  if (dh != 32 && dh != 64)
    return fail(OM_EINVAL, "BERT head width hidden/heads=%d unsupported (32 or 64; hidden=%d heads=%d)", dh, d.hidden,
                d.heads);
  // the relative position bias exists in the 64-wide attention instantiations only
  if (d.arch == OM_ARCH_MPNET && dh != 64)
    return fail(OM_EINVAL, "MPNet head width hidden/heads=%d unsupported (64 only; hidden=%d heads=%d)", dh, d.hidden,
                d.heads);
  if (d.arch == OM_ARCH_MPNET && (d.rel_buckets != 32 || d.rel_max_distance != 128))
    return fail(OM_EINVAL, "MPNet needs rel_buckets=32 and rel_max_distance=128 (got %d, %d)", d.rel_buckets,
                d.rel_max_distance);
  if (d.heads * dh > 2048 || (d.heads * dh) % 128 != 0)
    return fail(OM_EINVAL, "heads=%d unsupported (heads * head width %d must be a multiple of 128, at most 2048)", d.heads,
                dh);
  if (d.ffn <= 0 || d.ffn % 64 != 0) return fail(OM_EINVAL, "ffn=%d must be a positive multiple of 64", d.ffn);
  if (d.layers <= 0 || d.vocab <= 0) return fail(OM_EINVAL, "layers/vocab must be positive");
  if (d.has_head && (d.head_out <= 0)) return fail(OM_EINVAL, "head_out must be positive when has_head=1");
  if (d.max_batch_tokens <= 0) return fail(OM_EINVAL, "max_batch_tokens must be positive");
  om_encoder* e = new (std::nothrow) om_encoder();
  if (!e) return fail(OM_ENOMEM, "out of host memory");
  e->d = d;
  e->dh = dh;
  e->I = d.heads * dh;
  const int H = d.hidden, I = e->I, F = d.ffn;
  const bool bert = bert_like(d.arch);
  e->layers.resize(d.layers);
  int rc = 0;
  auto A = [&](auto** p, size_t n) {
    if (rc == 0) rc = dev_alloc(e, p, n);
  };
  // a parameter of shape [rows] (cols < 0) or [rows, cols] landing in *f32 and / or *bf16, allocated here unless it
  // already is: slot >= 0 makes it one of three q / k / v slices of its buffer
  auto param = [&](std::string name, int64_t rows, int64_t cols, float** f32, __nv_bfloat16** bf16, int slot = -1) {
    Param p{std::move(name), rows, cols, nullptr, nullptr, false};
    const size_t n = p.count(), off = slot < 0 ? 0 : slot * n;
    if (f32 && !*f32) A(f32, slot < 0 ? n : 3 * n);
    if (bf16 && !*bf16) A(bf16, slot < 0 ? n : 3 * n);
    if (rc != 0) return;
    p.f32 = f32 ? *f32 + off : nullptr;
    p.bf16 = bf16 ? *bf16 + off : nullptr;
    e->params.push_back(std::move(p));
  };
  if (bert) {
    // at least one row: token types are clamped into the table (without token types: one row, zeroed below)
    A(&e->type, (size_t)(has_token_types(d.arch) ? std::max(d.type_vocab, 1) : 1) * H);
    param("embeddings.word_embeddings.weight", d.vocab, H, &e->word, nullptr);
    param("embeddings.position_embeddings.weight", d.max_pos, H, &e->pos, nullptr);
    if (has_token_types(d.arch)) param("embeddings.token_type_embeddings.weight", d.type_vocab, H, &e->type, nullptr);
    param("embeddings.LayerNorm.weight", H, -1, &e->emb_g, nullptr);
    param("embeddings.LayerNorm.bias", H, -1, &e->emb_b, nullptr);
    if (ids_positions(d.arch)) A(&e->pos_ids, (size_t)d.max_batch_tokens);
  } else {
    param("shared.weight", d.vocab, H, &e->word, nullptr);
    param("encoder.final_layer_norm.weight", H, -1, &e->final_g, nullptr);
  }
  if (has_relbias(d.arch)) {
    param(d.arch == OM_ARCH_MPNET ? "encoder.relative_attention_bias.weight"
                                  : "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight",
          d.rel_buckets, d.heads, &e->rel_w, nullptr);
    A(&e->relbias_log2, (size_t)d.heads * (2 * kMaxL - 1));
    A(&e->relbias_long_log2, (size_t)d.heads * (2 * kMaxLongL - 1));
  }
  // each layer's modules, named after "encoder.layer.<i>." (BERT, MPNet) / "transformer.layer.<i>." (DistilBERT) /
  // "encoder.block.<i>." (T5): "<module>.weight" of shape [rows, cols] ([rows] for a norm) into f32 or bf16, and (all
  // but T5) "<module>.bias" of shape [rows].  The QKV and W1 weights land in fp32 staging buffers that
  // om_encoder_finalize folds into wqkv / w1.
  struct LayerModule {
    const char* name;
    int64_t rows, cols;
    float* LayerW::*f32;
    __nv_bfloat16* LayerW::*bf16;
    float* LayerW::*bias;
    int slot;
  };
  const std::vector<LayerModule> modules = d.arch == OM_ARCH_MPNET ? std::vector<LayerModule>{
      {"attention.attn.q", I, H, &LayerW::wqkv_f32, nullptr, &LayerW::bqkv, 0},
      {"attention.attn.k", I, H, &LayerW::wqkv_f32, nullptr, &LayerW::bqkv, 1},
      {"attention.attn.v", I, H, &LayerW::wqkv_f32, nullptr, &LayerW::bqkv, 2},
      {"attention.attn.o", H, I, nullptr, &LayerW::wo, &LayerW::bo, -1},
      {"attention.LayerNorm", H, -1, &LayerW::ln1_g, nullptr, &LayerW::ln1_b, -1},
      {"intermediate.dense", F, H, &LayerW::w1_f32, nullptr, &LayerW::b1, -1},
      {"output.dense", H, F, nullptr, &LayerW::w2, &LayerW::b2, -1},
      {"output.LayerNorm", H, -1, &LayerW::ln2_g, nullptr, &LayerW::ln2_b, -1},
  } : d.arch == OM_ARCH_DISTILBERT ? std::vector<LayerModule>{
      {"attention.q_lin", I, H, &LayerW::wqkv_f32, nullptr, &LayerW::bqkv, 0},
      {"attention.k_lin", I, H, &LayerW::wqkv_f32, nullptr, &LayerW::bqkv, 1},
      {"attention.v_lin", I, H, &LayerW::wqkv_f32, nullptr, &LayerW::bqkv, 2},
      {"attention.out_lin", H, I, nullptr, &LayerW::wo, &LayerW::bo, -1},
      {"sa_layer_norm", H, -1, &LayerW::ln1_g, nullptr, &LayerW::ln1_b, -1},
      {"ffn.lin1", F, H, &LayerW::w1_f32, nullptr, &LayerW::b1, -1},
      {"ffn.lin2", H, F, nullptr, &LayerW::w2, &LayerW::b2, -1},
      {"output_layer_norm", H, -1, &LayerW::ln2_g, nullptr, &LayerW::ln2_b, -1},
  } : bert ? std::vector<LayerModule>{
      {"attention.self.query", I, H, &LayerW::wqkv_f32, nullptr, &LayerW::bqkv, 0},
      {"attention.self.key", I, H, &LayerW::wqkv_f32, nullptr, &LayerW::bqkv, 1},
      {"attention.self.value", I, H, &LayerW::wqkv_f32, nullptr, &LayerW::bqkv, 2},
      {"attention.output.dense", H, I, nullptr, &LayerW::wo, &LayerW::bo, -1},
      {"attention.output.LayerNorm", H, -1, &LayerW::ln1_g, nullptr, &LayerW::ln1_b, -1},
      {"intermediate.dense", F, H, &LayerW::w1_f32, nullptr, &LayerW::b1, -1},
      {"output.dense", H, F, nullptr, &LayerW::w2, &LayerW::b2, -1},
      {"output.LayerNorm", H, -1, &LayerW::ln2_g, nullptr, &LayerW::ln2_b, -1},
  } : std::vector<LayerModule>{
      {"layer.0.SelfAttention.q", I, H, &LayerW::wqkv_f32, nullptr, nullptr, 0},
      {"layer.0.SelfAttention.k", I, H, &LayerW::wqkv_f32, nullptr, nullptr, 1},
      {"layer.0.SelfAttention.v", I, H, &LayerW::wqkv_f32, nullptr, nullptr, 2},
      {"layer.0.SelfAttention.o", H, I, nullptr, &LayerW::wo, nullptr, -1},
      {"layer.0.layer_norm", H, -1, &LayerW::ln1_g, nullptr, nullptr, -1},
      {"layer.1.DenseReluDense.wi", F, H, &LayerW::w1_f32, nullptr, nullptr, -1},
      {"layer.1.DenseReluDense.wo", H, F, nullptr, &LayerW::w2, nullptr, -1},
      {"layer.1.layer_norm", H, -1, &LayerW::ln2_g, nullptr, nullptr, -1},
  };
  for (int i = 0; i < d.layers; ++i) {
    LayerW& w = e->layers[i];
    A(&w.wqkv, (size_t)3 * I * H);
    A(&w.w1, (size_t)F * H);
    if (bert) {
      A(&w.bqkv_fold, (size_t)3 * I);
      A(&w.b1_fold, F);
    }
    const std::string prefix = std::string(d.arch == OM_ARCH_DISTILBERT ? "transformer.layer."
                                           : bert                         ? "encoder.layer."
                                                                          : "encoder.block.") +
                               std::to_string(i) + ".";
    for (const LayerModule& m : modules) {
      param(prefix + m.name + ".weight", m.rows, m.cols, m.f32 ? &(w.*m.f32) : nullptr, m.bf16 ? &(w.*m.bf16) : nullptr,
            m.slot);
      if (m.bias) param(prefix + m.name + ".bias", m.rows, -1, &(w.*m.bias), nullptr, m.slot);
    }
  }
  if (d.has_head) param("head.linear.weight", d.head_out, H, &e->head_w, nullptr);
  // workspace
  e->Tmax = d.max_batch_tokens;
  e->Tld = static_cast<int>(round_up(2 * static_cast<int64_t>(e->Tmax) + 128, 8));  // V^T pitch: <= 128 columns per tile
  const size_t T = e->Tmax;
  A(&e->h, T * H);
  A(&e->kmask, T);
  A(&e->xb, T * H);
  A(&e->qk, T * 2 * I);
  A(&e->vt, (size_t)I * e->Tld);
  A(&e->ctx, T * I);
  A(&e->inter, T * F);
  A(&e->stats[0], T * 2 * kStatParts);
  A(&e->stats[1], T * 2 * kStatParts);
  A(&e->pooled, T * H);  // at most Tmax sequences (L >= 1)
  A(&e->headed, (size_t)e->Tmax * std::max(d.head_out, 1));
  A(&e->pk_seqs, T);
  A(&e->rowmap, T);
  if (rc == 0 && (cudaHostAlloc(&e->pk_host, T * sizeof(PackedSeq), cudaHostAllocDefault) != cudaSuccess ||
                  cudaEventCreateWithFlags(&e->pk_copied, cudaEventDisableTiming) != cudaSuccess)) {
    cudaGetLastError();
    rc = fail(OM_ENOMEM, "om_encoder_create: out of pinned host memory");
  }
  if (rc != 0) {
    om_encoder_destroy(e);
    return rc;
  }
  // statistics slots a GEMM configuration never writes must read as zero (see RowNorm)
  if (cudaMemset(e->stats[0], 0, T * 2 * kStatParts * 4) != cudaSuccess ||
      cudaMemset(e->stats[1], 0, T * 2 * kStatParts * 4) != cudaSuccess ||
      cudaMemset(e->vt, 0, (size_t)I * e->Tld * 2) != cudaSuccess ||
      (bert && !has_token_types(d.arch) && cudaMemset(e->type, 0, (size_t)H * 4) != cudaSuccess)) {
    om_encoder_destroy(e);
    return fail(OM_ECUDA, "workspace memset failed");
  }
  *out = e;
  return 0;
}

void om_encoder_destroy(om_encoder* e) {
  if (!e) return;
  for (void* p : e->allocs) cudaFree(p);
  if (e->pk_host) cudaFreeHost(e->pk_host);
  if (e->pr_host) cudaFreeHost(e->pr_host);
  if (e->pk_copied) cudaEventDestroy(e->pk_copied);
  delete e;
}

int om_encoder_rep_dim(const om_encoder* e) { return e ? (e->d.has_head ? e->d.head_out : e->d.hidden) : 0; }

int om_encoder_set_weight(om_encoder* e, const char* name_c, const void* data, om_memkind kind, const int64_t* shape,
                          int ndim) {
  if (!e || !name_c || !data || !shape) return fail(OM_EINVAL, "om_encoder_set_weight: null argument");
  if (e->finalized) return fail(OM_ESTATE, "om_encoder_set_weight after om_encoder_finalize");
  std::string name(name_c);
  if (name.rfind("bert.", 0) == 0) name = name.substr(5);  // BertFor* checkpoints prefix the backbone
  if (name.rfind("roberta.", 0) == 0) name = name.substr(8);  // and RobertaFor* / XLMRobertaFor* ones
  if (name.rfind("mpnet.", 0) == 0) name = name.substr(6);    // MPNetFor*
  if (name.rfind("distilbert.", 0) == 0) name = name.substr(11);  // DistilBertFor*
  if (name == "encoder.embed_tokens.weight") name = "shared.weight";  // T5EncoderModel's name of the tied embedding
  if (name == "linear.weight") name = "head.linear.weight";           // LinearHead's own state_dict
  // the gated-GELU feed-forward (T5 v1.1, Flan-T5, mT5) has wi_0 / wi_1 where this one has wi: refused, not ignored
  int li = -1, end = 0;
  if (e->d.arch == OM_ARCH_T5ENC &&
      sscanf(name.c_str(), "encoder.block.%d.layer.1.DenseReluDense.wi_%*1[01].weight%n", &li, &end) == 1 &&
      end == static_cast<int>(name.size()) && li >= 0 && li < e->d.layers)
    return fail(OM_EINVAL, "gated-GELU T5 feed-forward (t5 v1.1) is not supported by this build");
  auto p = std::find_if(e->params.begin(), e->params.end(), [&](const Param& q) { return q.name == name; });
  if (p == e->params.end()) return 1;  // e.g. pooler.*: computed by HF, never used by OpenMatch
  const bool vec = p->cols < 0;
  if (ndim != (vec ? 1 : 2) || shape[0] != p->rows || (!vec && shape[1] != p->cols))
    return fail(OM_EINVAL, "om_encoder_set_weight: unexpected shape for '%s'", name_c);
  OM_TRY(upload(data, kind, p->count(), p->f32, p->bf16));
  p->set = true;
  return 0;
}

int om_encoder_finalize(om_encoder* e) {
  if (!e) return fail(OM_EINVAL, "om_encoder_finalize: null encoder");
  if (e->finalized) return fail(OM_ESTATE, "om_encoder_finalize called twice");
  std::string miss;
  int nmiss = 0;
  for (const Param& p : e->params)
    if (!p.set) {
      if (nmiss < 4) miss += (nmiss ? ", " : "") + p.name;
      ++nmiss;
    }
  if (nmiss) return fail(OM_ESTATE, "om_encoder_finalize: %d parameter(s) missing: %s%s", nmiss, miss.c_str(), nmiss > 4 ? ", ..." : "");
  if (has_relbias(e->d.arch)) {  // T5, MPNet: the bias of every relative position a kernel sees, log2 domain
    const int nh = e->d.heads;
    std::vector<float> bias((size_t)e->d.rel_buckets * nh);  // relative_attention_bias [buckets, heads]
    OM_CUDA(cudaMemcpy(bias.data(), e->rel_w, bias.size() * 4, cudaMemcpyDeviceToHost));
    for (int pass = 0; pass < 2; ++pass) {  // one table per attention kernel
      const int maxl = pass == 0 ? kMaxL : kMaxLongL, W = 2 * maxl - 1;
      std::vector<float> table((size_t)nh * W);
      for (int rel = -(maxl - 1); rel <= maxl - 1; ++rel) {
        const int b = t5_bucket(rel, e->d.rel_buckets, e->d.rel_max_distance);
        for (int h = 0; h < nh; ++h) table[(size_t)h * W + rel + maxl - 1] = bias[(size_t)b * nh + h] * kLog2e;
      }
      OM_CUDA(cudaMemcpy(pass == 0 ? e->relbias_log2 : e->relbias_long_log2, table.data(), table.size() * 4,
                         cudaMemcpyHostToDevice));
    }
  }
  static bool attr = false;
  if (!attr) {  // every instantiation: handles of both head widths may live in one process
    OM_CUDA(attn_opt_in<64>());
    OM_CUDA(attn_opt_in<32>());
    attr = true;
  }
  // fold every normalisation into the GEMM that consumes it (file header): BERT layer l's QKV takes the LayerNorm that
  // produced its input (embeddings.LayerNorm for l = 0, else layer l-1's output.LayerNorm) and W1 takes
  // attention.output.LayerNorm; T5 block l's QKV / wi take its own pre-norm RMS weights (no beta, no mean term).
  // Nothing can fail once the fp32 staging copies are freed: from then on the handle is finalized.
  const bool bert = bert_like(e->d.arch);
  const int H = e->d.hidden, I = e->I, F = e->d.ffn;
  for (int li = 0; li < e->d.layers; ++li) {
    LayerW& w = e->layers[li];
    const float* g_in = bert ? (li == 0 ? e->emb_g : e->layers[li - 1].ln2_g) : w.ln1_g;
    const float* b_in = bert ? (li == 0 ? e->emb_b : e->layers[li - 1].ln2_b) : nullptr;
    fold_norm_kernel<<<(3 * I + 7) / 8, 256>>>(w.wqkv_f32, g_in, b_in, bert ? w.bqkv : nullptr, 3 * I, H, bert ? 1 : 0,
                                               w.wqkv, w.bqkv_fold);
    fold_norm_kernel<<<(F + 7) / 8, 256>>>(w.w1_f32, bert ? w.ln1_g : w.ln2_g, bert ? w.ln1_b : nullptr,
                                           bert ? w.b1 : nullptr, F, H, bert ? 1 : 0, w.w1, w.b1_fold);
  }
  OM_CUDA(cudaGetLastError());
  OM_CUDA(cudaDeviceSynchronize());
  for (LayerW& w : e->layers) {
    dev_free(e, w.wqkv_f32);
    dev_free(e, w.w1_f32);
    w.wqkv_f32 = w.w1_f32 = nullptr;
  }
  e->finalized = true;
  return 0;
}

int om_encode(om_encoder* e, const int64_t* input_ids, const int64_t* attention_mask, const int64_t* token_type_ids,
              int B, int L, void* out_reps, om_dtype out_dtype, int64_t out_row_stride, float* out_hidden, void* stream) {
  if (!e || !input_ids || !attention_mask) return fail(OM_EINVAL, "om_encode: null argument");
  OM_TRY(check_out(e, "om_encode", out_reps, out_dtype, out_row_stride));
  if (B <= 0 || L <= 0) return fail(OM_EINVAL, "om_encode: B and L must be positive");
  const bool long_seq = L > kMaxL;
  if (long_seq && (L > kMaxLongL || L % 128 != 0))
    return fail(OM_EINVAL, "om_encode: L=%d unsupported (at most %d tokens, or 256 / 384 / 512: pad to a multiple of 128)", L,
                kMaxL);
  const om_encoder_desc& d = e->d;
  if (L > max_seq_len(d))
    return fail(OM_EINVAL, "om_encode: L=%d exceeds %d (%s)", L, max_seq_len(d), seq_limit_name(d.arch));
  const int64_t T64 = static_cast<int64_t>(B) * L;
  if (T64 > e->Tmax) return fail(OM_EINVAL, "om_encode: B*L=%lld exceeds max_batch_tokens=%d", (long long)T64, e->Tmax);
  const int sms = device_sm_count();
  if (sms < 0) return sms;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int T = static_cast<int>(T64), H = d.hidden, I = e->I;

  NvtxRange nvtx("om.encode");
  keymask_kernel<<<(T + 255) / 256, 256, 0, st>>>(attention_mask, e->kmask, T);
  // the residual stream s lives in e->h (fp32, un-normalised) with a bf16 copy in e->xb and row statistics in
  // e->stats[0] (input of a layer: from the embedding or the previous FFN2) / e->stats[1] (after the attention block)
  OM_TRY(embed_rows(e, input_ids, token_type_ids, T, L, nullptr, B, st));

  // attention geometry
  const int spt = L > 64 ? 1 : kMaxL / L;  // sequences per 128-row tile (long sequences: L / 128 tiles per sequence)
  AttnParams ap;
  ap.T = T;
  ap.L = L;
  ap.spt = spt;
  ap.I = I;
  ap.Tvalid_rows = long_seq ? 128 : spt * L;
  ap.scale_log2 = attn_scale_log2(e);
  ap.kmask = e->kmask;
  ap.relbias_log2 = has_relbias(d.arch) ? (long_seq ? e->relbias_long_log2 : e->relbias_log2) : nullptr;
  ap.ctx = e->ctx;
  ap.rowmap = nullptr;
  ap.seqs = nullptr;
  ap.tile0 = 0;
  const int n_tiles = long_seq ? T / 128 : (B + spt - 1) / spt;
  OM_TRY(encode_layers(e, T, ap, long_seq ? n_tiles : 0, ap, long_seq ? 0 : n_tiles, sms, st));
  if (out_hidden)
    OM_CUDA(cudaMemcpyAsync(out_hidden, e->h, static_cast<size_t>(T) * H * 4, cudaMemcpyDeviceToDevice, st));

  NvtxRange nvtx_pool("om.encode.pool_head_normalize");
  pool_kernel<<<B, 256, 0, st>>>(e->h, attention_mask, L, H, d.pooling == OM_POOL_MEAN ? 1 : 0, e->pooled);
  return finish_reps(e, B, out_reps, out_dtype, out_row_stride, st);
}

int om_encode_packed(om_encoder* e, const int64_t* tokens, const int64_t* token_type_ids, const int32_t* seqlens, int B,
                     void* out_reps, om_dtype out_dtype, int64_t out_row_stride, float* out_hidden, void* stream) {
  if (!e || !tokens || !seqlens) return fail(OM_EINVAL, "om_encode_packed: null argument");
  OM_TRY(check_out(e, "om_encode_packed", out_reps, out_dtype, out_row_stride));
  if (B < 0) return fail(OM_EINVAL, "om_encode_packed: B=%d is negative", B);
  const int max_len = packed_max_len(e);
  std::vector<int64_t> tok0(static_cast<size_t>(B));
  int64_t total = 0;
  for (int i = 0; i < B; ++i) {
    const int l = seqlens[i];
    if (l < 1 || l > max_len)
      return fail(OM_EINVAL, "om_encode_packed: seqlens[%d]=%d outside [1, %d] (%s, max_batch_tokens=%d)", i, l,
                  max_len, seq_limit_name(e->d.arch), e->Tmax);
    tok0[i] = total;
    total += l;
  }
  if (B == 0) return 0;
  const int sms = device_sm_count();
  if (sms < 0) return sms;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t out_elem = out_dtype == OM_F32 ? 4 : out_dtype == OM_I8 ? 1 : 2;

  NvtxRange nvtx("om.encode_packed");
  std::vector<PackedSeq> seqs;
  std::vector<PackedGroup> groups;
  // chunks of at most max_batch_tokens sequences (the pooled / head workspace rows); one chunk unless the batch holds
  // more sequences than that
  for (int c0 = 0; c0 < B; c0 += e->Tmax) {
    const int n = std::min(B - c0, e->Tmax);
    place_packed(seqlens + c0, tok0.data() + c0, n, e->Tmax, seqs, groups);
    OM_TRY(encode_packed_chunk(e, tokens, token_type_ids, seqs, groups, nullptr, n,
                               static_cast<char*>(out_reps) + static_cast<size_t>(c0) * out_row_stride * out_elem,
                               out_dtype, out_row_stride, out_hidden, sms, st));
  }
  return 0;
}

int om_encode_pairs(om_encoder* e, const int32_t* a_tokens, int64_t a_total, const int32_t* b_tokens, int64_t b_total,
                    const int64_t* spans, int B, const int32_t* prefix, int n_prefix, const int32_t* suffix, int n_suffix,
                    void* out_reps, om_dtype out_dtype, int64_t out_row_stride, void* stream) {
  if (!e || !a_tokens || !b_tokens || !spans || (n_prefix > 0 && !prefix) || (n_suffix > 0 && !suffix))
    return fail(OM_EINVAL, "om_encode_pairs: null argument");
  OM_TRY(check_out(e, "om_encode_pairs", out_reps, out_dtype, out_row_stride));
  if (B < 0) return fail(OM_EINVAL, "om_encode_pairs: B=%d is negative", B);
  if (a_total < 0 || b_total < 0)
    return fail(OM_EINVAL, "om_encode_pairs: negative store size (a_total=%lld, b_total=%lld)", (long long)a_total,
                (long long)b_total);
  if (n_prefix < 0 || n_prefix > 4 || n_suffix < 0 || n_suffix > 4)
    return fail(OM_EINVAL, "om_encode_pairs: n_prefix=%d / n_suffix=%d outside [0, 4]", n_prefix, n_suffix);
  const int max_len = packed_max_len(e);
  std::vector<int32_t> lens(static_cast<size_t>(B));
  for (int i = 0; i < B; ++i) {
    const int64_t a0 = spans[4 * (size_t)i], al = spans[4 * (size_t)i + 1];
    const int64_t b0 = spans[4 * (size_t)i + 2], bl = spans[4 * (size_t)i + 3];
    if (a0 < 0 || al < 0 || b0 < 0 || bl < 0)
      return fail(OM_EINVAL, "om_encode_pairs: pair %d has a negative start or length (%lld, %lld, %lld, %lld)", i,
                  (long long)a0, (long long)al, (long long)b0, (long long)bl);
    if (al > a_total - a0 || bl > b_total - b0)
      return fail(OM_EINVAL, "om_encode_pairs: pair %d reads past a store (a %lld + %lld of %lld, b %lld + %lld of %lld)",
                  i, (long long)a0, (long long)al, (long long)a_total, (long long)b0, (long long)bl, (long long)b_total);
    const int64_t l = n_prefix + al + bl + n_suffix;
    if (l < 1 || l > max_len)
      return fail(OM_EINVAL, "om_encode_pairs: pair %d assembles %lld tokens, outside [1, %d] (%s, "
                  "max_batch_tokens=%d)", i, (long long)l, max_len, seq_limit_name(e->d.arch), e->Tmax);
    lens[i] = static_cast<int32_t>(l);
  }
  if (B == 0) return 0;
  const int sms = device_sm_count();
  if (sms < 0) return sms;
  if (!e->pr_tokens) {  // first pair call on this handle
    int rc = 0;
    if (dev_alloc(e, &e->pr_spans, e->Tmax) != 0 || dev_alloc(e, &e->pr_tokens, e->Tmax) != 0) rc = OM_ECUDA;
    if (rc == 0 && cudaHostAlloc(&e->pr_host, (size_t)e->Tmax * sizeof(PairSpan), cudaHostAllocDefault) != cudaSuccess) {
      cudaGetLastError();
      rc = fail(OM_ENOMEM, "om_encode_pairs: out of pinned host memory");
    }
    if (rc != 0) {
      e->pr_tokens = nullptr;  // retried on the next call; what was allocated is freed with the handle
      return rc;
    }
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t out_elem = out_dtype == OM_F32 ? 4 : out_dtype == OM_I8 ? 1 : 2;

  NvtxRange nvtx("om.encode_pairs");
  PairChunk pc;
  pc.a = a_tokens;
  pc.b = b_tokens;
  pc.sp.n_prefix = n_prefix;
  pc.sp.n_suffix = n_suffix;
  for (int j = 0; j < 4; ++j) {
    pc.sp.prefix[j] = j < n_prefix ? prefix[j] : 0;
    pc.sp.suffix[j] = j < n_suffix ? suffix[j] : 0;
  }
  const std::vector<int64_t> no_tok0(static_cast<size_t>(B), 0);  // the token stream is assembled per row group
  std::vector<PackedSeq> seqs;
  std::vector<PackedGroup> groups;
  std::vector<PairSpan> chunk_spans;
  for (int c0 = 0; c0 < B; c0 += e->Tmax) {  // chunks as in om_encode_packed: the same layout, the same kernels
    const int n = std::min(B - c0, e->Tmax);
    place_packed(lens.data() + c0, no_tok0.data(), n, e->Tmax, seqs, groups);
    chunk_spans.resize(seqs.size());
    for (size_t k = 0; k < seqs.size(); ++k) {
      const int64_t* s = spans + 4 * (static_cast<size_t>(c0) + seqs[k].out);
      chunk_spans[k] = PairSpan{s[0], s[2], static_cast<int>(s[1]), static_cast<int>(s[3])};
      seqs[k].tok0 = seqs[k].row0;
    }
    pc.spans = chunk_spans.data();
    OM_TRY(encode_packed_chunk(e, nullptr, nullptr, seqs, groups, &pc, n,
                               static_cast<char*>(out_reps) + static_cast<size_t>(c0) * out_row_stride * out_elem,
                               out_dtype, out_row_stride, nullptr, sms, st));
  }
  return 0;
}

}  // extern "C"
