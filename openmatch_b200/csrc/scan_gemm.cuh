// Search scan for query batches: fp16 Q * X^T on CQ x CX CTA clusters with the top-k filter applied directly to the
// wgmma accumulator registers.
//
//   tile        a cluster owns CQ x 128 queries x CX x 256 corpus rows; cluster rank r is CTA (a, b) = (r % CQ, r / CQ),
//               which owns query box a (128 queries) x corpus tile b (256 rows), K = d in 64-wide k blocks
//   operands    corpus tile b is needed by the CQ CTAs of column b and query box a by the CX CTAs of row a: each CTA
//               TMA-loads a 256/CQ-row slice of its corpus tile and a 128/CX-row slice of its query box and multicasts
//               each slice to the CTAs that share it.  Slices land back to back at the same offset in every destination
//               (slice boundaries are multiples of the 8-row / 1 KB swizzle atom), so every CTA sees one K-major SW128
//               operand of 128 rows (A) and one of 256 rows (B).  L2 -> SM bytes per CTA and k block: 16/CX + 32/CQ KB
//               for 4.2 MFLOP
//   warp roles  warpgroup 0: one TMA producer lane (registers lowered to 40); warpgroups 1, 2: consumers (registers
//               raised to 232), consumer g issues wgmma m64n256k16 for queries [64 g, +64) of the CTA's 128 and holds the
//               64 x 256 fp32 accumulator tile in 128 registers per thread
//   ring        kScanStages x 48 KB; the producer of CTA c writes into every CTA of S(c) = {same a} U {same b}, so a slot
//               is released one wgmma group late on the empty barriers of all of S(c) (ScanCluster)
//   schedule    persistent, static, queries fastest: tile t -> query group t % qgroups, corpus group t / qgroups, so all
//               clusters work on neighbouring corpus tiles and the corpus streams from HBM about once.  Every CTA runs
//               every k block of every tile of its cluster, also when its corpus tile lies past n_cols or its query box
//               is all padding (TMA zero fill, every column masked): its peers wait on its slices and releases
//   epilogue    no staging through shared memory: FragFilter<64> (scan_epilogue.cuh) on the accumulator registers, a
//               thread owns two query rows x 64 corpus columns.  One 64-value max per row against the query's strict
//               threshold rejects the row in the common case; survivors go to a double-buffered shared-memory stash and
//               each quad reserves its list slots with one atomicAdd per row, consumed one tile later
#pragma once
#include <cuda_fp16.h>

#include <type_traits>

#include "scan_epilogue.cuh"

namespace om {

constexpr int kScanBlockN = 256;                             // corpus rows per tile
// 4 stages fit next to the stash too, but ran the C2 scan 2-4 % slower (H100 SXM, 700 W); at 400 W the largest C2 round
// took 130.5 / 136.8 ms with 3 / 4 stages on 2x1 clusters
constexpr int kScanStages = 3;
constexpr int kScanABytes = kBlockM * kBlockK * 2;           // 16 KB: the CTA's 128 queries
constexpr int kScanBBytes = kScanBlockN * kBlockK * 2;       // 32 KB: the CTA's corpus tile
constexpr int kScanStageBytes = kScanABytes + kScanBBytes;
constexpr int kScanConsumers = kStashThreads;                // two consumer warpgroups
constexpr int kScanStashOffset = kScanStages * kScanStageBytes;
constexpr int kScanBarOffset = kScanStashOffset + kFragStashBytes;
constexpr int kScanSmemBytes = kScanBarOffset + 2 * kScanStages * 8 + 1024;  // + slack for 1024-B alignment of the base
static_assert(kScanSmemBytes <= 232448, "scan ring + stash exceed the 227 KB of shared memory an H100 block may use");

// Cluster shape CQ x CX and the operand sharing it implies: the one place that knows which CTAs write into which ring
// and who releases it.  CTA c = (a, b) multicasts its query slice to S_q(c) = {(a, b') : b' < CX} and its corpus slice
// to S_x(c) = {(a', b) : a' < CQ}, so its producer writes into S(c) = S_q(c) U S_x(c), |S(c)| = CQ + CX - 1 CTAs.  A slot
// of c's ring is written by the producers of S(c) (the relation is symmetric), so c's empty barrier counts the consumer
// warps of all of S(c), and each consumer warp of c arrives on the empty barrier of every CTA in S(c).
template <int CQ, int CX>
struct ScanCluster {
  static_assert((CQ == 2 || CQ == 4) && (CX == 1 || CX == 2), "scan cluster shapes: CQ in {2, 4}, CX in {1, 2}");
  static constexpr int kSize = CQ * CX;
  static constexpr int kShare = CQ + CX - 1;       // |S(c)|, c included
  static constexpr int kQRows = kBlockM / CX;      // query rows of the slice a CTA loads per k block
  static constexpr int kXRows = kScanBlockN / CQ;  // corpus rows of the slice a CTA loads per k block
  static constexpr int kEmptyArrivals = kShare * (kScanConsumers / 32);
  // rank of the j-th CTA of S(c) other than c, j < kShare - 1: the other CTAs of corpus column b, then those of query row a
  __device__ static uint32_t peer_rank(uint32_t rank, int j) {
    const uint32_t a = rank % CQ, b = rank / CQ;
    if (j < CQ - 1) {
      const uint32_t o = static_cast<uint32_t>(j);
      return (o < a ? o : o + 1) + CQ * b;
    }
    const uint32_t o = static_cast<uint32_t>(j - (CQ - 1));
    return a + CQ * (o < b ? o : o + 1);
  }
  __device__ static uint16_t q_mask(uint32_t rank) {  // S_q(c)
    uint32_t m = 0;
#pragma unroll
    for (int b = 0; b < CX; ++b) m |= 1u << (rank % CQ + CQ * b);
    return static_cast<uint16_t>(m);
  }
  __device__ static uint16_t x_mask(uint32_t rank) {  // S_x(c)
    return static_cast<uint16_t>(((1u << CQ) - 1u) << (CQ * (rank / CQ)));
  }
};

// ALLOW: filtered search, survivors are also masked by the allowed-row bitmap `allow` (unread otherwise).
template <int CQ, int CX, bool ALLOW>
__global__ void __launch_bounds__(kGemmProducerThreads + kScanConsumers, 1)
scan_wide_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmX, int K,
                 const float* __restrict__ thr, unsigned long long* cand, int* count, int* overflow, int nq, int n_cols,
                 int C, uint32_t row_base, const uint32_t* __restrict__ allow) {
  using Cl = ScanCluster<CQ, CX>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  unsigned long long* stash = reinterpret_cast<unsigned long long*>(smem + kScanStashOffset);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kScanBarOffset);
  uint64_t* empty_bar = full_bar + kScanStages;
  const uint32_t rank = cluster_ctarank();
  const int qa = static_cast<int>(rank % CQ), xb = static_cast<int>(rank / CQ);
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = static_cast<int>(threadIdx.x & 31);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmX);
  }
  if (warp == 1 && lane == 0) {
    // full: the own producer's expect_tx, the bytes come from every producer of S(c)
    ring_init(full_bar, empty_bar, kScanStages, Cl::kEmptyArrivals);
    fence_barrier_init();
  }
  cluster_sync_all();  // every peer's barriers exist before any multicast or remote arrive

  const int qgroups = (nq + CQ * kBlockM - 1) / (CQ * kBlockM);
  const int num_tiles = qgroups * ((n_cols + CX * kScanBlockN - 1) / (CX * kScanBlockN));
  const int num_k = (K + kBlockK - 1) / kBlockK;

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      // ------------------------------ TMA producer ------------------------------
      const uint16_t qmask = Cl::q_mask(rank), xmask = Cl::x_mask(rank);
      Ring<kScanStages> ring;
      for (int tile = static_cast<int>(cluster_id_x()); tile < num_tiles; tile += static_cast<int>(cluster_count_x())) {
        const int m_blk = (tile % qgroups) * CQ + qa;
        const int n_blk = (tile / qgroups) * CX + xb;
        for (int kb = 0; kb < num_k; ++kb) {
          uint64_t* bar = ring_acquire_tx(full_bar, empty_bar, ring, kScanStageBytes, 30);
          uint8_t* sa = smem + ring.stage * kScanStageBytes;
          if constexpr (CX == 1)
            tma_load_2d(sa, &tmQ, bar, kb * kBlockK, m_blk * kBlockM);
          else
            tma_load_2d_multicast(sa + xb * (Cl::kQRows * kBlockK * 2), &tmQ, bar, kb * kBlockK,
                                  m_blk * kBlockM + xb * Cl::kQRows, qmask);
          tma_load_2d_multicast(sa + kScanABytes + qa * (Cl::kXRows * kBlockK * 2), &tmX, bar, kb * kBlockK,
                                n_blk * kScanBlockN + qa * Cl::kXRows, xmask);
          ring.advance();
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ------------------------------ consumers: wgmma + filter ------------------------------
    const int et = static_cast<int>(threadIdx.x) - kGemmProducerThreads;  // 0 .. 255
    const int wg = et >> 7;                                               // queries [64 wg, +64) of the CTA's 128
    const int frow = 64 * wg + 16 * (warp & 3) + (lane >> 2);             // fragment rows frow, frow + 8
    Ring<kScanStages> ring;
    FragFilter<64, ALLOW> filter{stash + et, cand, count, overflow, C, row_base, lane, allow};

    // lane 0 of every consumer warp releases a slot on the empty barrier of each CTA of S(c)
    uint32_t peers[Cl::kShare - 1];
#pragma unroll
    for (int j = 0; j < Cl::kShare - 1; ++j) peers[j] = Cl::peer_rank(rank, j);
    auto release = [&](uint32_t s) {
      if (lane == 0) {
        mbar_arrive(&empty_bar[s]);
#pragma unroll
        for (int j = 0; j < Cl::kShare - 1; ++j) mbar_arrive_remote(&empty_bar[s], peers[j]);
      }
    };

    for (int tile = static_cast<int>(cluster_id_x()); tile < num_tiles; tile += static_cast<int>(cluster_count_x())) {
      const int m_blk = (tile % qgroups) * CQ + qa;
      const int n_blk = (tile / qgroups) * CX + xb;
      const int row0 = m_blk * kBlockM + frow, row1 = row0 + 8;
      const int col0 = n_blk * kScanBlockN;
      const float inf = __int_as_float(0x7f800000);
      const float t0 = row0 < nq ? thr[row0] : inf, t1 = row1 < nq ? thr[row1] : inf;

      float acc[128];
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = 0.f;
      ring_consume(
          full_bar, ring, 0, num_k, 31,
          [&](uint32_t stage, uint32_t accumulate) {
            const uint32_t a_addr = smem_u32(smem + stage * kScanStageBytes) + wg * (64 * 128);
            const uint32_t b_addr = smem_u32(smem + stage * kScanStageBytes + kScanABytes);
#pragma unroll
            for (int k = 0; k < kBlockK / kWgmmaK; ++k)
              wgmma_m64n256k16_f16<0, 0>(acc, wgmma_desc(a_addr + k * 32, kDescKMajorSW128),
                                         wgmma_desc(b_addr + k * 32, kDescKMajorSW128), (accumulate | k) != 0 ? 1u : 0u);
          },
          release);
      wgmma_fence_regs(acc);

      filter.tile(acc, t0, t1, row0, col0, n_cols);
    }
    filter.drain();
  }

  __syncthreads();
  cluster_sync_all();  // the peer may still be signalling this CTA's barriers or writing into its ring
}

// Clusters of the CQ x CX scan that are co-resident on the device (cached per shape, one device per process); 0 when
// none fits.  The persistent schedule wants every cluster co-resident (a second wave would double the run time).
template <int CQ, int CX, bool ALLOW>
static inline cudaError_t scan_wide_max_clusters(int num_sms, int* out) {
  static int max_clusters = -1;
  if (max_clusters < 0) {
    constexpr int kSize = ScanCluster<CQ, CX>::kSize;
    cudaError_t e =
        cudaFuncSetAttribute(scan_wide_kernel<CQ, CX, ALLOW>, cudaFuncAttributeMaxDynamicSharedMemorySize, kScanSmemBytes);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(kSize * (num_sms / kSize));
    cfg.blockDim = dim3(kGemmProducerThreads + kScanConsumers);
    cfg.dynamicSmemBytes = kScanSmemBytes;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim = {static_cast<unsigned>(kSize), 1, 1};
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n = 0;
    e = cudaOccupancyMaxActiveClusters(&n, scan_wide_kernel<CQ, CX, ALLOW>, &cfg);
    if (e != cudaSuccess) return e;
    max_clusters = n < num_sms / kSize ? n : num_sms / kSize;
  }
  *out = max_clusters;
  return cudaSuccess;
}

template <int CQ, int CX, bool ALLOW>
static inline cudaError_t launch_scan_wide(const __half* Q, int64_t ldq, const __half* X, int64_t ldx, int nq, int n_cols,
                                           int K, const float* thr, unsigned long long* cand, int* count, int* overflow,
                                           int C, uint32_t row_base, const uint32_t* allow, int num_sms,
                                           cudaStream_t stream, int* max_clusters_out) {
  using Cl = ScanCluster<CQ, CX>;
  CUtensorMap tmQ, tmX;
  if (make_tmap_bf16_2d(&tmQ, Q, (uint64_t)K, (uint64_t)nq, (uint64_t)ldq * 2, kBlockK, Cl::kQRows) != 0)
    return cudaErrorInvalidValue;
  if (make_tmap_bf16_2d(&tmX, X, (uint64_t)K, (uint64_t)n_cols, (uint64_t)ldx * 2, kBlockK, Cl::kXRows) != 0)
    return cudaErrorInvalidValue;
  int max_clusters = 0;
  cudaError_t e = scan_wide_max_clusters<CQ, CX, ALLOW>(num_sms, &max_clusters);
  if (e != cudaSuccess) return e;
  *max_clusters_out = max_clusters;
  if (max_clusters < 1) return cudaErrorNotSupported;
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(kGemmProducerThreads + kScanConsumers);
  cfg.dynamicSmemBytes = kScanSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim = {static_cast<unsigned>(Cl::kSize), 1, 1};
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const int qgroups = (nq + CQ * kBlockM - 1) / (CQ * kBlockM);
  const int64_t num_tiles = static_cast<int64_t>(qgroups) * ((n_cols + CX * kScanBlockN - 1) / (CX * kScanBlockN));
  const int clusters = num_tiles < max_clusters ? static_cast<int>(num_tiles) : max_clusters;
  cfg.gridDim = dim3(Cl::kSize * clusters);
  return cudaLaunchKernelEx(&cfg, scan_wide_kernel<CQ, CX, ALLOW>, tmQ, tmX, K, thr, cand, count, overflow, nq, n_cols, C,
                            row_base, allow);
}

// Host launcher of the wide scan on cq x cx clusters (cq in {2, 4}, cx in {1, 2}).  Q: [nq, K] fp16 queries, row pitch
// ldq elements; X: [n_cols, K] fp16 corpus rows, row pitch ldx.  Survivors (score > thr[q]) are appended to
// cand[q * C ...] as make_key(score, row_base + column); a list that would grow beyond C sets *overflow.  allow: nullptr, or
// the allowed-row bitmap of a filtered search (indexed by row_base + column), which survivors must also pass.  Every shape
// computes each score with the same wgmma sequence, so the candidate lists hold the same keys whatever the shape.
// *max_clusters: the clusters of the shape (of its bitmap variant with allow) that are co-resident on the device, 0 when
// none fits or the shape is not one of the four.  Returns cudaSuccess / a CUDA error; tensor-map failures and other
// shapes map to cudaErrorInvalidValue, and cudaErrorNotSupported means that no cluster of the shape fits on the device.
static inline cudaError_t launch_scan_cluster(int cq, int cx, const __half* Q, int64_t ldq, const __half* X, int64_t ldx,
                                              int nq, int n_cols, int K, const float* thr, unsigned long long* cand,
                                              int* count, int* overflow, int C, uint32_t row_base, const uint32_t* allow,
                                              int num_sms, cudaStream_t stream, int* max_clusters) {
  *max_clusters = 0;
  if (nq <= 0 || n_cols <= 0 || K <= 0) return cudaSuccess;
  auto launch = [&](auto cq_c, auto cx_c) {
    constexpr int CQ = decltype(cq_c)::value, CX = decltype(cx_c)::value;
    return allow ? launch_scan_wide<CQ, CX, true>(Q, ldq, X, ldx, nq, n_cols, K, thr, cand, count, overflow, C, row_base,
                                                  allow, num_sms, stream, max_clusters)
                 : launch_scan_wide<CQ, CX, false>(Q, ldq, X, ldx, nq, n_cols, K, thr, cand, count, overflow, C, row_base,
                                                   nullptr, num_sms, stream, max_clusters);
  };
  using I1 = std::integral_constant<int, 1>;
  using I2 = std::integral_constant<int, 2>;
  using I4 = std::integral_constant<int, 4>;
  if (cq == 2 && cx == 1) return launch(I2{}, I1{});
  if (cq == 4 && cx == 1) return launch(I4{}, I1{});
  if (cq == 2 && cx == 2) return launch(I2{}, I2{});
  if (cq == 4 && cx == 2) return launch(I4{}, I2{});
  return cudaErrorInvalidValue;
}

}  // namespace om
