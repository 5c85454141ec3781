// Exact inner-product top-k over an HBM-resident flat index — the H100 replacement of
// faiss.IndexFlatIP.{add,search,reset} as the reference uses it
// (src/openmatch/retriever/dense_retriever.py:38-41,105,133-137,180) and of the IndexShards merge behind
// index_cpu_to_gpu_multiple(shard=True) (:43-58).
//
// Storage per index shard: fp32 master rows [n, d] (what index.add received; used for exact re-scoring)
// plus an fp16 scan copy [n, dpad] (tensor-core operand; IEEE half keeps 3 more significand bits than bf16 at the
// same tensor-core rate, which is what makes the exactness certificate below affordable).
// An index created with fp16 storage (om_index_create_typed) keeps only the fp16 rows [n, dpad]: they are the scan
// operand and the row store at once, FINAL and the exact scan read them, and every "fp32 score" below is the fp32
// inner product of the fp32 query with the STORED fp16 row (same summation order).  The corpus error term of the
// certificate is then exactly 0.
// An index created with int8 storage keeps rows of int8 codes and a per-row fp32 scale (quant_i8.cuh); every round scans
// on scan_i8.cuh (s8 tensor cores, a two-level int8 split of the query), and FINAL, the exact scan and the certificate
// treat fp32(s * c) as the stored row, with a corpus term of 0 as for fp16.
//
// search(q, k):
//   1. SCAN    fp16 Q * X^T on wgmma with the top-k filter fused into the epilogue (query batches: scan_gemm.cuh, 2-CTA
//              clusters, filter on the accumulator registers; the first round and <= 128 queries: the gemm.cuh mainloop):
//              scores never leave the SM (registers / shared memory); each query row's scores are compared against that
//              query's running threshold and the rare survivors are appended
//              (key = orderable(score) << 32 | ~row) to the query's candidate list in HBM.
//              The corpus is swept in rounds of geometrically growing size; after each round
//   2. SELECT  a per-query radix select keeps the best kp = k + slack candidates and publishes the kp-th score
//              as the next round's (strict) threshold.  An overflowing list (adversarially sorted corpus) is
//              detected and the level is redone with an overflow-proof fixed-size round schedule.
//   3. FINAL   the kp candidates are re-scored against the fp32 master rows (fp32 FMA, fixed summation order),
//              sorted by (score desc, row asc) and the top k emitted as (D fp32, I int64) — faiss's output contract.
//   4. CERTIFY per query, a rigorous a-posteriori bound E(q) on |stage score - fp32 score| over ALL rows
//              (measured quantisation-error norms of the corpus and of the query + an fp32 accumulation term)
//              proves that no row outside the candidate list can reach the k-th fp32 score:
//                  s_k(fp32) - tau(stage, kp-th) > E(q).
//              Queries that fail it are re-run with the widest candidate list (k + slack = 4096) and, if still
//              uncertified (e.g. thousands of near-duplicate rows that collide in half precision), by an exact
//              fp32 scan on the CUDA cores that uses the same summation order as FINAL.  The result is therefore
//              always the exact top-k by fp32 inner product, ties by row id — never "top-k up to fp16 noise".
#include <cuda_fp16.h>
#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <new>
#include <type_traits>
#include <vector>

#include "common.h"
#include "gemm.cuh"
#include "nccl_dyn.h"
#include "quant_i8.cuh"
#include "scan_epilogue.cuh"
#include "scan_gemm.cuh"
#include "scan_i8.cuh"

namespace om {

// ---------------------------------------------------------------------------------------------------
// shared-memory bitonic sort (descending) of P = 2^m keys by nthreads threads
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void bitonic_sort_desc(unsigned long long* s, int P, int tid, int nthreads) {
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < (P >> 1); t += nthreads) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // insert a 0 bit at position log2(j)
        const int p = i | j;
        const unsigned long long a = s[i], b = s[p];
        const bool desc = (i & k) == 0;
        if ((a < b) == desc) {
          s[i] = b;
          s[p] = a;
        }
      }
      __syncthreads();
    }
  }
}

// SELECT: one CTA per query.  MSB-first radix select of the kp-th largest key among the cnt candidates, then
// compaction of the keys >= it to the head of the list (unordered) and publication of its score as the new
// strict threshold.  The 32 score bits are resolved with three 11/11/10-bit passes; the 32 row bits are only
// walked (four 8-bit passes) when the kp-th score is tied with more candidates than there are slots left.
// (A full shared-memory sort here costs ~35 GB of smem traffic per round at nq = 6980 — it was 43 % of the
// search time.)
__global__ void __launch_bounds__(256) select_kernel(unsigned long long* cand, int* count, float* thr, int C, int kp,
                                                     int cnt_override) {
  extern __shared__ unsigned long long skeys[];
  __shared__ int hist[2048];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_remaining, s_out, s_bin_count, s_wsum[8];
  const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  unsigned long long* mine = cand + static_cast<size_t>(q) * C;
  int cnt = cnt_override >= 0 ? cnt_override : count[q];
  cnt = cnt < C ? cnt : C;
  if (cnt < kp) {  // nothing to drop yet: no threshold
    if (tid == 0) {
      count[q] = cnt;
      thr[q] = __int_as_float(0xff800000);
    }
    return;
  }
  if (cnt == kp) {
    // exactly kp entries (a round without survivors, or a shard of exactly kp rows): the list stays as it is and
    // the threshold is its smallest key.  (Resetting it to -inf here let the next round accept every row.)
    unsigned long long m = ~0ull;
    for (int i = tid; i < cnt; i += blockDim.x) m = min(m, mine[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) skeys[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) {
      for (int i = 1; i < static_cast<int>(blockDim.x >> 5); ++i) m = min(m, skeys[i]);
      count[q] = cnt;
      thr[q] = key_score(m);
    }
    return;
  }
  for (int i = tid; i < cnt; i += blockDim.x) skeys[i] = mine[i];
  if (tid == 0) {
    s_prefix = 0ull;
    s_remaining = kp;
    s_out = 0;
  }
  __syncthreads();
  unsigned long long mask = 0ull;
  // digit schedule: (shift, bits)
  const int shifts[7] = {53, 42, 32, 24, 16, 8, 0};
  const int widths[7] = {11, 11, 10, 8, 8, 8, 8};
  for (int pass = 0; pass < 7; ++pass) {
    const int shift = shifts[pass], nbins = 1 << widths[pass];
    for (int i = tid; i < nbins; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const unsigned long long prefix = s_prefix;
    for (int i0 = 0; i0 < cnt; i0 += blockDim.x) {
      const int i = i0 + tid;
      const bool live = i < cnt && (skeys[i] & mask) == prefix;
      const int digit = live ? static_cast<int>((skeys[i] >> shift) & static_cast<unsigned long long>(nbins - 1)) : -1;
      // warp-aggregate equal digits (top bits of similar scores collide heavily)
      const unsigned peers = __match_any_sync(0xffffffffu, digit);
      if (live && lane == (__ffs(peers) - 1)) atomicAdd(&hist[digit], __popc(peers));
    }
    __syncthreads();
    {
      // Block-wide scan from the top bin down: thread t owns the `per` consecutive bins at positions
      // [t * per, (t + 1) * per) counted from the top (read in a per-lane rotated order so the 32 lanes hit 32
      // banks); find the bin where the running count reaches `remaining`.
      const int per = nbins >> 8;  // 8, 4 or 1
      const int remaining = s_remaining;
      const int rot = per > 1 ? lane / (32 / per) : 0;
      int sum = 0;
      for (int j = 0; j < per; ++j) sum += hist[nbins - 1 - (tid * per + ((j + rot) & (per - 1)))];
      int incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      if (lane == 31) s_wsum[tid >> 5] = incl;
      __syncthreads();
      int base = 0;
      for (int w = 0; w < (tid >> 5); ++w) base += s_wsum[w];
      const int excl = base + incl - sum;
      if (excl < remaining && remaining <= excl + sum) {  // exactly one thread
        int run = excl;
        for (int j = 0; j < per; ++j) {
          const int bin = nbins - 1 - (tid * per + j), c = hist[bin];
          if (run < remaining && remaining <= run + c) {
            s_prefix = prefix | (static_cast<unsigned long long>(bin) << shift);
            s_remaining = remaining - run;
            s_bin_count = c;
          }
          run += c;
        }
      }
    }
    mask |= static_cast<unsigned long long>(nbins - 1) << shift;
    __syncthreads();
    // after the score bits: if every candidate sharing the kp-th score fits, no need to look at row bits
    if (pass == 2 && s_bin_count == s_remaining) break;
  }
  // keys >= kth under `mask` (keys are unique, so with all 64 bits resolved exactly kp keys qualify; with only
  // the score bits resolved the whole tie group qualifies and it fits by the check above)
  const unsigned long long kth = s_prefix;
  for (int i0 = 0; i0 < cnt; i0 += blockDim.x) {  // compaction, one shared-memory atomic per warp
    const int i = i0 + tid;
    const bool keep = i < cnt && (skeys[i] & mask) >= kth;
    const unsigned b = __ballot_sync(0xffffffffu, keep);
    int base = 0;
    if (lane == 0 && b) base = atomicAdd(&s_out, __popc(b));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (keep) mine[base + __popc(b & ((1u << lane) - 1u))] = skeys[i];
  }
  if (tid == 0) {
    count[q] = kp;
    thr[q] = key_score(kth);
  }
}

// Stored row formats, one per row type: the row pitch in elements (host and device), and a view of row r that reads
// element i, or group i of 4 consecutive elements (d % 4 == 0; the pitch keeps the groups aligned), as fp32.  fp16 -> fp32
// is exact and an int8 element reads as fp32(s * c), so a stored row scores bit for bit like the same values held as fp32.
// finite(v): whether a stored value v leaves the row finite, the storage's rule for the rows om_index_commit counts.
template <typename RowT>
struct StoredRow;
// fp32 master rows [n, d]
template <>
struct StoredRow<float> {
  __host__ __device__ static int pitch(int d) { return d; }
  const float4* q;  // the row in groups (d % 4 == 0)
  const float* p;   // the row in elements
  __device__ StoredRow(const float* xs, size_t r, int d)
      : q(reinterpret_cast<const float4*>(xs) + r * (pitch(d) >> 2)), p(xs + r * pitch(d)) {}
  __device__ float4 quad(int i) const { return __ldg(q + i); }
  __device__ float elem(int i) const { return __ldg(p + i); }
};
// fp16 rows [n, dpad], dpad = d rounded up to 8 (om_index_create_typed); a row with a non-finite element is non-finite
template <>
struct StoredRow<__half> {
  __host__ __device__ static int pitch(int d) { return (d + 7) & ~7; }
  const uint2* q;  // the row in groups of 4 halves
  const __half* p;
  __device__ StoredRow(const __half* xs, size_t r, int d)
      : q(reinterpret_cast<const uint2*>(xs) + r * (pitch(d) >> 2)), p(xs + r * pitch(d)) {}
  __device__ float4 quad(int i) const {
    const uint2 u = __ldg(q + i);
    const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
    const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    return make_float4(lo.x, lo.y, hi.x, hi.y);
  }
  __device__ float elem(int i) const { return __half2float(__ldg(p + i)); }
  __device__ bool finite(float v) const { return isfinite(v); }
};
// int8 rows of i8_dpad(d) + 16 bytes (quant_i8.cuh): 4 codes per group, and the row's scale, loaded once per view.  A row
// is non-finite when its scale is; a finite scale whose products s * c overflow leaves the row accepted.
template <>
struct StoredRow<int8_t> {
  __host__ __device__ static int pitch(int d) { return i8_dpad(d) + 16; }
  const int8_t* p;
  float s;
  __device__ StoredRow(const int8_t* xs, size_t r, int d)
      : p(xs + r * pitch(d)), s(__ldg(reinterpret_cast<const float*>(p + i8_dpad(d)))) {}
  __device__ float4 quad(int i) const {
    const uint32_t u = __ldg(reinterpret_cast<const unsigned int*>(p) + i);
    return make_float4(__fmul_rn(s, static_cast<float>(static_cast<int8_t>(u))),
                       __fmul_rn(s, static_cast<float>(static_cast<int8_t>(u >> 8))),
                       __fmul_rn(s, static_cast<float>(static_cast<int8_t>(u >> 16))),
                       __fmul_rn(s, static_cast<float>(static_cast<int8_t>(u >> 24))));
  }
  __device__ float elem(int i) const { return __fmul_rn(s, static_cast<float>(__ldg(p + i))); }
  __device__ bool finite(float) const { return isfinite(s); }
};

// Excluded ids of a filtered search: CSR offsets over the caller's queries and ids in the result id space (id_offset +
// local row).  Query q of a launch is the caller's query qmap[q_base + q] (an escalation level's sub-batch), or q_base + q
// without a map.  At most kMaxExcluded ids per query, the smallest re-score slack: a full first-level list then still
// holds k rows that are not excluded.
constexpr int kMaxExcluded = 128;
struct Excluded {
  const int64_t* off;  // nullptr: no exclusions
  const int64_t* ids;
  const int* qmap;
  int q_base;
  int64_t id_offset;
  // Query q's excluded ids as local rows in s[0], s[stride], ... s[(n - 1) stride], loaded by threads tid, tid + nthreads,
  // ...; returns n.  An id outside [id_offset, id_offset + 2^32 - 1) becomes 0xffffffff, which is no row of a shard.
  __device__ int load(int q, uint32_t* s, int stride, int tid, int nthreads) const {
    if (!off) return 0;
    const int g = qmap ? qmap[q_base + q] : q_base + q;
    const int64_t a = off[g];
    const int n = static_cast<int>(off[g + 1] - a);
    for (int i = tid; i < n; i += nthreads) {
      const int64_t r = ids[a + i] - id_offset;
      s[i * stride] = (r >= 0 && r < 0xffffffffll) ? static_cast<uint32_t>(r) : 0xffffffffu;
    }
    return n;
  }
};

// The fp32 score of stored row `row` against the query sq (d floats in shared memory), computed by one warp: a lane-strided
// 4-element FMA chain, then the xor-butterfly; every lane returns the sum.  FINAL and the range re-score share it, so a
// range result scores bit for bit as search reports the same row.
template <typename RowT>
__device__ __forceinline__ float row_dot(const RowT* __restrict__ xs, uint32_t row, int d, const float* sq, int lane) {
  float acc = 0.f;
  if ((d & 3) == 0) {
    const StoredRow<RowT> x(xs, row, d);
    const float4* q4 = reinterpret_cast<const float4*>(sq);
    for (int i = lane; i < (d >> 2); i += 32) {
      const float4 a = x.quad(i), b = q4[i];
      acc = fmaf(a.x, b.x, acc);
      acc = fmaf(a.y, b.y, acc);
      acc = fmaf(a.z, b.z, acc);
      acc = fmaf(a.w, b.w, acc);
    }
  } else {
    const StoredRow<RowT> x(xs, row, d);
    for (int i = lane; i < d; i += 32) acc = fmaf(x.elem(i), sq[i], acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

// FINAL: one CTA per query: exact fp32 re-score of the candidates against the stored rows (fp32 master rows or fp16
// rows), sort by (score desc, row asc), emit the top k_out.  8 CTAs per SM (32 registers): the row
// gathers are HBM-bound and want every warp resident.
// FILTER: candidates whose rows the query excludes (ex, <= kMaxExcluded ids in shared memory after the query) are dropped
// before their re-score; their keys (0) sort last and are emitted as missing slots.
template <typename RowT, bool FILTER = false>
__global__ void __launch_bounds__(256, 8) finalize_kernel(const unsigned long long* cand, const int* count, int C,
                                                          const float* __restrict__ qf, const RowT* __restrict__ xs,
                                                          int d, float* D, int64_t* I, int64_t id_offset, int k_out,
                                                          int stage_scores, Excluded ex) {
  extern __shared__ unsigned long long fsm[];
  const int q = blockIdx.x;
  const int cnt = count[q];
  int P = 2;
  while (P < cnt) P <<= 1;
  unsigned long long* skeys = fsm;
  float* sq = reinterpret_cast<float*>(fsm + P);
  for (int i = threadIdx.x; i < d; i += blockDim.x) sq[i] = qf[static_cast<size_t>(q) * d + i];
  for (int i = cnt + threadIdx.x; i < P; i += blockDim.x) skeys[i] = 0ull;
  uint32_t* sx = reinterpret_cast<uint32_t*>(sq + d);
  int nx = 0;
  if constexpr (FILTER) nx = ex.load(q, sx, 1, threadIdx.x, blockDim.x);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const unsigned long long* mine = cand + static_cast<size_t>(q) * C;
  for (int j = warp; j < cnt; j += nw) {
    const uint32_t row = key_row(mine[j]);
    if constexpr (FILTER) {
      bool hit = false;
      for (int e = lane; e < nx; e += 32) hit |= sx[e] == row;
      if (__any_sync(0xffffffffu, hit)) {
        if (lane == 0) skeys[j] = 0ull;
        continue;
      }
    }
    float acc = row_dot(xs, row, d, sq, lane);
    if (stage_scores) acc = key_score(mine[j]);  // debug: report the candidate-stage score instead
    if (lane == 0) skeys[j] = make_key(acc, row);
  }
  __syncthreads();
  bitonic_sort_desc(skeys, P, threadIdx.x, blockDim.x);
  // k_out entries are written per query (row pitch k_out): the sharded exchange ships a fixed-width prefix
  for (int r = threadIdx.x; r < k_out; r += blockDim.x) {
    float s = -FLT_MAX;
    int64_t id = -1;
    if (r < cnt && (!FILTER || skeys[r] != 0ull)) {
      s = key_score(skeys[r]);
      id = id_offset + static_cast<int64_t>(key_row(skeys[r]));
    }
    D[static_cast<size_t>(q) * k_out + r] = s;
    I[static_cast<size_t>(q) * k_out + r] = id;
  }
}

// fp32 [n, d] -> fp16 [n, dpad] (pad columns zeroed; finite values beyond the half range saturate — the measured
// error norm below then makes the certificate fail and the exact path takes over), one warp per row.
// Optional outputs: per-row ||x_h|| and ||x - x_h|| (queries) and running maxima of ||x|| and ||x - x_h|| over all
// rows ever committed (index): the inputs of the exactness certificate.  Non-negative floats order like ints, so
// the maxima are kept with atomicMax on the bit patterns.
__global__ void __launch_bounds__(256) rows_to_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst,
                                                          int64_t n, int d, int dpad, float* __restrict__ hnorm,
                                                          float* __restrict__ enorm, float* gstats) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  float mx = 0.f, me = 0.f;
  for (int64_t r = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += nwarps) {
    const float* x = src + r * d;
    __half* y = dst + r * dpad;
    float sx = 0.f, sh = 0.f, se = 0.f;
    for (int c = 2 * lane; c < dpad; c += 64) {  // dpad is a multiple of 8
      const float a = c < d ? x[c] : 0.f, b = c + 1 < d ? x[c + 1] : 0.f;
      const float ac = fminf(fmaxf(a, -65504.f), 65504.f), bc = fminf(fmaxf(b, -65504.f), 65504.f);
      const __half2 h = __floats2half2_rn(ac, bc);  // NaN stays NaN (fmin/fmax return the other operand: guard below)
      *reinterpret_cast<__half2*>(y + c) = h;
      const float ha = __low2float(h), hb = __high2float(h);
      const float ea = a - ha, eb = b - hb;
      sx = fmaf(a, a, fmaf(b, b, sx));
      sh = fmaf(ha, ha, fmaf(hb, hb, sh));
      se = fmaf(ea, ea, fmaf(eb, eb, se));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sx += __shfl_xor_sync(0xffffffffu, sx, o);
      sh += __shfl_xor_sync(0xffffffffu, sh, o);
      se += __shfl_xor_sync(0xffffffffu, se, o);
    }
    // NaN / inf inputs poison the norms on purpose: the certificate then never holds and the exact scan answers
    const float nx = sqrtf(sx), nh = sqrtf(sh), ne = sqrtf(se);
    if (lane == 0) {
      if (hnorm) hnorm[r] = nh;
      if (enorm) enorm[r] = ne;
    }
    mx = (nx > mx || nx != nx) ? nx : mx;
    me = (ne > me || ne != ne) ? ne : me;
  }
  if (gstats && lane == 0) {
    atomicMax(reinterpret_cast<int*>(gstats), __float_as_int(mx != mx ? __int_as_float(0x7fc00000) : mx));
    atomicMax(reinterpret_cast<int*>(gstats) + 1, __float_as_int(me != me ? __int_as_float(0x7fc00000) : me));
  }
}

// fp16 storage, add: src [n, d] (fp32 / bf16 / fp16) -> dst fp16 [n, dpad], round to nearest even.  Elements that become
// ±inf or NaN in fp16 (NaN, |x| >= 65520) are counted in *bad: the caller then refuses the whole add.
template <typename T>
__global__ void to_f16_rows_kernel(const T* __restrict__ src, int64_t n, int d, __half* __restrict__ dst, int dpad, int* bad) {
  int nb = 0;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n * d;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / d;
    const __half h = __float2half_rn(static_cast<float>(src[i]));
    dst[r * dpad + (i - r * d)] = h;
    nb += (__hisinf(h) || __hisnan(h)) ? 1 : 0;
  }
  if (nb) atomicAdd(bad, nb);
}

// int8 storage, add: src [n, d] (fp32 / bf16 / fp16, converted exactly to fp32) -> rows of quant_i8.cuh, one warp per row.
// Rows holding inf or NaN are counted in *bad: the caller then refuses the whole add.
template <typename T>
__global__ void __launch_bounds__(256) quantize_rows_i8_kernel(const T* __restrict__ src, int64_t n, int d, int8_t* __restrict__ dst,
                                                               int64_t pitch, int* bad) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  int nb = 0;
  for (int64_t r = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += nwarps) {
    const T* x = src + r * d;
    const bool finite = quantize_row_i8([&](int j) { return static_cast<float>(x[j]); }, d, i8_dpad(d), dst + r * pitch, lane);
    nb += finite ? 0 : 1;
  }
  if (lane == 0 && nb) atomicAdd(bad, nb);
}

// fp16 / int8 storage, commit: the stored rows are read in place.  Running maximum of ||x^|| over the rows, x^_j the stored
// value of element j (gstats[0], summed in the order of rows_to_f16_kernel, so an fp32 index of the same values gets the
// same bits); gstats[1] stays as it is (the stored values are the rows).  Rows that StoredRow<RowT>::finite rejects are
// counted in *nonfinite: searches refuse the index until a reset.
template <typename RowT>
__global__ void __launch_bounds__(256) commit_rows_kernel(const RowT* __restrict__ x, int64_t n, int d, float* gstats,
                                                          int* nonfinite) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  float mx = 0.f;
  int nbad = 0;
  for (int64_t r = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += nwarps) {
    const StoredRow<RowT> row(x, r, d);
    float sx = 0.f;
    bool finite = true;
    for (int c = 2 * lane; c < d; c += 64) {
      const float a = row.elem(c), b = c + 1 < d ? row.elem(c + 1) : 0.f;
      finite = finite && row.finite(a) && row.finite(b);
      sx = fmaf(a, a, fmaf(b, b, sx));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sx += __shfl_xor_sync(0xffffffffu, sx, o);
    const float nx = sqrtf(sx);
    mx = (nx > mx || nx != nx) ? nx : mx;
    if (!__all_sync(0xffffffffu, finite) && lane == 0) ++nbad;
  }
  if (lane == 0) {
    atomicMax(reinterpret_cast<int*>(gstats), __float_as_int(mx != mx ? __int_as_float(0x7fc00000) : mx));
    if (nbad) atomicAdd(nonfinite, nbad);
  }
}

// Queries of an int8 index: fp32 [nq, d] -> the two-level split q ~ q_h = sig_hi q_hi + sig_lo q_lo of scan_i8.cuh
// (sig_hi = amax / 127, sig_lo = sig_hi / 254, codes rounded half to even after an IEEE division; pad columns zero), one
// warp per query.  Certificate inputs: hn = ||sig_hi q_hi|| + ||sig_lo q_lo|| (>= ||q_h||, bounds the magnitude of the
// scan's two products) and en = ||q - q_h|| (each element's residual with two FMAs: both are exact up to one rounding of
// a value far below the residual).  A non-finite query gets en = NaN: its certificate fails and the exact scan answers.
__global__ void __launch_bounds__(256) queries_to_i8_kernel(const float* __restrict__ qf, int64_t nq, int d, int dpad,
                                                            int8_t* __restrict__ qhi, int8_t* __restrict__ qlo,
                                                            float2* __restrict__ sig, float* __restrict__ hn,
                                                            float* __restrict__ en) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  for (int64_t r = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); r < nq; r += nwarps) {
    const float* x = qf + r * d;
    float amax = 0.f;
    bool finite = true;
    for (int j = lane; j < d; j += 32) {
      finite = finite && isfinite(x[j]);
      amax = fmaxf(amax, fabsf(x[j]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    finite = __all_sync(0xffffffffu, finite);
    const float sh = __fdiv_rn(amax, 127.f), sl = __fdiv_rn(sh, 254.f);
    float nh = 0.f, nl = 0.f, ne = 0.f;
    for (int j = lane; j < dpad; j += 32) {
      const float v = j < d ? x[j] : 0.f;
      const float ch = sh > 0.f ? fminf(fmaxf(rintf(__fdiv_rn(v, sh)), -127.f), 127.f) : 0.f;
      const float res = __fmaf_rn(-sh, ch, v);
      const float cl = sl > 0.f ? fminf(fmaxf(rintf(__fdiv_rn(res, sl)), -127.f), 127.f) : 0.f;
      const float e = __fmaf_rn(-sl, cl, res);
      qhi[r * dpad + j] = static_cast<int8_t>(ch);
      qlo[r * dpad + j] = static_cast<int8_t>(cl);
      const float ph = sh * ch, pl = sl * cl;
      nh = fmaf(ph, ph, nh);
      nl = fmaf(pl, pl, nl);
      ne = fmaf(e, e, ne);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      nh += __shfl_xor_sync(0xffffffffu, nh, o);
      nl += __shfl_xor_sync(0xffffffffu, nl, o);
      ne += __shfl_xor_sync(0xffffffffu, ne, o);
    }
    if (lane == 0) {
      sig[r] = make_float2(sh, sl);
      hn[r] = sqrtf(nh) + sqrtf(nl);
      en[r] = finite ? sqrtf(ne) : __int_as_float(0x7fc00000);
    }
  }
}

template <typename T>
__global__ void to_f32(const T* __restrict__ src, float* __restrict__ dst, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] = static_cast<float>(src[i]);
}
__global__ void fill_i32(int* p, int v, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// MERGE (sharded search exchange step): one CTA per query over nparts * k candidates.  Part p's lists start at
// Dp + p * stride_d / Ip + p * stride_i (elements), [nq, k] row-major each.
__global__ void __launch_bounds__(256) merge_kernel(const float* Dp, const int64_t* Ip, int64_t stride_d,
                                                    int64_t stride_i, int nparts, int nq, int k, int k_out, float* D,
                                                    int64_t* I) {
  // keys: orderable(score) << 32 | ~slot, with ties broken by id through a second pass on equal scores
  extern __shared__ unsigned long long msm[];
  const int q = blockIdx.x;
  const int total = nparts * k;
  int P = 2;
  while (P < total) P <<= 1;
  unsigned long long* skeys = msm;           // [P] (score, slot)
  int64_t* sid = reinterpret_cast<int64_t*>(msm + P);  // [total]
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    unsigned long long key = 0ull;
    if (i < total) {
      const int part = i / k, r = i - part * k;
      const size_t off = static_cast<size_t>(q) * k + r;
      const int64_t id = Ip[part * stride_i + off];
      sid[i] = id;
      if (id >= 0) key = (static_cast<unsigned long long>(f32_orderable(Dp[part * stride_d + off])) << 32) | (0xffffffffu - i);
    }
    skeys[i] = key;
  }
  __syncthreads();
  bitonic_sort_desc(skeys, P, threadIdx.x, blockDim.x);
  // Shards hold disjoint, increasing id ranges and each shard list is already (score desc, id asc), so slot
  // order == id order among equal scores: the (score, slot) sort is the (score, id) sort.
  for (int r = threadIdx.x; r < k_out; r += blockDim.x) {
    const unsigned long long key = r < P ? skeys[r] : 0ull;
    float s = -FLT_MAX;
    int64_t id = -1;
    if (key != 0ull) {
      s = f32_from_orderable(static_cast<uint32_t>(key >> 32));
      id = sid[0xffffffffu - static_cast<uint32_t>(key & 0xffffffffull)];
    }
    D[static_cast<size_t>(q) * k_out + r] = s;
    I[static_cast<size_t>(q) * k_out + r] = id;
  }
}

// CERTIFY: one warp per query.  Every row outside the re-scored candidate set has a stage score <= tau, and
// |stage - fp32| <= E(q) for every row of the corpus, so s_k - tau > E(q) proves that the emitted top-k is the
// exact fp32 top-k.  With x_h / q_h the half-precision operands, B the exact product sum of the rounded operands:
//   |fp32 - exact|   <= 30 * 2^-24 * |q||x|                      (FINAL's 24-FMA chain + 5-level tree at d = 768)
//   |exact - B|      <= ||q_h|| * ||x - x_h|| + ||q - q_h|| * ||x||          (Cauchy-Schwarz on the two error terms)
//   |B - stage|      <= d * 2^-22 * ||q_h|| * ||x_h||            (fp32 accumulation of exact products in the tensor
//                       core: d adds, each off by at most 2^-23 of the running magnitude if the hardware truncates
//                       instead of rounding; x2 head-room.  tests/test_search_gpu.py measures the real value.)
// with the corpus norms replaced by their maxima over the index (kept by rows_to_f16_kernel; sharded search: over all
// shards).  tau is the kp-th stage score of the candidate list — sharded search: the largest of the shards' floors.
// A NaN anywhere makes the comparison false: the query is flagged and answered by the exact path.
// cert_bound: E(q) from the query's hn = ||q_h||, en = ||q - q_h|| and the corpus maxima xmax, exmax (the 1.001 covers the
// roundings of this fp32 expression itself).
__device__ __forceinline__ float cert_bound(float hn, float en, float xmax, float exmax, int d) {
  return 1.001f * (hn * exmax + en * xmax + static_cast<float>(d + 16) * 2.384185791015625e-07f * (hn + en) * (xmax + exmax));
}
__global__ void __launch_bounds__(256) certify_kernel(const float* __restrict__ D, const int64_t* __restrict__ I, int k,
                                                      const float* __restrict__ floors, int64_t floor_stride, int nparts,
                                                      const float* __restrict__ gstats, int64_t stats_stride,
                                                      const float* __restrict__ hn, const float* __restrict__ en, int d,
                                                      int nq, int q_base, int* flags, int* nflag) {
  const int q = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (q >= nq) return;
  // tau: no row outside the re-scored candidate lists has a stage score above the largest per-shard floor (kp-th stage
  // score of the shard's list; -inf when the shard's list holds every row of the shard); error-norm maxima likewise
  float tau = __int_as_float(0xff800000), xmax = 0.f, exmax = 0.f;
  for (int p = 0; p < nparts; ++p) {
    tau = fmaxf(tau, floors[p * floor_stride + q]);
    const float a = gstats[p * stats_stride], b = gstats[p * stats_stride + 1];
    xmax = (a > xmax || a != a) ? a : xmax;  // NaN sticks: the comparison below then fails
    exmax = (b > exmax || b != b) ? b : exmax;
  }
  const float E = cert_bound(hn[q], en[q], xmax, exmax, d);
  // tau = -inf: every list holds every row of its shard, nothing was left out.  Otherwise k results are needed to compare.
  const bool full = I[static_cast<size_t>(q) * k + (k - 1)] >= 0;
  const bool ok = !(tau > __int_as_float(0xff800000)) ? true : (full && D[static_cast<size_t>(q) * k + (k - 1)] - tau > E);
  // flags, not an appended list: the order of the uncertified queries must be the same on every rank of a sharded search
  if (lane == 0) {
    flags[q_base + q] = ok ? 0 : 1;
    if (!ok) atomicAdd(nflag, 1);
  }
}

// EXACT fp32 scan on the CUDA cores (the certificate's last resort and the "exact_only" test mode): one warp per
// row group, queries of the tile in shared memory, rows of type RowT (as finalize_kernel reads them).
// Per (query, row) the summation order is EXACTLY the one of finalize_kernel (lane-strided 4-element FMA chain, then the
// xor-butterfly), so both produce bit-identical scores.
// Survivors (score > the query's strict threshold) are appended to the same candidate lists the tensor-core scan
// uses; dense = 1: first round, every score stored at position = column.
// FILTER (dense = 0 only: a filtered first round runs at threshold -inf): survivors must also be allowed by the bitmap
// `allow` (nullable) and not excluded by their query (ex: kMaxExcluded x NQT ids in shared memory after the queries,
// interleaved, id e of query j at e * NQT + j, so the lanes of the active queries read consecutive words).
template <int NQT, int ROWS, typename RowT, bool FILTER = false>
__global__ void __launch_bounds__(256) exact_scan_kernel(const RowT* __restrict__ xs, int64_t n_rows,
                                                         uint32_t row_base,
                                                         const float* __restrict__ qf, int nq, int d, int nqt,
                                                         const float* __restrict__ thr, unsigned long long* cand,
                                                         int* count, int* overflow, int C, int dense,
                                                         const uint32_t* __restrict__ allow, Excluded ex) {
  extern __shared__ float sq[];
  const int q0 = blockIdx.y * nqt;
  const int nact = min(nqt, nq - q0);
  for (int i = threadIdx.x; i < nact * d; i += blockDim.x) sq[i] = qf[static_cast<size_t>(q0) * d + i];
  int nx = 0;  // lane j: query j's excluded rows, sx[0, nx)
  if constexpr (FILTER) {
    for (int j = 0; j < nact; ++j) {
      const int n = ex.load(q0 + j, reinterpret_cast<uint32_t*>(sq + static_cast<size_t>(nqt) * d) + j, NQT, threadIdx.x,
                            blockDim.x);
      if (static_cast<int>(threadIdx.x & 31) == j) nx = n;
    }
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const uint32_t* sx = reinterpret_cast<const uint32_t*>(sq + static_cast<size_t>(nqt) * d) + lane;
  float t = __int_as_float(0x7f800000);
  if (lane < nact && !dense) t = thr[q0 + lane];
  const int64_t wg = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5), nw = static_cast<int64_t>(gridDim.x) * 8;
  for (int64_t r0 = wg * ROWS; r0 < n_rows; r0 += nw * ROWS) {
    float acc[ROWS][NQT];
#pragma unroll
    for (int rr = 0; rr < ROWS; ++rr)
#pragma unroll
      for (int j = 0; j < NQT; ++j) acc[rr][j] = 0.f;
    if ((d & 3) == 0) {
      const int d4 = d >> 2;
      for (int i = lane; i < d4; i += 32) {
        float4 a[ROWS];
#pragma unroll
        for (int rr = 0; rr < ROWS; ++rr)
          a[rr] = r0 + rr < n_rows ? StoredRow<RowT>(xs, r0 + rr, d).quad(i) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < NQT; ++j) {
          if (j < nact) {
            const float4 b = reinterpret_cast<const float4*>(sq + static_cast<size_t>(j) * d)[i];
#pragma unroll
            for (int rr = 0; rr < ROWS; ++rr) {
              float s = acc[rr][j];
              s = fmaf(a[rr].x, b.x, s);
              s = fmaf(a[rr].y, b.y, s);
              s = fmaf(a[rr].z, b.z, s);
              s = fmaf(a[rr].w, b.w, s);
              acc[rr][j] = s;
            }
          }
        }
      }
    } else {
      for (int i = lane; i < d; i += 32) {
        float a[ROWS];
#pragma unroll
        for (int rr = 0; rr < ROWS; ++rr) a[rr] = r0 + rr < n_rows ? StoredRow<RowT>(xs, r0 + rr, d).elem(i) : 0.f;
#pragma unroll
        for (int j = 0; j < NQT; ++j)
          if (j < nact) {
            const float b = sq[static_cast<size_t>(j) * d + i];
#pragma unroll
            for (int rr = 0; rr < ROWS; ++rr) acc[rr][j] = fmaf(a[rr], b, acc[rr][j]);
          }
      }
    }
#pragma unroll
    for (int rr = 0; rr < ROWS; ++rr)
#pragma unroll
      for (int j = 0; j < NQT; ++j)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[rr][j] += __shfl_xor_sync(0xffffffffu, acc[rr][j], o);
#pragma unroll
    for (int rr = 0; rr < ROWS; ++rr) {
      float mine = acc[rr][0];  // lane j keeps query j's score (all lanes hold identical sums)
#pragma unroll
      for (int j = 1; j < NQT; ++j)
        if (lane == j) mine = acc[rr][j];
      const int64_t col = r0 + rr;
      if (lane < nact && col < n_rows) {
        const int q = q0 + lane;
        const unsigned long long key = make_key(mine, row_base + static_cast<uint32_t>(col));
        if (dense) {
          cand[static_cast<size_t>(q) * C + col] = key;
        } else if (mine > t) {
          if constexpr (FILTER) {
            const uint32_t r = row_base + static_cast<uint32_t>(col);
            bool keep = !allow || ((__ldg(allow + (r >> 5)) >> (r & 31)) & 1u);
            for (int e = 0; keep && e < nx; ++e) keep = sx[e * NQT] != r;
            if (!keep) continue;
          }
          const int pos = atomicAdd(count + q, 1);
          if (pos < C)
            cand[static_cast<size_t>(q) * C + pos] = key;
          else
            *overflow = 1;
        }
      }
    }
  }
}

// Argument rules of a filter's exclusions, per query: *bad |= 1 for decreasing offsets (or a negative first one, or ids
// missing), 2 for more than kMaxExcluded ids, 4 for a negative id.
__global__ void check_exclusions_kernel(const int64_t* __restrict__ off, const int64_t* __restrict__ ids, int nq, int* bad) {
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x) {
    const int64_t a = off[q], b = off[q + 1];
    int f = 0;
    if (a < 0 || b < a || (b > a && !ids))
      f = 1;
    else if (b - a > kMaxExcluded)
      f = 2;
    else
      for (int64_t i = a; i < b; ++i) f |= ids[i] < 0 ? 4 : 0;
    if (f) atomicOr(bad, f);
  }
}

// Allowed rows of a filtered search's bitmap in each 256-row block of the shard's n rows (bits past n are ignored).
__global__ void allow_block_counts_kernel(const uint32_t* __restrict__ allow, int64_t n, int64_t nblocks, int* __restrict__ out) {
  for (int64_t b = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; b < nblocks;
       b += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    int c = 0;
    for (int w = 0; w < 8 && b * 256 + 32 * w < n; ++w) {
      const int64_t r0 = b * 256 + 32 * w;
      uint32_t m = allow[r0 >> 5];
      if (n - r0 < 32) m &= (1u << (n - r0)) - 1u;
      c += __popc(m);
    }
    out[b] = c;
  }
}

// dst[i] = src[list[i]] (rows of d floats): the queries (or radii) of a sub-batch
__global__ void gather_rows_kernel(const float* __restrict__ src, const int* __restrict__ list, int n, int d,
                                   float* __restrict__ dst) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < static_cast<int64_t>(n) * d;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / d);
    dst[i] = src[static_cast<size_t>(list[r]) * d + (i - static_cast<int64_t>(r) * d)];
  }
}
// D[list[i]] = Dsub[i], I[list[i]] = Isub[i] (rows of k)
__global__ void scatter_results_kernel(const float* __restrict__ Dsub, const int64_t* __restrict__ Isub,
                                       const int* __restrict__ list, int n, int k, float* __restrict__ D,
                                       int64_t* __restrict__ I) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < static_cast<int64_t>(n) * k;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / k);
    const size_t o = static_cast<size_t>(list[r]) * k + (i - static_cast<int64_t>(r) * k);
    D[o] = Dsub[i];
    I[o] = Isub[i];
  }
}

// ---------------------------------------------------------------------------------------------------
// range search: every row whose fp32 score is strictly above the query's radius rho
// ---------------------------------------------------------------------------------------------------
// THRESHOLD of the one sweep.  Every row has |b - s| <= E(q) (the certificate's bound, b the stage score, s the fp32
// score), so a row with s > rho has b >= s - E > rho - E >= t with t = rho - E rounded toward -inf: b > t, the scans'
// strict test, keeps it.  The sweep's candidate set therefore holds every row of the answer, at any threshold round and
// on any scan kernel, and the exact re-score decides.  t <= rho is never NaN while E is finite; t = -inf (rho = -inf, or
// rho - E below -FLT_MAX) keeps every row, still a superset.  A non-finite E (a query holding inf / NaN, overflowed norms)
// proves nothing: the query gets t = +inf here (no candidates) and is answered by the exact scan, which compares exact
// scores with rho itself (exact = 1 sweeps: thr = rho).
__global__ void range_threshold_kernel(const float* __restrict__ rho, const float* __restrict__ hn, const float* __restrict__ en,
                                       const float* __restrict__ gstats, int d, int nq, int exact, float* __restrict__ thr,
                                       int* __restrict__ to_exact) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  if (exact) {
    thr[q] = rho[q];
    to_exact[q] = 0;
    return;
  }
  const float E = cert_bound(hn[q], en[q], gstats[0], gstats[1], d);
  const bool ok = isfinite(E);
  thr[q] = ok ? __fsub_rd(rho[q], E) : __int_as_float(0x7f800000);
  to_exact[q] = ok ? 0 : 1;
}

// After each round: the scans count every survivor (atomicAdd on count) but store only below C.  The round's survivors
// are added to the 64-bit total and count is clamped back to the list's fill, so no round (< 2^30 columns) can wrap it.
__global__ void range_fold_kernel(int* __restrict__ count, int* __restrict__ filled, long long* __restrict__ total, int C, int nq) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  const int c = count[q];
  total[q] += c - filled[q];
  const int f = min(c, C);
  filled[q] = f;
  count[q] = f;
}

// RE-SCORE and CUT: one warp per candidate (grid.y = query), the query in shared memory, the score of FINAL (row_dot).  A
// candidate becomes make_key(s, row) if s > rho, else 0, which is no row's key and sorts last; surv counts the kept ones.
// Queries whose list overflowed (total > C) are swept again and skipped here.
// FILTER: candidates whose rows the query excludes (ex, <= kMaxExcluded ids in shared memory after the query) become 0
// before their re-score and are not counted, as finalize_kernel<RowT, true> drops them.
template <typename RowT, bool FILTER = false>
__global__ void __launch_bounds__(256, 4) range_rescore_kernel(unsigned long long* __restrict__ cand, const int* __restrict__ count,
                                                            const long long* __restrict__ total, int C,
                                                            const float* __restrict__ qf, const RowT* __restrict__ xs, int d,
                                                            const float* __restrict__ rho, int* __restrict__ surv, Excluded ex) {
  extern __shared__ float4 rsm[];
  float* sq = reinterpret_cast<float*>(rsm);
  const int q = blockIdx.y;
  const int cnt = count[q];
  if (total[q] > C || static_cast<int>(blockIdx.x) * 8 >= cnt) return;
  for (int i = threadIdx.x; i < d; i += blockDim.x) sq[i] = qf[static_cast<size_t>(q) * d + i];
  uint32_t* sx = reinterpret_cast<uint32_t*>(sq + d);
  int nx = 0;
  if constexpr (FILTER) nx = ex.load(q, sx, 1, threadIdx.x, blockDim.x);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float r = rho[q];
  unsigned long long* mine = cand + static_cast<size_t>(q) * C;
  int kept = 0;
  for (int j = blockIdx.x * 8 + warp; j < cnt; j += gridDim.x * 8) {
    const uint32_t row = key_row(mine[j]);
    if constexpr (FILTER) {
      bool hit = false;
      for (int e = lane; e < nx; e += 32) hit |= sx[e] == row;
      if (__any_sync(0xffffffffu, hit)) {
        if (lane == 0) mine[j] = 0ull;
        continue;
      }
    }
    const float s = row_dot(xs, row, d, sq, lane);
    const bool keep = s > r;
    if (lane == 0) mine[j] = keep ? make_key(s, row) : 0ull;
    kept += keep ? 1 : 0;
  }
  if (lane == 0 && kept) atomicAdd(surv + q, kept);
}

// SORT, step 1: every block of kRangeSortKeys keys of a query's list (grid.x = block, grid.y = query) is sorted descending in
// shared memory.  A list of at most kRangeSortKeys keys is then sorted; longer ones are merged by range_merge_kernel.
constexpr int kRangeSortKeys = 16384;
__global__ void __launch_bounds__(512) range_sort_kernel(unsigned long long* __restrict__ cand, const int* __restrict__ count,
                                                         const long long* __restrict__ total, int C) {
  extern __shared__ unsigned long long ssk[];
  const int q = blockIdx.y;
  const int cnt = count[q], base = blockIdx.x * kRangeSortKeys;
  if (total[q] > C || base >= cnt) return;
  const int n = min(cnt - base, kRangeSortKeys);
  int P = 2;
  while (P < n) P <<= 1;
  unsigned long long* mine = cand + static_cast<size_t>(q) * C + base;
  for (int i = threadIdx.x; i < P; i += blockDim.x) ssk[i] = i < n ? mine[i] : 0ull;
  __syncthreads();
  bitonic_sort_desc(ssk, P, threadIdx.x, blockDim.x);
  for (int i = threadIdx.x; i < n; i += blockDim.x) mine[i] = ssk[i];
}

// SORT, step 2 (lists longer than kRangeSortKeys): merges the sorted runs of w keys pairwise, src -> dst.  Each key goes to
// its run's start + its place in its run + the keys of the partner run before it: those greater than it for a key of the
// left run, those not smaller for one of the right run, so the cut keys (0, repeated) also land on distinct places.
__global__ void __launch_bounds__(256) range_merge_kernel(const unsigned long long* __restrict__ src, unsigned long long* __restrict__ dst,
                                                          const int* __restrict__ count, const long long* __restrict__ total,
                                                          int C, int w) {
  const int q = blockIdx.y;
  const int cnt = count[q];
  if (total[q] > C || cnt <= kRangeSortKeys) return;
  const unsigned long long* s = src + static_cast<size_t>(q) * C;
  unsigned long long* o = dst + static_cast<size_t>(q) * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += gridDim.x * blockDim.x) {
    const int run = i / w, j = i - run * w, p0 = (run ^ 1) * w;
    const int plen = max(0, min(cnt - p0, w));
    const unsigned long long key = s[i];
    const bool left = (run & 1) == 0;
    int lo = 0, hi = plen;  // first partner place whose key does not precede this one
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      const unsigned long long pk = s[p0 + mid];
      if (left ? pk > key : pk >= key)
        lo = mid + 1;
      else
        hi = mid;
    }
    o[min(run, run ^ 1) * w + j + lo] = key;
  }
}

// EMIT: the sorted survivors of the queries a sweep answered (off[q] >= 0) to the results' key store at off[q].  Lists
// longer than kRangeSortKeys ended in `alt` when their merge took an odd number of steps.
__global__ void __launch_bounds__(256) range_emit_kernel(const unsigned long long* __restrict__ cand,
                                                         const unsigned long long* __restrict__ alt, int alt_above,
                                                         const int* __restrict__ count, const int* __restrict__ surv,
                                                         const long long* __restrict__ off, int C,
                                                         unsigned long long* __restrict__ store) {
  const int q = blockIdx.y;
  const long long o = off[q];
  if (o < 0) return;
  const unsigned long long* s = (count[q] > alt_above ? alt : cand) + static_cast<size_t>(q) * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < surv[q]; i += gridDim.x * blockDim.x) store[o + i] = s[i];
}

// Results of a shard in query order: query q's keys store[src[q] ...] -> (score, id_offset + row) at lims[q] (grid.x =
// query, grid.y = CTAs per query).
__global__ void __launch_bounds__(256) range_gather_kernel(const unsigned long long* __restrict__ store,
                                                           const long long* __restrict__ src, const long long* __restrict__ lims,
                                                           int64_t id_offset, float* __restrict__ D, int64_t* __restrict__ I) {
  const int q = blockIdx.x;
  const long long a = lims[q], n = lims[q + 1] - a, s = src[q];
  for (long long i = blockIdx.y * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.y) * blockDim.x) {
    const unsigned long long k = store[s + i];
    D[a + i] = key_score(k);
    I[a + i] = id_offset + static_cast<int64_t>(key_row(k));
  }
}

// MERGE of a sharded range search: part p's results (Dp + p stride_d, Ip + p stride_i; its lims at plims + p (nq + 1))
// are sorted runs per query by (score desc, id asc).  Each entry goes to glims[q] + its place in its run + the entries of
// the other parts' runs that precede it: higher score, or equal score and lower id (equal ids: lower part).  Ids are
// compared themselves, so any id_offset per rank gives the single-index order.  grid.y = part.
__global__ void __launch_bounds__(256, 4) range_merge_parts_kernel(const float* __restrict__ Dp, const int64_t* __restrict__ Ip,
                                                                int64_t stride_d, int64_t stride_i,
                                                                const long long* __restrict__ plims, int W, int nq,
                                                                const long long* __restrict__ glims, float* __restrict__ D,
                                                                int64_t* __restrict__ I) {
  const int p = blockIdx.y;
  const long long* lp = plims + static_cast<size_t>(p) * (nq + 1);
  const long long T = lp[nq];
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < T;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    int lo = 0, hi = nq;  // the query: the last q with lp[q] <= e
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (lp[mid] <= e) lo = mid; else hi = mid;
    }
    const int q = lo;
    const float s = Dp[p * stride_d + e];
    const int64_t id = Ip[p * stride_i + e];
    long long pos = glims[q] + (e - lp[q]);
    for (int p2 = 0; p2 < W; ++p2) {
      if (p2 == p) continue;
      const long long* l2 = plims + static_cast<size_t>(p2) * (nq + 1);
      const float* D2 = Dp + p2 * stride_d;
      const int64_t* I2 = Ip + p2 * stride_i;
      long long a = l2[q], b = l2[q + 1];
      while (a < b) {  // first entry of the run that does not precede (s, id, p)
        const long long mid = (a + b) >> 1;
        const float s2 = D2[mid];
        const int64_t id2 = I2[mid];
        if (s2 > s || (s2 == s && (id2 < id || (id2 == id && p2 < p))))
          a = mid + 1;
        else
          b = mid;
      }
      pos += a - l2[q];
    }
    D[pos] = s;
    I[pos] = id;
  }
}

// 1 in *bad if any radius is NaN
__global__ void check_radius_kernel(const float* __restrict__ rho, int nq, int* bad) {
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x)
    if (rho[q] != rho[q]) atomicOr(bad, 1);
}

}  // namespace om

using namespace om;

// ---------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------
struct om_comm {
  void* nccl = nullptr;
  int rank = 0, world = 1;
};

namespace {

constexpr int kQueryChunk = 16384;
constexpr int kMaxCandidates = 4096;  // k + slack ceiling (finalize sorts the list in shared memory)

struct DevBuf {  // grow-only device scratch
  void* p = nullptr;
  size_t bytes = 0;
  int reserve(size_t need) {
    if (need <= bytes) return 0;
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
    OM_CUDA(dev_malloc(&p, need));
    bytes = need;
    return 0;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
  }
};

// The stored rows a search reads: n rows in the index's storage (fp32 master rows xf + fp16 scan copy xh, fp16 rows xh, or
// int8 rows xq).  A device index's own buffers, or one partition of a host-resident index in its device window.
struct Rows {
  int64_t n = 0;
  const float* xf = nullptr;
  const __half* xh = nullptr;
  const int8_t* xq = nullptr;
};

// One pass of the pipeline (scan -> select -> re-score [-> exchange -> merge] -> certify) over nq device-resident
// queries and the rows X; all pointers lie in the index's level workspace (level_layout).
struct Level {
  Rows X;
  int nq = 0, k = 0, kp = 0, kp_target = 0, C = 0, growth = 2, mode = 0, world = 1, kc = 0, nqc_max = 0;
  const float* qf = nullptr;  // [nq, d] fp32 (not owned by the workspace)
  __half* qh = nullptr;       // [nq, dpad] scan operand
  int8_t* q8 = nullptr;       // int8 index, in qh's region: q_hi [nq, dpad] then q_lo [nq, dpad]
  float2* qsig = nullptr;     // int8 index: per query (sig_hi, sig_lo)
  float *hn = nullptr, *en = nullptr;  // per query ||q_h|| (int8 index: ||sig_hi q_hi|| + ||sig_lo q_lo||), ||q - q_h||
  unsigned long long* cand = nullptr;
  int* count = nullptr;
  float* thr = nullptr;
  int* status = nullptr;  // [0] list overflow, [2] uncertified queries
  uint8_t *send = nullptr, *recv = nullptr;
  const uint32_t* allow = nullptr;  // filtered search: the allowed-row bitmap of X's rows
  // with allow: allowed rows before each 256-row block of X, relative to allow_prefix[0] (a slice of ix->allow_prefix)
  const int64_t* allow_prefix = nullptr;
  Excluded ex{};  // filtered search: excluded ids (ex.off nullptr: none), ex.qmap the level's queries in the caller's batch
};

}  // namespace

struct om_index {
  int d = 0, dpad = 0;
  int storage = OM_F32;  // OM_F32: fp32 master rows xf + fp16 scan copy xh; OM_F16: xh only; OM_I8: xq only
  int64_t n = 0, cap = 0;
  float* xf = nullptr;
  __half* xh = nullptr;
  int8_t* xq = nullptr;  // int8 rows of quant_i8.cuh, pitch dpad + 16 bytes (dpad = d rounded up to 16)
  // device [4]: [0] max ||x||, [1] max ||x - x_h|| over the committed rows (float bit patterns); fp16 / int8 storage: [2]
  // rows with a non-finite element (fp16) or scale (int8) committed since the last reset (int), [3] scratch (int: rejected
  // elements or rows of an add, the all-reduced [2] of a sharded search, a filter's or the radii's check, an agreed error)
  float* gstats = nullptr;
  int* scratch() const { return reinterpret_cast<int*>(gstats) + 3; }  // gstats[3]
  bool gstats_stale = false;  // set by om_index_reset: gstats[0..2] are zeroed on the stream of the next commit / search
  int64_t st_nonfinite = 0;   // gstats[2] as the last search read it
  int64_t rescore_slack = -1;
  int force_safe = 0;
  int pair_scan = 1;      // > 128 queries: rounds after the first on the wide scan (scan_gemm.cuh); 0 = single-CTA tiles
  int scan_cq = 0, scan_cx = 0;  // cluster shape of the wide scan (CQ CTAs along the queries x CX along the corpus); 0 = auto
  int growth = 0;         // each round scans (growth - 1) x the rows seen so far; 0 = auto: 2 for query batches (fewest
                          // filter survivors), 8 for <= 256 queries (HBM-bound streaming regime: 5 instead of 13
                          // dependent scan + select launch pairs over 8.8 M rows)
  int certify = 1;        // 0: legacy behaviour (top-k of the half-precision candidate stage, no proof)
  int exact_only = 0;     // 1: answer every query with the exact fp32 scan (testing / reference timing)
  int stage_scores = 0;   // 1: emit candidate-stage scores instead of fp32 re-scores (measuring the error model)
  int64_t st_rounds = 0, st_retries = 0, st_capacity = 0, st_launches = 0;
  int64_t st_flagged = 0, st_flagged_wide = 0, st_exact = 0;
  int64_t st_scan_cluster = 0, st_scan_clusters = 0;  // last wide scan: 10 CQ + CX and its co-resident clusters (0: none ran)
  // optional per-phase device timing (CUDA events on the launching stream), enabled by set_param("profile", 1)
  int profile = 0;
  double st_scan_us = 0, st_select_us = 0, st_final_us = 0, st_other_us = 0;
  std::vector<cudaEvent_t> ev;  // pool: [2i] start, [2i+1] stop
  std::vector<int> ev_kind;     // 0 scan, 1 select, 2 finalize, 3 exchange / merge / certify
  size_t ev_used = 0;
  DevBuf ws, ows, sws;  // level workspace / whole-search staging / escalation sub-batch
  // filtered search with a bitmap: allowed rows in [0, min(256 b, n)) for b = 0 .. ceil(n / 256), set by check_filter
  std::vector<int64_t> allow_prefix;
  int* h_status = nullptr;  // pinned host copy of the device ints a call decides on (read_decision)
  // range search: first list capacity per query; the last range search's results (D fp32 then I int64, r_total of each) in
  // rout, r_total = -1 when there are none (before any range search, after a search or a reset); rkeys: its key store
  int range_list = 4096;
  int64_t r_total = -1;
  DevBuf rkeys, rout;
  size_t r_keep_ws = 0;  // the workspace of the last range search's first sweeps (kept after the call)
  int64_t st_range_candidates = 0, st_range_resweeps = 0;
  // Host-resident index (om_index_create_host; window > 0): the stored rows live in pinned host chunks of `window` rows
  // each, in the stored row format (fp32 storage: the master rows only), and xf / xh / xq stay null.  A search uploads
  // partition p (rows [p window, (p + 1) window)) into device window p % 2 on copy_st while it searches the other one.
  int64_t window = 0;
  std::vector<void*> chunks;
  DevBuf win[2];
  int64_t win_rows[2] = {0, 0};  // rows each window holds
  cudaStream_t copy_st = nullptr;
  cudaEvent_t ev_entry = nullptr, ev_ready[2] = {nullptr, nullptr}, ev_free[2] = {nullptr, nullptr};
  int64_t st_partitions = 0;
  double st_upload_wait_us = 0;
};

// Calls f with the index's stored rows as a typed pointer: the fp32 master rows, the fp16 rows or the int8 rows.  Kernels
// over stored rows deduce their row type from it.
template <typename F>
static decltype(auto) with_rows(const om_index* ix, F&& f) {
  switch (ix->storage) {
    case OM_I8: return f(ix->xq);
    case OM_F16: return f(ix->xh);
    default: return f(ix->xf);
  }
}
// The same for the rows of a view X in the index's storage.
template <typename F>
static decltype(auto) with_rows(const om_index* ix, const Rows& X, F&& f) {
  switch (ix->storage) {
    case OM_I8: return f(X.xq);
    case OM_F16: return f(X.xh);
    default: return f(X.xf);
  }
}
// A device index's rows as a view.
static Rows device_rows(const om_index* ix) { return Rows{ix->n, ix->xf, ix->xh, ix->xq}; }

// row pitch in elements of the rows behind a typed pointer
template <typename RowT>
static int64_t pitch_of(const RowT*, int d) { return StoredRow<RowT>::pitch(d); }

// one row buffer of an index (the index member that holds it) and its bytes per row, named for the out-of-memory message
struct RowBuf {
  void** p;
  size_t row_bytes;
  const char* name;
};
template <typename RowT>
static RowBuf row_buf(RowT** p, int d, const char* name) {
  return {reinterpret_cast<void**>(p), StoredRow<RowT>::pitch(d) * sizeof(RowT), name};
}

// Device window of a host-resident index for `rows` rows: the fp32 master rows then their fp16 scan copy (fp32 storage),
// the fp16 rows, or the int8 rows.  Returns its bytes; with base, points X's buffers there.
static size_t window_layout(const om_index* ix, int64_t rows, void* base, Rows* X) {
  Layout lay;
  const size_t r = static_cast<size_t>(rows);
  const size_t o_f = lay.add(ix->storage == OM_F32 ? r * ix->d * 4 : 0);
  const size_t o_h = lay.add(ix->storage != OM_I8 ? r * ix->dpad * 2 : 0);
  const size_t o_q = lay.add(ix->storage == OM_I8 ? r * pitch_of(ix->xq, ix->d) : 0);
  if (base) {
    X->xf = ix->storage == OM_F32 ? region<const float>(base, o_f) : nullptr;
    X->xh = ix->storage != OM_I8 ? region<const __half>(base, o_h) : nullptr;
    X->xq = ix->storage == OM_I8 ? region<const int8_t>(base, o_q) : nullptr;
  }
  return lay.bytes;
}

// Bytes of one stored row in a host chunk of a host-resident index (fp32 storage: the master row only).
static size_t host_row_bytes(const om_index* ix) {
  return with_rows(ix, [&](const auto* xs) -> size_t { return pitch_of(xs, ix->d) * sizeof(*xs); });
}

// Makes device window w of a host-resident index hold at least `rows` rows (at most one partition); its view in *X, with
// X->n = rows.  Growing a window frees it first: no upload or search may be using it.
static int window_reserve(om_index* ix, int w, int64_t rows, Rows* X) {
  const int64_t need = std::min(ix->window, round_up(rows, 256));
  if (need > ix->win_rows[w]) {
    ix->win_rows[w] = 0;
    OM_TRY(ix->win[w].reserve(window_layout(ix, need, nullptr, nullptr)));
    ix->win_rows[w] = need;
  }
  window_layout(ix, ix->win_rows[w], ix->win[w].p, X);
  X->n = rows;
  return 0;
}

// Grows every row buffer of the index's storage to hold at least `need` rows.
static int index_grow(om_index* ix, int64_t need) {
  if (need <= ix->cap) return 0;
  int64_t ncap = std::max<int64_t>(need, ix->cap + ix->cap / 2);
  ncap = round_up(std::max<int64_t>(ncap, 1024), 256);
  std::vector<RowBuf> bufs;
  switch (ix->storage) {
    case OM_I8: bufs = {row_buf(&ix->xq, ix->d, "int8")}; break;
    case OM_F16: bufs = {row_buf(&ix->xh, ix->d, "fp16")}; break;
    default: bufs = {row_buf(&ix->xf, ix->d, "fp32"), row_buf(&ix->xh, ix->d, "fp16")};  // master rows, scan copy
  }
  void* fresh[2] = {};
  // rows may still be in flight on the caller's stream(s) (encoder writing reserved rows, a pending commit)
  OM_CUDA(cudaDeviceSynchronize());
  for (size_t b = 0; b < bufs.size(); ++b) {
    if (dev_malloc(&fresh[b], static_cast<size_t>(ncap) * bufs[b].row_bytes) != cudaSuccess) {
      for (void* p : fresh) cudaFree(p);
      cudaGetLastError();
      return fail(OM_ENOMEM, "index: cannot allocate the %s rows for %lld rows", bufs[b].name, (long long)ncap);
    }
    if (ix->n > 0)
      OM_CUDA(cudaMemcpy(fresh[b], *bufs[b].p, static_cast<size_t>(ix->n) * bufs[b].row_bytes, cudaMemcpyDeviceToDevice));
  }
  OM_CUDA(cudaDeviceSynchronize());
  for (size_t b = 0; b < bufs.size(); ++b) {
    cudaFree(*bufs[b].p);
    *bufs[b].p = fresh[b];
  }
  ix->cap = ncap;
  return 0;
}

static inline int grid_for(int64_t n, int threads) {
  int64_t g = (n + threads - 1) / threads;
  return static_cast<int>(std::min<int64_t>(std::max<int64_t>(g, 1), 132 * 16));
}

// Zeroes the error-norm maxima a reset left stale, on the stream of the commit or search that reads them next.  A reset
// cannot zero them itself: a memset on any stream other than the caller's next one may land after that call's atomicMax
// and leave maxima of 0, with which the certificate would prove wrong candidate lists exact.
static int settle_reset(om_index* ix, cudaStream_t st) {
  if (!ix->gstats_stale) return 0;
  OM_CUDA(cudaMemsetAsync(ix->gstats, 0, 3 * sizeof(float), st));
  ix->gstats_stale = false;
  return 0;
}

#define OM_NCCL(expr)                                                                                   \
  do {                                                                                                  \
    int r__ = (expr);                                                                                   \
    if (r__ != 0) return fail(OM_ECUDA, "%s failed: %s", #expr, nccl_api().GetErrorString(r__));        \
  } while (0)

// Reads the n device ints at `dev` into ix->h_status[0, n) with one host synchronisation, for the host to branch on.  With
// a communicator (nullptr: none), dev[0] is first all-reduced over the ranks with op (kNcclMax or kNcclSum) into dev[to]
// (0: in place, else an int within the n read), so that every rank takes the same decision.
static int read_decision(om_index* ix, om_comm* comm, int* dev, int n, int op, int to, cudaStream_t st) {
  if (comm) OM_NCCL(nccl_api().AllReduce(dev, dev + to, 1, kNcclInt32, op, comm->nccl, st));
  OM_CUDA(cudaMemcpyAsync(ix->h_status, dev, n * sizeof(int), cudaMemcpyDeviceToHost, st));
  OM_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// The device rows an add reads: x itself, or for host input a temporary device buffer *tmp filled on st, which the caller
// frees once st is synchronised.
static int stage_input(const void* x, om_memkind kind, size_t bytes, cudaStream_t st, const void** src, void** tmp) {
  *src = x;
  if (kind != OM_HOST) return 0;
  OM_CUDA(cudaMalloc(tmp, bytes));
  OM_CUDA(cudaMemcpyAsync(*tmp, x, bytes, cudaMemcpyHostToDevice, st));
  *src = *tmp;
  return 0;
}

// Calls f with an add's input rows as a typed pointer: fp32, bf16 or fp16.
template <typename F>
static decltype(auto) with_input(const void* src, om_dtype dtype, F&& f) {
  if (dtype == OM_F32) return f(static_cast<const float*>(src));
  if (dtype == OM_BF16) return f(static_cast<const __nv_bfloat16*>(src));
  return f(static_cast<const __half*>(src));
}

extern "C" {

int om_index_create(int d, om_index** out) { return om_index_create_typed(d, OM_F32, out); }

int om_index_create_typed(int d, om_dtype storage, om_index** out) {
  if (!out || d <= 0) return fail(OM_EINVAL, "om_index_create: d must be positive");
  if (storage != OM_F32 && storage != OM_F16 && storage != OM_I8)
    return fail(OM_EINVAL, "om_index_create_typed: storage must be OM_F32, OM_F16 or OM_I8");
  OM_TRY(device_sm_count());
  om_index* ix = new (std::nothrow) om_index();
  if (!ix) return fail(OM_ENOMEM, "om_index_create: out of host memory");
  ix->d = d;
  ix->dpad = storage == OM_I8 ? i8_dpad(d) : StoredRow<__half>::pitch(d);  // scan operand pitch: 16-byte rows for TMA
  ix->storage = storage;
  if (cudaMalloc(&ix->gstats, 4 * sizeof(float)) != cudaSuccess || cudaMemset(ix->gstats, 0, 4 * sizeof(float)) != cudaSuccess ||
      cudaHostAlloc(&ix->h_status, 8 * sizeof(int), cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    cudaFree(ix->gstats);
    delete ix;
    return fail(OM_ENOMEM, "om_index_create: cannot allocate index state");
  }
  *out = ix;
  return 0;
}

int om_index_create_host(int d, om_dtype storage, int64_t window_rows, om_index** out) {
  if (!out || d <= 0) return fail(OM_EINVAL, "om_index_create_host: d must be positive");
  if (window_rows < 0 || window_rows % 256 != 0)
    return fail(OM_EINVAL, "om_index_create_host: window_rows = %lld must be 0 (automatic) or a positive multiple of 256",
                (long long)window_rows);
  om_index* ix = nullptr;
  OM_TRY(om_index_create_typed(d, storage, &ix));
  if (window_rows == 0) {  // two windows in at most a quarter of the free device memory
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) {
      cudaGetLastError();
      om_index_destroy(ix);
      return fail(OM_ECUDA, "om_index_create_host: cannot read the free device memory");
    }
    const size_t row =window_layout(ix, 256, nullptr, nullptr) / 256;
    window_rows = std::max<int64_t>(256, static_cast<int64_t>(free_b / 4 / (2 * row)) / 256 * 256);
  }
  ix->window = window_rows;
  if (cudaStreamCreateWithFlags(&ix->copy_st, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&ix->ev_entry, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&ix->ev_ready[0], cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&ix->ev_ready[1], cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&ix->ev_free[0], cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&ix->ev_free[1], cudaEventDisableTiming) != cudaSuccess) {
    cudaGetLastError();
    om_index_destroy(ix);
    return fail(OM_ECUDA, "om_index_create_host: cannot create the upload stream and its events");
  }
  *out = ix;
  return 0;
}

void om_index_destroy(om_index* ix) {
  if (!ix) return;
  if (ix->copy_st) {
    cudaStreamSynchronize(ix->copy_st);
    cudaStreamDestroy(ix->copy_st);
  }
  for (cudaEvent_t e : {ix->ev_entry, ix->ev_ready[0], ix->ev_ready[1], ix->ev_free[0], ix->ev_free[1]})
    if (e) cudaEventDestroy(e);
  for (void* c : ix->chunks) cudaFreeHost(c);
  ix->win[0].release();
  ix->win[1].release();
  cudaFree(ix->xf);
  cudaFree(ix->xh);
  cudaFree(ix->xq);
  cudaFree(ix->gstats);
  if (ix->h_status) cudaFreeHost(ix->h_status);
  ix->ws.release();
  ix->ows.release();
  ix->sws.release();
  ix->rkeys.release();
  ix->rout.release();
  for (cudaEvent_t e : ix->ev) cudaEventDestroy(e);
  delete ix;
}

int64_t om_index_ntotal(const om_index* ix) { return ix ? ix->n : 0; }
int om_index_dim(const om_index* ix) { return ix ? ix->d : 0; }
int om_index_storage(const om_index* ix) { return ix ? ix->storage : fail(OM_EINVAL, "om_index_storage: null index"); }

int om_index_reset(om_index* ix) {
  if (!ix) return fail(OM_EINVAL, "om_index_reset: null index");
  ix->n = 0;
  ix->gstats_stale = true;  // host only: see settle_reset
  ix->st_nonfinite = 0;
  ix->r_total = -1;
  ix->rout.release();
  return 0;
}

int om_index_reserve_rows(om_index* ix, int64_t n, void** dev_rows, int64_t* row_pitch_elems) {
  if (!ix || n < 0 || !dev_rows || !row_pitch_elems) return fail(OM_EINVAL, "om_index_reserve_rows: bad arguments");
  if (ix->window) return fail(OM_ESTATE, "om_index_reserve_rows: a host-resident index has no device rows to write in place");
  if (ix->n + n > 0xfffffff0ll) return fail(OM_EINVAL, "index shard limited to 2^32-16 rows; shard the corpus");
  OM_TRY(index_grow(ix, ix->n + n));
  with_rows(ix, [&](auto* xs) {
    *row_pitch_elems = pitch_of(xs, ix->d);
    *dev_rows = xs + ix->n * *row_pitch_elems;
  });
  return 0;
}

int om_index_reserve(om_index* ix, int64_t n, float** dev_rows) {
  if (!ix || n < 0 || !dev_rows) return fail(OM_EINVAL, "om_index_reserve: bad arguments");
  if (ix->window) return fail(OM_ESTATE, "om_index_reserve: a host-resident index has no device rows to write in place");
  if (ix->storage != OM_F32)
    return fail(OM_ESTATE, "om_index_reserve: the index stores %s rows; use om_index_reserve_rows",
                ix->storage == OM_F16 ? "fp16" : "int8");
  void* rows = nullptr;
  int64_t pitch = 0;
  OM_TRY(om_index_reserve_rows(ix, n, &rows, &pitch));
  *dev_rows = static_cast<float*>(rows);
  return 0;
}

int om_index_commit(om_index* ix, int64_t n, void* stream) {
  if (ix && ix->window) return fail(OM_ESTATE, "om_index_commit: a host-resident index has no rows written in place to commit");
  if (!ix || n < 0 || ix->n + n > ix->cap) return fail(OM_EINVAL, "om_index_commit: more rows than reserved");
  if (n == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  OM_TRY(settle_reset(ix, st));
  with_rows(ix, [&](auto* xs) {
    auto* rows = xs + ix->n * pitch_of(xs, ix->d);
    if constexpr (std::is_same<decltype(rows), float*>::value)  // the fp32 commit also writes the fp16 scan copy
      rows_to_f16_kernel<<<grid_for(n, 8), 256, 0, st>>>(rows, ix->xh + static_cast<size_t>(ix->n) * ix->dpad, n, ix->d,
                                                         ix->dpad, nullptr, nullptr, ix->gstats);
    else
      commit_rows_kernel<<<grid_for(n, 8), 256, 0, st>>>(rows, n, ix->d, ix->gstats, reinterpret_cast<int*>(ix->gstats) + 2);
  });
  OM_CUDA(cudaGetLastError());
  ix->n += n;
  return 0;
}

// fp16 / int8 storage: n input rows at src (device) -> stored rows at `rows` (row pitch in elements), converting to fp16 or
// quantising; elements (fp16) or rows (int8) the storage cannot hold are added to *bad.
static cudaError_t convert_rows(const om_index* ix, const void* src, om_dtype dtype, int64_t n, void* rows, int64_t pitch, int* bad,
                                cudaStream_t st) {
  return with_input(src, dtype, [&](const auto* in) {
    if (ix->storage == OM_I8)
      quantize_rows_i8_kernel<<<grid_for(n, 8), 256, 0, st>>>(in, n, ix->d, static_cast<int8_t*>(rows), pitch, bad);
    else
      to_f16_rows_kernel<<<grid_for(n * ix->d, 256), 256, 0, st>>>(in, n, ix->d, static_cast<__half*>(rows), ix->dpad, bad);
    return cudaGetLastError();
  });
}

// fp32 storage: `elems` input values at src (device, or host fp32 when kind is OM_HOST) -> fp32 rows at dst.
static int fp32_rows(float* dst, const void* src, om_memkind kind, om_dtype dtype, size_t elems, cudaStream_t st) {
  return with_input(src, dtype, [&](const auto* in) -> int {
    if constexpr (std::is_same<decltype(in), const float*>::value) {
      OM_CUDA(cudaMemcpyAsync(dst, in, elems * 4, kind == OM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, st));
    } else {
      to_f32<<<grid_for(elems, 256), 256, 0, st>>>(in, dst, (int64_t)elems);
      OM_CUDA(cudaGetLastError());
    }
    return 0;
  });
}

// The refusal of an add to fp16 / int8 storage that holds `bad` values the storage cannot hold.
static int refuse_add(const om_index* ix, int bad) {
  if (ix->storage == OM_I8)
    return fail(OM_EINVAL, "om_index_add: %d rows hold inf or NaN; int8 storage cannot hold them and no row was added", bad);
  return fail(OM_EINVAL, "om_index_add: %d elements are NaN or round to +-inf in fp16 (|x| >= 65520); fp16 storage cannot "
              "hold them and no row was added", bad);
}

// om_index_add on fp16 / int8 storage: convert into the reserved rows, count what the storage cannot hold, and commit only
// if nothing was out of range (the converted rows stay beyond ntotal otherwise).  Synchronises `st` to read the count.
static int add_converted(om_index* ix, const void* x, om_memkind kind, om_dtype dtype, int64_t n, cudaStream_t st) {
  void* rows = nullptr;
  int64_t pitch = 0;
  OM_TRY(om_index_reserve_rows(ix, n, &rows, &pitch));
  const size_t elems = static_cast<size_t>(n) * ix->d;
  const void* src = nullptr;
  void* tmp = nullptr;
  OM_TRY(stage_input(x, kind, elems * (dtype == OM_F32 ? 4 : 2), st, &src, &tmp));
  int* bad = ix->scratch();
  cudaError_t e = cudaMemsetAsync(bad, 0, sizeof(int), st);
  if (e == cudaSuccess) e = convert_rows(ix, src, dtype, n, rows, pitch, bad, st);
  const int rc = e == cudaSuccess ? read_decision(ix, nullptr, bad, 1, kNcclMax, 0, st) : 0;
  if (tmp) cudaFree(tmp);
  OM_CUDA(e);
  OM_TRY(rc);
  if (ix->h_status[0] > 0) return refuse_add(ix, ix->h_status[0]);
  return om_index_commit(ix, n, st);
}

// om_index_add on a host-resident index.  The rows pass through device window 0 in pieces that each end inside one host
// chunk: converted there by the kernels of a device index's add (fp32 storage: committed at once, which builds the scan copy
// and the error-norm maxima), then copied out to the chunk, beyond ntotal.  fp16 / int8 storage counts what it cannot
// hold over all pieces and, when nothing is refused, commits every piece (re-uploaded from its chunk unless the add was one
// piece) with commit_rows_kernel.  A refused add leaves ntotal, the stored rows and the maxima as they were.  Synchronises st.
static int add_host(om_index* ix, const void* x, om_memkind kind, om_dtype dtype, int64_t n, cudaStream_t st) {
  if (ix->n + n > 0xfffffff0ll) return fail(OM_EINVAL, "index shard limited to 2^32-16 rows; shard the corpus");
  const int64_t W = ix->window, n0 = ix->n, end = n0 + n;
  const size_t hrow = host_row_bytes(ix), in_row = static_cast<size_t>(ix->d) * (dtype == OM_F32 ? 4 : 2);
  while (static_cast<int64_t>(ix->chunks.size()) * W < end) {  // growth adds chunks; the rows already held stay where they are
    void* c = nullptr;
    if (cudaHostAlloc(&c, static_cast<size_t>(W) * hrow, cudaHostAllocDefault) != cudaSuccess) {
      cudaGetLastError();
      return fail(OM_ENOMEM, "om_index_add: cannot allocate %lld rows of pinned host memory for the host-resident index",
                  (long long)W);
    }
    ix->chunks.push_back(c);
  }
  Rows X;
  OM_TRY(window_reserve(ix, 0, std::min(W, n), &X));
  void* rows = const_cast<void*>(with_rows(ix, X, [](const auto* xs) -> const void* { return xs; }));
  const bool f32 = ix->storage == OM_F32;
  // host input the window cannot take as it is goes through a device staging buffer of one piece
  struct Tmp {
    void* p = nullptr;
    ~Tmp() { cudaFree(p); }
  } tmp;
  const bool staged = kind == OM_HOST && !(f32 && dtype == OM_F32);
  if (staged) OM_CUDA(cudaMalloc(&tmp.p, static_cast<size_t>(std::min(W, n)) * in_row));
  OM_TRY(settle_reset(ix, st));
  int* bad = ix->scratch();
  OM_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), st));
  auto piece_end = [&](int64_t a) { return std::min(end, (a / W + 1) * W); };
  for (int64_t a = n0; a < end; a = piece_end(a)) {
    const int64_t m = piece_end(a) - a;
    const void* in = static_cast<const uint8_t*>(x) + static_cast<size_t>(a - n0) * in_row;
    if (staged) {
      OM_CUDA(cudaMemcpyAsync(tmp.p, in, static_cast<size_t>(m) * in_row, cudaMemcpyHostToDevice, st));
      in = tmp.p;
    }
    if (f32) {
      OM_TRY(fp32_rows(static_cast<float*>(rows), in, staged ? OM_DEVICE : kind, dtype, static_cast<size_t>(m) * ix->d, st));
      rows_to_f16_kernel<<<grid_for(m, 8), 256, 0, st>>>(static_cast<float*>(rows), const_cast<__half*>(X.xh), m, ix->d, ix->dpad,
                                                         nullptr, nullptr, ix->gstats);
      OM_CUDA(cudaGetLastError());
    } else {
      const int64_t pitch = with_rows(ix, X, [&](const auto* xs) { return pitch_of(xs, ix->d); });
      OM_CUDA(convert_rows(ix, in, dtype, m, rows, pitch, bad, st));
    }
    uint8_t* chunk = static_cast<uint8_t*>(ix->chunks[a / W]) + static_cast<size_t>(a % W) * hrow;
    OM_CUDA(cudaMemcpyAsync(chunk, rows, static_cast<size_t>(m) * hrow, cudaMemcpyDeviceToHost, st));
  }
  OM_TRY(read_decision(ix, nullptr, bad, 1, kNcclMax, 0, st));
  if (ix->h_status[0] > 0) return refuse_add(ix, ix->h_status[0]);
  if (!f32) {
    const bool one_piece = piece_end(n0) == end;  // the window still holds it
    for (int64_t a = n0; a < end; a = piece_end(a)) {
      const int64_t m = piece_end(a) - a;
      if (!one_piece)
        OM_CUDA(cudaMemcpyAsync(rows, static_cast<const uint8_t*>(ix->chunks[a / W]) + static_cast<size_t>(a % W) * hrow,
                                static_cast<size_t>(m) * hrow, cudaMemcpyHostToDevice, st));
      with_rows(ix, X, [&](const auto* xs) {
        if constexpr (!std::is_same<decltype(xs), const float*>::value)
          commit_rows_kernel<<<grid_for(m, 8), 256, 0, st>>>(xs, m, ix->d, ix->gstats, reinterpret_cast<int*>(ix->gstats) + 2);
      });
      OM_CUDA(cudaGetLastError());
    }
  }
  OM_CUDA(cudaStreamSynchronize(st));
  ix->n = end;
  return 0;
}

int om_index_add(om_index* ix, const void* x, om_memkind kind, om_dtype dtype, int64_t n, void* stream) {
  if (!ix || (!x && n > 0) || n < 0) return fail(OM_EINVAL, "om_index_add: bad arguments");
  if (n == 0) return 0;
  if (dtype != OM_F32 && dtype != OM_BF16 && dtype != OM_F16) return fail(OM_EINVAL, "om_index_add: unsupported dtype %d", (int)dtype);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (ix->window) return add_host(ix, x, kind, dtype, n, st);
  if (ix->storage != OM_F32) return add_converted(ix, x, kind, dtype, n, st);
  float* dst = nullptr;
  OM_TRY(om_index_reserve(ix, n, &dst));
  const size_t elems = static_cast<size_t>(n) * ix->d;
  const void* src = x;
  void* tmp = nullptr;
  if (dtype != OM_F32) OM_TRY(stage_input(x, kind, elems * 2, st, &src, &tmp));  // fp32 rows are copied straight in
  OM_TRY(fp32_rows(dst, src, kind, dtype, elems, st));
  if (tmp) {
    OM_CUDA(cudaStreamSynchronize(st));
    cudaFree(tmp);
  }
  OM_TRY(om_index_commit(ix, n, stream));
  if (kind == OM_HOST) OM_CUDA(cudaStreamSynchronize(st));  // caller may free / reuse its host buffer
  return 0;
}

int om_index_set_param(om_index* ix, const char* name, int64_t value) {
  if (!ix || !name) return fail(OM_EINVAL, "om_index_set_param: bad arguments");
  if (!strcmp(name, "rescore_slack")) {
    ix->rescore_slack = value;
  } else if (!strcmp(name, "force_safe_rounds")) {
    ix->force_safe = value != 0;
  } else if (!strcmp(name, "round_growth")) {
    if (value != 0 && (value < 2 || value > 8)) return fail(OM_EINVAL, "round_growth must be 0 (auto) or in [2, 8]");
    ix->growth = static_cast<int>(value);
  } else if (!strcmp(name, "pair_scan")) {
    ix->pair_scan = value != 0;
  } else if (!strcmp(name, "scan_cluster_q")) {
    if (value != 0 && value != 2 && value != 4) return fail(OM_EINVAL, "scan_cluster_q must be 0 (auto), 2 or 4");
    ix->scan_cq = static_cast<int>(value);
  } else if (!strcmp(name, "scan_cluster_x")) {
    if (value != 0 && value != 1 && value != 2) return fail(OM_EINVAL, "scan_cluster_x must be 0 (auto), 1 or 2");
    ix->scan_cx = static_cast<int>(value);
  } else if (!strcmp(name, "profile")) {
    ix->profile = static_cast<int>(value);
  } else if (!strcmp(name, "certify")) {
    ix->certify = value != 0;
  } else if (!strcmp(name, "exact_only")) {
    ix->exact_only = value != 0;
  } else if (!strcmp(name, "debug_stage_scores")) {
    ix->stage_scores = value != 0;
  } else if (!strcmp(name, "range_list")) {
    if (value < 256 || value > (1 << 24)) return fail(OM_EINVAL, "range_list must be in [256, 2^24]");
    ix->range_list = static_cast<int>(value);
  } else {
    return fail(OM_EINVAL, "om_index_set_param: unknown parameter '%s'", name);
  }
  return 0;
}

int64_t om_index_get_stat(const om_index* ix, const char* name) {
  if (!ix || !name) return -1;
  if (!strcmp(name, "rounds")) return ix->st_rounds;
  if (!strcmp(name, "overflow_retries")) return ix->st_retries;
  if (!strcmp(name, "candidates")) return ix->st_capacity;
  if (!strcmp(name, "launches")) return ix->st_launches;
  if (!strcmp(name, "uncertified")) return ix->st_flagged;
  if (!strcmp(name, "uncertified_wide")) return ix->st_flagged_wide;
  if (!strcmp(name, "exact_queries")) return ix->st_exact;
  if (!strcmp(name, "nonfinite_rows")) return ix->st_nonfinite;
  if (!strcmp(name, "scan_cluster")) return ix->st_scan_cluster;
  if (!strcmp(name, "scan_max_clusters")) return ix->st_scan_clusters;
  if (!strcmp(name, "scan_ns")) return static_cast<int64_t>(ix->st_scan_us * 1e3);
  if (!strcmp(name, "select_ns")) return static_cast<int64_t>(ix->st_select_us * 1e3);
  if (!strcmp(name, "finalize_ns")) return static_cast<int64_t>(ix->st_final_us * 1e3);
  if (!strcmp(name, "other_ns")) return static_cast<int64_t>(ix->st_other_us * 1e3);
  if (!strcmp(name, "range_candidates")) return ix->st_range_candidates;
  if (!strcmp(name, "range_resweeps")) return ix->st_range_resweeps;
  if (!strcmp(name, "partitions")) return ix->st_partitions;
  if (!strcmp(name, "upload_wait_ns")) return static_cast<int64_t>(ix->st_upload_wait_us * 1e3);
  return -1;
}

}  // extern "C"

namespace {

// profiling helpers: bracket a launch with events from the index's pool
struct Timed {
  om_index* ix;
  cudaStream_t st;
  bool on;
  Timed(om_index* ix_, cudaStream_t st_, int kind) : ix(ix_), st(st_), on(ix_->profile != 0) {
    static const char* nvtx_names[5] = {"om.search.scan", "om.search.select", "om.search.rescore", "om.search.exchange_certify",
                                        "om.search.upload_wait"};
    nvtxRangePushA(nvtx_names[kind]);
    if (!on) return;
    if (ix->ev_used + 2 > ix->ev.size()) {
      cudaEvent_t a, b;
      if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) {
        on = false;
        return;
      }
      ix->ev.push_back(a);
      ix->ev.push_back(b);
      ix->ev_kind.push_back(0);
    }
    ix->ev_kind[ix->ev_used / 2] = kind;
    cudaEventRecord(ix->ev[ix->ev_used], st);
  }
  ~Timed() {
    nvtxRangePop();
    if (!on) return;
    cudaEventRecord(ix->ev[ix->ev_used + 1], st);
    ix->ev_used += 2;
  }
};

void collect_profile(om_index* ix) {
  static const char* names[5] = {"scan", "select", "finalize", "exchange+certify", "upload wait"};
  double* sums[5] = {&ix->st_scan_us, &ix->st_select_us, &ix->st_final_us, &ix->st_other_us, &ix->st_upload_wait_us};
  for (size_t i = 0; i + 1 < ix->ev_used; i += 2) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ix->ev[i], ix->ev[i + 1]) != cudaSuccess) continue;
    const int kind = ix->ev_kind[i / 2];
    *sums[kind] += ms * 1e3;
    if (ix->profile >= 2) fprintf(stderr, "[om profile] launch %zu %s %.3f ms\n", i / 2, names[kind], ms);
  }
  ix->ev_used = 0;
}

// Shared-memory opt-ins, once per process (one device per process, enforced by device_sm_count): the select and merge
// kernels, and with an index those over its stored rows, once per row type.
int once_attrs(const om_index* ix) {
  static bool done = false;
  if (!done) {
    OM_CUDA(cudaFuncSetAttribute(select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * 8));
    OM_CUDA(cudaFuncSetAttribute(merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 16));
    OM_CUDA(cudaFuncSetAttribute(range_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kRangeSortKeys * 8));
    done = true;
  }
  return !ix ? 0 : with_rows(ix, [](const auto* xs) -> int {
    using RowT = std::decay_t<decltype(*xs)>;
    static bool rows_done = false;  // one flag per row type: each instantiation of this operator has its own
    if (rows_done) return 0;
    OM_CUDA(cudaFuncSetAttribute(finalize_kernel<RowT>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxCandidates * 8 + 65536));
    OM_CUDA(cudaFuncSetAttribute(exact_scan_kernel<8, 2, RowT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    OM_CUDA(cudaFuncSetAttribute(finalize_kernel<RowT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 kMaxCandidates * 8 + 65536 + kMaxExcluded * 4));
    OM_CUDA(cudaFuncSetAttribute(exact_scan_kernel<8, 2, RowT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 96 * 1024 + 8 * kMaxExcluded * 4));
    OM_CUDA(cudaFuncSetAttribute(range_rescore_kernel<RowT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * 4));
    OM_CUDA(cudaFuncSetAttribute(range_rescore_kernel<RowT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 16384 * 4 + kMaxExcluded * 4));
    rows_done = true;
    return 0;
  });
}

// Packed per-shard block of the sharded exchange for nqc queries shipping kc entries each:
//   [D f32 nqc x kc | I i64 nqc x kc | floor f32 nqc (kp-th stage score of the shard's list) | error-norm maxima f32 x 2]
struct ExchangeBlock {
  size_t off_i, off_floor, off_stats, bytes;
};
inline ExchangeBlock exchange_block(size_t nqc, size_t kc) {
  ExchangeBlock b;
  b.off_i = round_up(nqc * kc * 4, 256);
  b.off_floor = b.off_i + round_up(nqc * kc * 8, 256);
  b.off_stats = b.off_floor + round_up(nqc * 4, 256);
  b.bytes = b.off_stats + 256;
  return b;
}
inline size_t exchange_block_bytes(size_t nqc, size_t kc) { return exchange_block(nqc, kc).bytes; }

// The tensor-core scan operand of the level's queries L.qf (fp16, or the int8 split of an int8 index) and their
// certificate norms L.hn, L.en.
int convert_queries(om_index* ix, Level& L, cudaStream_t st) {
  const int nq = L.nq, d = ix->d, dpad = ix->dpad;
  if (ix->storage == OM_I8)
    queries_to_i8_kernel<<<grid_for(nq, 8), 256, 0, st>>>(L.qf, nq, d, dpad, L.q8, L.q8 + static_cast<size_t>(nq) * dpad, L.qsig,
                                                          L.hn, L.en);
  else
    rows_to_f16_kernel<<<grid_for(nq, 8), 256, 0, st>>>(L.qf, L.qh, nq, d, dpad, L.hn, L.en, nullptr);
  OM_CUDA(cudaGetLastError());
  ix->st_launches += 1;
  return 0;
}

// A level's own buffers at the start of the level workspace: the scan operand and certificate norms of its nq queries,
// the lists of C keys, counts and thresholds of nqc queries (one chunk), the status word.  Returns their bytes, after
// which callers lay out their own regions; with the reserved workspace at base (else nullptr), points L's buffers there.
size_t level_layout(Level& L, void* base, size_t nq, size_t nqc, int C, int dpad) {
  Layout lay;
  const size_t o_qh = lay.add(nq * dpad * 2), o_hn = lay.add(nq * 4), o_en = lay.add(nq * 4), o_cand = lay.add(nqc * C * 8),
               o_count = lay.add(nqc * 4), o_thr = lay.add(nqc * 4), o_status = lay.add(256), o_sig = lay.add(nq * 8);
  if (base) {
    L.qh = region<__half>(base, o_qh);
    L.q8 = region<int8_t>(base, o_qh);
    L.qsig = region<float2>(base, o_sig);
    L.hn = region<float>(base, o_hn);
    L.en = region<float>(base, o_en);
    L.cand = region<unsigned long long>(base, o_cand);
    L.count = region<int>(base, o_count);
    L.thr = region<float>(base, o_thr);
    L.status = region<int>(base, o_status);
  }
  return lay.bytes;
}

// sizes the candidate lists of a level over the rows L.X, lays out the level workspace and converts the queries
int level_prepare(om_index* ix, Level& L, const float* qf, int nq, int k, int kp_target, int mode, int world,
                  cudaStream_t st) {
  if (k > kMaxCandidates) return fail(OM_EINVAL, "om_index_search: k = %d exceeds %d", k, kMaxCandidates);
  L.qf = qf;
  L.nq = nq;
  L.k = k;
  L.mode = mode;
  L.world = world;
  L.kp_target = std::min(std::max(kp_target, k), kMaxCandidates);
  // Row-sharded search: the global top-(k + slack) draws ~(k + slack) / W rows from every shard (binomial: mean m = kp / W,
  // deviation sqrt(m)), so each shard keeps a list of m + 6 sqrt(m) + 32 rows instead of k + slack: scan survivors, select
  // and re-score work all shrink W-fold and the whole list is shipped (no agreement phase).  A shard that holds more of the answer than its list (skewed shards) shows up
  // as a high floor: the certificate fails and the query is escalated to the 4096-wide level, which keeps full lists.
  if (world > 1 && mode == 0 && L.kp_target < kMaxCandidates) {
    const double m = static_cast<double>(L.kp_target) / world;
    L.kp_target = static_cast<int>(std::min<int64_t>(L.kp_target, round_up(static_cast<int64_t>(m + 6.0 * sqrt(m) + 32.0), 32)));
  }
  L.kp = static_cast<int>(std::min<int64_t>(L.kp_target, std::max<int64_t>(L.X.n, 1)));
  // Expected list length after a round that multiplies the rows seen by g is ~g kp (kp kept + ~(g-1) kp new
  // survivors); 25 % + 512 entries of head-room cover its spread for exchangeable row order.
  for (L.growth = ix->growth > 0 ? ix->growth : (nq <= 256 ? 8 : 2);; --L.growth) {  // large k: slower-growing schedule that fits the 16384-entry select
    L.C = 1024;
    while (L.C < (5 * L.growth * L.kp) / 4 + 512) L.C <<= 1;
    if (L.C <= 16384 || L.growth == 2) break;
  }
  if (L.C > 16384) return fail(OM_EINVAL, "om_index_search: candidate list of %d entries exceeds 16384; lower k", L.C);
  L.kc = std::min(k, L.kp_target);  // entries a shard ships per query (it cannot contribute more than k)
  L.nqc_max = std::min(nq, kQueryChunk);
  ix->st_capacity = L.C;
  Layout lay{level_layout(L, nullptr, nq, L.nqc_max, L.C, ix->dpad)};
  const size_t blk = world > 1 ? exchange_block_bytes(L.nqc_max, L.kc) : 0;
  const size_t o_send = lay.add(blk), o_recv = lay.add(blk * world);
  OM_TRY(ix->ws.reserve(lay.bytes));
  level_layout(L, ix->ws.p, nq, L.nqc_max, L.C, ix->dpad);
  L.send = world > 1 ? region<uint8_t>(ix->ws.p, o_send) : nullptr;
  L.recv = world > 1 ? region<uint8_t>(ix->ws.p, o_recv) : nullptr;
  return mode == 0 ? convert_queries(ix, L, st) : 0;
}

// One scan round over rows [pos, pos + step) of L.X for queries [q0, q0 + nqc) of the level, on the kernel the level
// and the storage choose: mode 1 the exact fp32 scan; mode 0 the int8 scan on an int8 index, else the wide cluster scan
// for threshold rounds of more than 128 queries with pair_scan on, else the GEMM core.  Survivors of thr go to the level's
// lists; dense: every score at position = column.
int scan_round(om_index* ix, const Level& L, int q0, int nqc, int64_t pos, int64_t step, bool dense, int sms, cudaStream_t st) {
  Timed t(ix, st, 0);
  const int C = L.C;
  int* overflow = L.status;
  const int ncols = static_cast<int>(step);
  const uint32_t row_base = static_cast<uint32_t>(pos);
  if (L.mode == 0 && ix->storage == OM_I8) {
    // every round on the int8 scan (pair_scan and the cluster shape do not apply)
    const int8_t* qhi = L.q8 + static_cast<size_t>(q0) * ix->dpad;
    const int8_t* qlo = L.q8 + (static_cast<size_t>(L.nq) + q0) * ix->dpad;
    const int64_t pitch = pitch_of(L.X.xq, ix->d);
    const cudaError_t e = launch_scan_i8(dense, L.allow, qhi, qlo, ix->dpad, L.qsig + q0, L.X.xq + pos * pitch, pitch,
                                         ix->dpad, nqc, ncols, ix->d, L.thr, L.cand, L.count, overflow, C, row_base, sms, st);
    if (e != cudaSuccess) return fail(OM_ECUDA, "int8 scan kernel launch failed: %s", cudaGetErrorString(e));
  } else if (L.mode == 0) {
    const __half* qh = L.qh + static_cast<size_t>(q0) * ix->dpad;
    const __half* xrows = L.X.xh + static_cast<size_t>(pos) * ix->dpad;
    cudaError_t e;
    // a cluster owns at least 2 x 128 query rows per tile: with <= 128 queries the peers' boxes would be padding (and the sweep is
    // HBM-bound there, where the dynamic tile order of the single-CTA kernel matters more than operand sharing).  The
    // first, dense round (C rows, every score stored) stays on the single-CTA kernel as well.
    const bool pair = ix->pair_scan != 0 && nqc > kBlockM;
    if (!dense && pair) {
      // cluster shape CQ x CX: the index parameters, else 2 x 1.  The wider shapes cut L2 -> SM traffic by 25 - 50 %, but
      // only 30 clusters of 4 and 15 of 8 CTAs fit an H100 SXM (120 SMs, against 66 pairs on all 132), and the whole
      // search measured no faster on any of them beyond run-to-run noise at C2 and slower at C5 (DESIGN §7)
      const int cq = ix->scan_cq ? ix->scan_cq : 2, cx = ix->scan_cx ? ix->scan_cx : 1;
      int clusters = 0;
      e = launch_scan_cluster(cq, cx, qh, ix->dpad, xrows, ix->dpad, nqc, ncols, ix->d, L.thr, L.cand, L.count, overflow, C,
                              row_base, L.allow, sms, st, &clusters);
      ix->st_scan_cluster = 10 * cq + cx;
      ix->st_scan_clusters = clusters;
    } else {
      e = launch_scan_core(dense, L.allow, qh, ix->dpad, xrows, ix->dpad, nqc, ncols, ix->d, L.thr, L.cand, L.count, overflow,
                           C, row_base, sms, st);
    }
    if (e != cudaSuccess) return fail(OM_ECUDA, "scan kernel launch failed: %s", cudaGetErrorString(e));
  } else {
    // the filter variant (a filtered exact round) keeps the queries' excluded ids in shared memory after the queries
    const bool exact_filter = L.allow || L.ex.off;
    Excluded ex = L.ex;
    ex.q_base = q0;
    const float* qf = L.qf + static_cast<size_t>(q0) * ix->d;
    const int nqt = std::max(1, std::min(8, (96 * 1024) / (ix->d * 4)));
    dim3 grid(static_cast<unsigned>(std::min<int64_t>((step + 15) / 16, static_cast<int64_t>(sms) * 4)),
              static_cast<unsigned>((nqc + nqt - 1) / nqt));
    const size_t smem = static_cast<size_t>(nqt) * ix->d * 4 + (exact_filter ? 8 * kMaxExcluded * 4 : 0);
    with_rows(ix, L.X, [&](const auto* xs) {
      using RowT = std::decay_t<decltype(*xs)>;
      const auto kernel = exact_filter ? exact_scan_kernel<8, 2, RowT, true> : exact_scan_kernel<8, 2, RowT>;
      kernel<<<grid, 256, smem, st>>>(xs + pos * pitch_of(xs, ix->d), step, row_base, qf, nqc, ix->d, nqt, L.thr, L.cand,
                                      L.count, overflow, C, dense ? 1 : 0, L.allow, exact_filter ? ex : Excluded{});
    });
    OM_CUDA(cudaGetLastError());
  }
  return 0;
}

// One sweep of the rows L.X for queries [q0, q0 + nqc) of the level.  safe = false: doubling rounds; safe = true: fixed
// rounds of C - kp rows, which cannot overflow.  mode 0: tensor-core scan (fp16; int8 index: scan_i8.cuh), 1: exact fp32
// scan.
int sweep_chunk(om_index* ix, const Level& L, int q0, int nqc, bool safe, int sms, cudaStream_t st) {
  const int64_t growth = L.growth;
  const int64_t N = L.X.n;
  const int C = L.C, kp = L.kp;
  if (N == 0) {
    fill_i32<<<(nqc + 255) / 256, 256, 0, st>>>(L.count, 0, nqc);
    fill_i32<<<(nqc + 255) / 256, 256, 0, st>>>(reinterpret_cast<int*>(L.thr), static_cast<int>(0xff800000), nqc);
    OM_CUDA(cudaGetLastError());
    return 0;
  }
  int64_t pos = 0;
  const size_t sel_smem = static_cast<size_t>(C) * 8;
  bool first = true;
  // Filtered search: the scan must not store the rows the filter drops, so instead of the dense first round (every score
  // at position = column, kp counted over all C rows) the first round is a threshold round at -inf: every allowed row
  // survives, and select counts the list, which holds allowed rows only.  Later rounds filter as usual.  The exact scan
  // drops excluded ids as well, so its lists (k rows) hold no excluded row either.
  const bool sparse_first = L.allow || (L.mode == 1 && L.ex.off);
  // With a bitmap, rounds are sized in allowed rows (L.allow_prefix, per 256-row block), as they would be in rows on an
  // index of the allowed rows alone: the first round takes up to C allowed rows, a doubling round (growth - 1) x the
  // allowed rows seen, a safe round C - kp.  So a round at threshold -inf (fewer than kp allowed rows seen) cannot
  // overflow its list however the allowed rows are placed, and stretches of disallowed rows join the next round.
  // Returns the end of the round from pos: the last block boundary (or N) whose allowed rows since pos stay within
  // budget, one block at least.  seen(b): allowed rows of X before block b.
  const int64_t* A = L.allow_prefix;
  auto seen = [&](int64_t b) { return A[b] - A[0]; };
  auto allowed_end = [&](int64_t from, int64_t budget) -> int64_t {
    const int64_t b0 = from / 256;
    int64_t b = std::upper_bound(A + b0 + 1, A + (N + 255) / 256 + 1, A[b0] + budget) - A - 1;
    b = std::max(b, b0 + 1);
    return std::min<int64_t>(b * 256, N);
  };
  if (sparse_first) {
    fill_i32<<<(nqc + 255) / 256, 256, 0, st>>>(L.count, 0, nqc);
    fill_i32<<<(nqc + 255) / 256, 256, 0, st>>>(reinterpret_cast<int*>(L.thr), static_cast<int>(0xff800000), nqc);
    OM_CUDA(cudaGetLastError());
  }
  while (pos < N) {
    int64_t step;
    if (L.allow)
      step = allowed_end(pos, first ? C : safe ? C - kp : (growth - 1) * seen(pos / 256)) - pos;
    else if (first)
      step = std::min<int64_t>(N, C);
    else if (safe)
      step = std::min<int64_t>(N - pos, std::max<int64_t>(256, ((C - kp) / 256) * 256));
    else
      step = std::min<int64_t>(N - pos, (growth - 1) * pos);
    // a first round of allowed rows only (an allow-all bitmap, a sub-collection at the start of the shard) stores densely
    // as the unfiltered search does: nothing there for the filter to drop
    const bool dense = first && (!sparse_first || (L.mode == 0 && L.allow && seen((pos + step + 255) / 256) == step));
    OM_TRY(scan_round(ix, L, q0, nqc, pos, step, dense, sms, st));
    {
      Timed t(ix, st, 1);
      select_kernel<<<nqc, 256, sel_smem, st>>>(L.cand, L.count, L.thr, C, kp, dense ? static_cast<int>(step) : -1);
    }
    OM_CUDA(cudaGetLastError());
    ix->st_launches += 2;
    pos += step;
    first = false;
    ix->st_rounds++;
  }
  return 0;
}

int finalize_chunk(om_index* ix, const Level& L, int q0, int nqc, float* D, int64_t* I, int k_out, int64_t id_offset,
                   cudaStream_t st) {
  int P2 = 2;
  while (P2 < L.kp) P2 <<= 1;
  const bool filter = L.ex.off != nullptr;  // the filter variant keeps the query's excluded ids after the query
  const size_t fin_smem = static_cast<size_t>(P2) * 8 + static_cast<size_t>(ix->d) * 4 + (filter ? kMaxExcluded * 4 : 0);
  {
    Timed t(ix, st, 2);
    const float* qf = L.qf + static_cast<size_t>(q0) * ix->d;
    Excluded ex = L.ex;
    ex.q_base = q0;
    with_rows(ix, L.X, [&](const auto* xs) {
      using RowT = std::decay_t<decltype(*xs)>;
      const auto kernel = filter ? finalize_kernel<RowT, true> : finalize_kernel<RowT>;
      kernel<<<nqc, 256, fin_smem, st>>>(L.cand, L.count, L.C, qf, xs, ix->d, D, I, id_offset, k_out, ix->stage_scores,
                                         filter ? ex : Excluded{});
    });
  }
  OM_CUDA(cudaGetLastError());
  ix->st_launches += 1;
  return 0;
}

// Merge of nparts [nq, k_in] lists -> [nq, k_out]; more than 8192 entries per query are merged hierarchically.
int merge_parts(const float* Dp, const int64_t* Ip, int64_t stride_d, int64_t stride_i, int nparts, int nq, int k_in,
                int k_out, float* D, int64_t* I, cudaStream_t st) {
  OM_TRY(once_attrs(nullptr));
  if (k_in > 8192) return fail(OM_EINVAL, "om_topk_merge_n: k_in = %d exceeds 8192", k_in);
  if (static_cast<int64_t>(nparts) * k_in <= 8192) {
    int P = 2;
    while (P < nparts * k_in) P <<= 1;
    const size_t smem = static_cast<size_t>(P) * 8 + static_cast<size_t>(nparts) * k_in * 8;
    merge_kernel<<<nq, 256, smem, st>>>(Dp, Ip, stride_d, stride_i, nparts, nq, k_in, k_out, D, I);
    OM_CUDA(cudaGetLastError());
    return 0;
  }
  // groups of g parts -> intermediate lists of width k_mid, then recurse on the groups.  Each level shrinks only if a
  // group of g >= 2 parts fits one merge (k_in <= 4096) and the groups' lists stay that narrow (k_out <= 4096); otherwise
  // the part count never drops and the recursion would not end.
  if (k_in > 4096 || k_out > 4096)
    return fail(OM_EINVAL, "om_topk_merge_n: %d parts x %d entries exceed one merge of 8192 and need k_in, k_out <= 4096 "
                "(got k_in = %d, k_out = %d)", nparts, k_in, k_in, k_out);
  const int g = std::max(2, 8192 / k_in);
  const int ngroups = (nparts + g - 1) / g;
  const int k_mid = static_cast<int>(std::min<int64_t>(k_out, static_cast<int64_t>(g) * k_in));
  float* Dm = nullptr;
  int64_t* Im = nullptr;
  const size_t per = static_cast<size_t>(nq) * k_mid;
  OM_CUDA(cudaMallocAsync(&Dm, per * ngroups * 4, st));
  OM_CUDA(cudaMallocAsync(&Im, per * ngroups * 8, st));
  int rc = 0;
  for (int gi = 0; gi < ngroups && rc == 0; ++gi) {
    const int p0 = gi * g, np = std::min(g, nparts - p0);
    rc = merge_parts(Dp + p0 * stride_d, Ip + p0 * stride_i, stride_d, stride_i, np, nq, k_in, k_mid, Dm + gi * per,
                     Im + gi * per, st);
  }
  if (rc == 0) rc = merge_parts(Dm, Im, static_cast<int64_t>(per), static_cast<int64_t>(per), ngroups, nq, k_mid, k_out, D, I, st);
  cudaFreeAsync(Dm, st);
  cudaFreeAsync(Im, st);
  return rc;
}

// Exchange of one query chunk of a row-sharded level: every shard re-scores its (shard-sized) candidate list in fp32 and
// ships it whole — sorted scores, global ids, the list's stage-score floor and the shard's error-norm maxima — in ONE
// packed all-gather; every rank then merges the W lists.  (The certificate is run by the caller on the merged result.)
int exchange_chunk(om_index* ix, om_comm* comm, const Level& L, int q0, int nqc, float* dD, int64_t* dI, int64_t id_offset,
                   cudaStream_t st) {
  NcclApi& nc = nccl_api();
  const int W = comm->world;
  const ExchangeBlock b = exchange_block(nqc, L.kc);
  OM_TRY(finalize_chunk(ix, L, q0, nqc, reinterpret_cast<float*>(L.send), reinterpret_cast<int64_t*>(L.send + b.off_i), L.kc,
                        id_offset, st));
  {
    Timed t(ix, st, 3);
    OM_CUDA(cudaMemcpyAsync(L.send + b.off_floor, L.thr, static_cast<size_t>(nqc) * 4, cudaMemcpyDeviceToDevice, st));
    OM_CUDA(cudaMemcpyAsync(L.send + b.off_stats, ix->gstats, 8, cudaMemcpyDeviceToDevice, st));
    OM_NCCL(nc.AllGather(L.send, L.recv, b.bytes, kNcclInt8, comm->nccl, st));
    OM_TRY(merge_parts(reinterpret_cast<const float*>(L.recv), reinterpret_cast<const int64_t*>(L.recv + b.off_i),
                       static_cast<int64_t>(b.bytes / 4), static_cast<int64_t>(b.bytes / 8), W, nqc, L.kc, L.k,
                       dD + static_cast<size_t>(q0) * L.k, dI + static_cast<size_t>(q0) * L.k, st));
  }
  ix->st_launches += 2;
  return 0;
}

// Runs one level over all its queries and lists the uncertified ones, ascending, in `uncertified`.  One host
// synchronisation at the end (status word), and one more to read the certificate's per-query flags when a query is
// uncertified; a list overflow redoes the level with the safe schedule.  comm: a row-sharded level (nullptr: one shard).
int run_level(om_index* ix, om_comm* comm, Level& L, float* dD, int64_t* dI, int64_t id_offset, int* flags,
              std::vector<int>& uncertified, cudaStream_t st) {
  const int sms = device_sm_count();
  if (sms < 0) return sms;
  NvtxRange nvtx(L.mode == 1 ? "om.search.level_exact" : (L.kp_target >= kMaxCandidates ? "om.search.level_wide" : "om.search.level0"));
  const bool sharded = comm != nullptr;
  bool safe = ix->force_safe != 0;
  const bool certify = ix->certify && L.mode == 0 && !ix->stage_scores;
  for (int attempt = 0; attempt < 4; ++attempt) {
    OM_CUDA(cudaMemsetAsync(L.status, 0, 32, st));
    for (int q0 = 0; q0 < L.nq; q0 += kQueryChunk) {
      const int nqc = std::min(kQueryChunk, L.nq - q0);
      OM_TRY(sweep_chunk(ix, L, q0, nqc, safe, sms, st));
      if (sharded)
        OM_TRY(exchange_chunk(ix, comm, L, q0, nqc, dD, dI, id_offset, st));
      else
        OM_TRY(finalize_chunk(ix, L, q0, nqc, dD + static_cast<size_t>(q0) * L.k, dI + static_cast<size_t>(q0) * L.k, L.k,
                              id_offset, st));
      if (certify) {
        Timed t(ix, st, 3);
        const ExchangeBlock b = exchange_block(nqc, L.kc);
        const float* floors = sharded ? reinterpret_cast<const float*>(L.recv + b.off_floor) : L.thr;
        const float* gst = sharded ? reinterpret_cast<const float*>(L.recv + b.off_stats) : ix->gstats;
        certify_kernel<<<(nqc + 7) / 8, 256, 0, st>>>(dD + static_cast<size_t>(q0) * L.k, dI + static_cast<size_t>(q0) * L.k,
                                                      L.k, floors, static_cast<int64_t>(b.bytes / 4), sharded ? comm->world : 1,
                                                      gst, static_cast<int64_t>(b.bytes / 4), L.hn + q0, L.en + q0, ix->d, nqc,
                                                      q0, flags, L.status + 2);
        OM_CUDA(cudaGetLastError());
        ix->st_launches += 1;
      }
    }
    // every rank must take the same retry decision (list overflow on any shard)
    OM_TRY(read_decision(ix, comm, L.status, 4, kNcclMax, 0, st));
    const unsigned int fault = read_clear_dev_fault();
    if (fault) return fail(OM_EFAULT, "scan kernel pipeline fault 0x%08x", fault);
    if (ix->h_status[0]) {
      if (safe) return fail(OM_EFAULT, "candidate list overflow in the overflow-proof schedule (bug)");
      safe = true;
      ix->st_retries++;
      continue;
    }
    uncertified.clear();
    if (certify && ix->h_status[2] > 0) {  // the flags, and so the list, are identical on every rank
      std::vector<int> flagged(L.nq);
      OM_CUDA(cudaMemcpyAsync(flagged.data(), flags, flagged.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
      OM_CUDA(cudaStreamSynchronize(st));
      for (int i = 0; i < L.nq; ++i)
        if (flagged[i]) uncertified.push_back(i);
    }
    return 0;
  }
  return fail(OM_EFAULT, "search level did not converge (bug)");
}

// fp16 / int8 storage: rows written in place may hold values the storage cannot represent (inf from an overflowing encoder
// output, NaN; int8: a non-finite scale), and there is no fp32 copy to answer from, so the search is refused until
// om_index_reset.  Sharded: the shards' counts are summed into the scratch int so that every rank takes the same decision.
// One host synchronisation; fp32 indices skip the check.
int check_finite_rows(om_index* ix, om_comm* comm, cudaStream_t st) {
  if (ix->storage == OM_F32) return 0;
  const bool sharded = comm && comm->world > 1;
  OM_TRY(read_decision(ix, sharded ? comm : nullptr, reinterpret_cast<int*>(ix->gstats) + 2, 2, kNcclSum, 1, st));
  ix->st_nonfinite = ix->h_status[0];
  const int total = sharded ? ix->h_status[1] : ix->h_status[0];
  if (total > 0)
    return fail(OM_EINVAL, "search: %d committed %s rows hold inf or NaN (%d on this shard); the storage cannot answer "
                "exactly over them: reset the index", total, ix->storage == OM_I8 ? "int8" : "fp16", ix->h_status[0]);
  return 0;
}

// A search filter's argument rules (om_search_filter), checked on `st` before the search writes anything: the bitmap
// covers the shard, and every query excludes at most kMaxExcluded ids, none negative, through monotone offsets.
// Sharded (comm): every rank takes part (its filter may be null or empty) and takes the decision of all of them.  A valid
// bitmap also leaves its allowed rows per 256-row block in ix->allow_prefix, from which sweep_chunk sizes the rounds.  One
// host synchronisation.
int check_filter(om_index* ix, om_comm* comm, const om_search_filter* f, int nq, cudaStream_t st) {
  const om_search_filter none = {nullptr, 0, nullptr, nullptr};
  if (!f) f = &none;
  int* bad = ix->scratch();
  const bool short_bits = f->allow_bits && f->allow_words < (ix->n + 31) / 32;
  fill_i32<<<1, 1, 0, st>>>(bad, short_bits ? 8 : 0, 1);
  if (f->exclude_offsets)
    check_exclusions_kernel<<<grid_for(nq, 256), 256, 0, st>>>(f->exclude_offsets, f->exclude_ids, nq, bad);
  OM_CUDA(cudaGetLastError());
  const int64_t nblocks = (ix->n + 255) / 256;
  std::vector<int> counts;
  if (f->allow_bits && !short_bits && nblocks > 0) {
    OM_TRY(ix->ows.reserve(static_cast<size_t>(nblocks) * 4));
    allow_block_counts_kernel<<<grid_for(nblocks, 256), 256, 0, st>>>(f->allow_bits, ix->n, nblocks,
                                                                       static_cast<int*>(ix->ows.p));
    OM_CUDA(cudaGetLastError());
    counts.resize(nblocks);
    OM_CUDA(cudaMemcpyAsync(counts.data(), ix->ows.p, static_cast<size_t>(nblocks) * 4, cudaMemcpyDeviceToHost, st));
  }
  OM_TRY(read_decision(ix, comm, bad, 1, kNcclMax, 0, st));
  ix->allow_prefix.assign(1, 0);
  for (int c : counts) ix->allow_prefix.push_back(ix->allow_prefix.back() + c);
  const int b = ix->h_status[0];
  if (b & 8)
    return fail(OM_EINVAL, "search filter: allow_words = %lld is fewer than the %lld words of the %lld rows%s",
                (long long)f->allow_words, (long long)((ix->n + 31) / 32), (long long)ix->n, comm ? " (or on another rank)" : "");
  if (b & 2) return fail(OM_EINVAL, "search filter: a query excludes more than %d ids", kMaxExcluded);
  if (b & 1) return fail(OM_EINVAL, "search filter: exclude_offsets must be non-negative and non-decreasing, with exclude_ids given");
  if (b & 4) return fail(OM_EINVAL, "search filter: an excluded id is negative");
  return 0;
}

// The start of a search or a range search (`who` in the messages), before it writes anything: the per-call stats, the
// shared-memory opt-ins, the d limit, the host queries staged in ix->ows after the caller's regions in `ows`, and the
// stored rows' finiteness.  A range search passes its radii: staged likewise, and refused on every rank if one is NaN.
// *qf (and *rho): the device queries (and radii).
int call_prologue(om_index* ix, om_comm* comm, const char* who, const void* q, om_memkind q_kind, int nq, const float* radius,
                  Layout& ows, const float** qf, const float** rho, cudaStream_t st) {
  ix->st_rounds = ix->st_retries = ix->st_launches = 0;
  ix->st_flagged = ix->st_flagged_wide = ix->st_exact = 0;
  ix->st_scan_cluster = ix->st_scan_clusters = 0;
  ix->st_scan_us = ix->st_select_us = ix->st_final_us = ix->st_other_us = ix->st_upload_wait_us = 0;
  ix->st_partitions = 1;
  ix->ev_used = 0;
  OM_TRY(once_attrs(ix));
  if (ix->d > 16384) return fail(OM_EINVAL, "%s: d > 16384 unsupported", who);
  const bool host = q_kind == OM_HOST;
  const size_t q_bytes = static_cast<size_t>(nq) * ix->d * 4, rho_bytes = static_cast<size_t>(nq) * 4;
  const size_t o_q = ows.add(host ? q_bytes : 0), o_rho = ows.add(host && radius ? rho_bytes : 0);
  OM_TRY(ix->ows.reserve(ows.bytes));
  *qf = static_cast<const float*>(q);
  if (host) {
    OM_CUDA(cudaMemcpyAsync(region<void>(ix->ows.p, o_q), q, q_bytes, cudaMemcpyHostToDevice, st));
    *qf = region<const float>(ix->ows.p, o_q);
  }
  if (radius) {
    *rho = radius;
    if (host) {
      OM_CUDA(cudaMemcpyAsync(region<void>(ix->ows.p, o_rho), radius, rho_bytes, cudaMemcpyHostToDevice, st));
      *rho = region<const float>(ix->ows.p, o_rho);
    }
    int* bad = ix->scratch();
    OM_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), st));
    check_radius_kernel<<<grid_for(nq, 256), 256, 0, st>>>(*rho, nq, bad);
    OM_CUDA(cudaGetLastError());
    OM_TRY(read_decision(ix, comm, bad, 1, kNcclMax, 0, st));
    if (ix->h_status[0]) return fail(OM_EINVAL, "%s: a radius is NaN%s", who, comm ? " (on some rank)" : "");
  }
  return check_finite_rows(ix, comm, st);
}

// Uploads `list` (indices into the call's queries) to dlist and gathers the listed rows of src (rows of d floats) into
// dst: the queries of a sub-batch.
int gather_listed(const std::vector<int>& list, int* dlist, const float* src, int d, float* dst, cudaStream_t st) {
  const int m = static_cast<int>(list.size());
  OM_CUDA(cudaMemcpyAsync(dlist, list.data(), list.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  gather_rows_kernel<<<grid_for(static_cast<int64_t>(m) * d, 256), 256, 0, st>>>(src, dlist, m, d, dst);
  OM_CUDA(cudaGetLastError());
  return 0;
}

// The levels of a search over the rows X, the rows [p0, p0 + X.n) of the index (p0 a multiple of 256): level 0 (all
// queries, k + slack candidates) -> level 1 (uncertified queries, widest list) -> level 2 (still uncertified: exact fp32
// scan), into the device results (dD, dI) with ids id_offset + p0 + row.  comm == nullptr: single shard.  f: nullptr, or a
// checked filter with at least one part, over all the index's rows.  flags: nq ints of scratch.
int search_rows(om_index* ix, om_comm* comm, const Rows& X, int64_t p0, const float* qf, int nq, int k, float* dD, int64_t* dI,
                int64_t id_offset, const om_search_filter* f, int* flags, cudaStream_t st) {
  const int d = ix->d;
  const int world = comm ? comm->world : 1;
  // the filter of every level: X's slice of the bitmap, and the exclusions of the level's queries (qmap: the escalated ones)
  auto filter = [&](Level& L, const int* qmap) {
    if (!f) return;
    L.allow = f->allow_bits ? f->allow_bits + p0 / 32 : nullptr;
    L.allow_prefix = ix->allow_prefix.data() + p0 / 256;
    L.ex = Excluded{f->exclude_offsets, f->exclude_ids, qmap, 0, id_offset + p0};
  };
  const int64_t slack = ix->rescore_slack >= 0 ? ix->rescore_slack : std::max<int64_t>(128, k / 5);
  const int kp0 = static_cast<int>(std::min<int64_t>(static_cast<int64_t>(k) + slack, kMaxCandidates));
  std::vector<int> list, sub;  // uncertified queries: indices into the call's queries, into the last sub-batch
  {  // level 0; exact_only: the exact scan of every query, which leaves none uncertified
    Level L;
    L.X = X;
    if (ix->exact_only) ix->st_exact += nq;
    OM_TRY(level_prepare(ix, L, qf, nq, k, ix->exact_only ? k : kp0, ix->exact_only ? 1 : 0, world, st));
    filter(L, nullptr);
    OM_TRY(run_level(ix, comm, L, dD, dI, id_offset + p0, flags, list, st));
    ix->st_flagged += static_cast<int64_t>(list.size());
  }
  // Escalation: the queries in `list` are gathered into a compact sub-batch, answered by one more level and scattered back
  // over their rows of (dD, dI); `sub` lists the ones the level left uncertified.  sws holds the uploaded list (the
  // sub-batch's qmap), the gathered queries and the level's results.
  auto run_sub = [&](int kp_target, int mode) -> int {
    const size_t n_sub = list.size();
    Layout sws;
    const size_t s_list = sws.add(n_sub * 4), s_q = sws.add(n_sub * d * 4), s_D = sws.add(n_sub * k * 4),
                 s_I = sws.add(n_sub * k * 8);
    OM_TRY(ix->sws.reserve(sws.bytes));
    int* dlist = region<int>(ix->sws.p, s_list);
    float* qsub = region<float>(ix->sws.p, s_q);
    float* Ds = region<float>(ix->sws.p, s_D);
    int64_t* Is = region<int64_t>(ix->sws.p, s_I);
    OM_TRY(gather_listed(list, dlist, qf, d, qsub, st));
    Level Ls;
    Ls.X = X;
    OM_TRY(level_prepare(ix, Ls, qsub, static_cast<int>(n_sub), k, kp_target, mode, world, st));
    filter(Ls, dlist);
    OM_TRY(run_level(ix, comm, Ls, Ds, Is, id_offset + p0, flags, sub, st));
    scatter_results_kernel<<<grid_for(static_cast<int64_t>(n_sub) * k, 256), 256, 0, st>>>(Ds, Is, dlist, static_cast<int>(n_sub),
                                                                                            k, dD, dI);
    OM_CUDA(cudaGetLastError());
    ix->st_launches += 2;
    return 0;
  };
  if (!list.empty()) {
    // level 1: widest candidate list the select / sort kernels take.  (Sharded: the decision must not depend on this
    // rank's row count — every rank runs the same levels.)
    if (kp0 < kMaxCandidates && (world > 1 || X.n > kp0)) {
      OM_TRY(run_sub(kMaxCandidates, 0));
      for (int& i : sub) i = list[i];
      list.swap(sub);
    }
    ix->st_flagged_wide += static_cast<int64_t>(list.size());
    if (!list.empty()) {  // level 2: exact fp32 scan
      ix->st_exact += static_cast<int64_t>(list.size());
      OM_TRY(run_sub(k, 1));
    }
  }
  return 0;
}

// The partition p upload of a host-resident index into window p % 2, on the copy stream: it waits until the search has
// left the window (ev_free), copies the partition's chunk in one piece and marks the window ready (ev_ready).
int upload_partition(om_index* ix, int64_t p) {
  const int w = static_cast<int>(p & 1);
  const int64_t rows = std::min(ix->window, ix->n - p * ix->window);
  Rows X;
  OM_TRY(window_reserve(ix, w, rows, &X));
  const void* dst = with_rows(ix, X, [](const auto* xs) -> const void* { return xs; });
  OM_CUDA(cudaStreamWaitEvent(ix->copy_st, ix->ev_free[w], 0));
  OM_CUDA(cudaMemcpyAsync(const_cast<void*>(dst), ix->chunks[p], static_cast<size_t>(rows) * host_row_bytes(ix),
                          cudaMemcpyHostToDevice, ix->copy_st));
  OM_CUDA(cudaEventRecord(ix->ev_ready[w], ix->copy_st));
  return 0;
}

// The search of a host-resident index: each partition of `window` rows is uploaded while the previous one is searched,
// searched by search_rows with its row offset, and merged into the running result by (score desc, id asc).  Each
// partition's result is the exact top-k of its rows, and an fp32 score does not depend on the rows around it, so the merge
// is bitwise the search of one device index of all the rows.  R, RI: [2, nq, k] scratch (running result, partition result).
int search_host(om_index* ix, const float* qf, int nq, int k, float* dD, int64_t* dI, int64_t id_offset,
                const om_search_filter* f, int* flags, float* R, int64_t* RI, cudaStream_t st) {
  const int64_t W = ix->window, N = ix->n;
  const int64_t np = (N + W - 1) / W;
  if (np <= 1) {
    ix->st_partitions = 1;
    if (N == 0) return search_rows(ix, nullptr, Rows{}, 0, qf, nq, k, dD, dI, id_offset, f, flags, st);
  } else {
    ix->st_partitions = np;
  }
  // whatever way the call ends, no upload is left running into the windows
  struct CopyDone {
    cudaStream_t s;
    ~CopyDone() { cudaStreamSynchronize(s); }
  } copy_done{ix->copy_st};
  // both windows are sized before the first upload: a reservation that grows a window frees it
  Rows X;
  OM_TRY(window_reserve(ix, 0, std::min(W, N), &X));
  if (np > 1) OM_TRY(window_reserve(ix, 1, std::min(W, N - W), &X));
  OM_CUDA(cudaEventRecord(ix->ev_entry, st));  // uploads start after the caller's earlier work on st
  OM_CUDA(cudaStreamWaitEvent(ix->copy_st, ix->ev_entry, 0));
  OM_TRY(upload_partition(ix, 0));
  const size_t slot = static_cast<size_t>(nq) * k;
  for (int64_t p = 0; p < np; ++p) {
    if (p + 1 < np) OM_TRY(upload_partition(ix, p + 1));
    const int w = static_cast<int>(p & 1);
    {
      Timed t(ix, st, 4);
      OM_CUDA(cudaStreamWaitEvent(st, ix->ev_ready[w], 0));
    }
    OM_TRY(window_reserve(ix, w, std::min(W, N - p * W), &X));
    if (ix->storage == OM_F32) {  // the scan copy, as om_index_commit builds it
      rows_to_f16_kernel<<<grid_for(X.n, 8), 256, 0, st>>>(X.xf, const_cast<__half*>(X.xh), X.n, ix->d, ix->dpad, nullptr,
                                                           nullptr, nullptr);
      OM_CUDA(cudaGetLastError());
      ix->st_launches += 1;
    }
    float* Dp = np == 1 ? dD : R + (p > 0 ? slot : 0);
    int64_t* Ip = np == 1 ? dI : RI + (p > 0 ? slot : 0);
    OM_TRY(search_rows(ix, nullptr, X, p * W, qf, nq, k, Dp, Ip, id_offset, f, flags, st));
    OM_CUDA(cudaEventRecord(ix->ev_free[w], st));
    if (p > 0) {
      OM_TRY(merge_parts(R, RI, static_cast<int64_t>(slot), static_cast<int64_t>(slot), 2, nq, k, k, dD, dI, st));
      ix->st_launches += 1;
      if (p + 1 < np) {
        OM_CUDA(cudaMemcpyAsync(R, dD, slot * 4, cudaMemcpyDeviceToDevice, st));
        OM_CUDA(cudaMemcpyAsync(RI, dI, slot * 8, cudaMemcpyDeviceToDevice, st));
      }
    }
  }
  return 0;
}

// The whole search of a device index (search_rows over its rows) or of a host-resident one (search_host), from the
// caller's queries to the caller's results.
int search_impl(om_index* ix, om_comm* comm, const void* q, om_memkind q_kind, int nq, int k, float* D, int64_t* I,
                om_memkind out_kind, int64_t id_offset, const om_search_filter* f, cudaStream_t st) {
  NvtxRange nvtx("om.search");
  const bool host_rows = ix->window > 0;
  // whole-search staging: results (if they leave to the host), the certificate's per-query flags, a host-resident index's
  // running and partition results, queries (in the prologue)
  Layout ows;
  const size_t o_D = ows.add(out_kind == OM_HOST ? static_cast<size_t>(nq) * k * 4 : 0);
  const size_t o_I = ows.add(out_kind == OM_HOST ? static_cast<size_t>(nq) * k * 8 : 0);
  const size_t o_flags = ows.add(static_cast<size_t>(nq) * 4);
  const size_t o_R = ows.add(host_rows ? 2 * static_cast<size_t>(nq) * k * 4 : 0);
  const size_t o_RI = ows.add(host_rows ? 2 * static_cast<size_t>(nq) * k * 8 : 0);
  const float* qf = nullptr;
  OM_TRY(call_prologue(ix, comm, "om_index_search", q, q_kind, nq, nullptr, ows, &qf, nullptr, st));
  float* dD = out_kind == OM_HOST ? region<float>(ix->ows.p, o_D) : D;
  int64_t* dI = out_kind == OM_HOST ? region<int64_t>(ix->ows.p, o_I) : I;
  int* flags = region<int>(ix->ows.p, o_flags);
  if (host_rows)
    OM_TRY(search_host(ix, qf, nq, k, dD, dI, id_offset, f, flags, region<float>(ix->ows.p, o_R), region<int64_t>(ix->ows.p, o_RI),
                       st));
  else
    OM_TRY(search_rows(ix, comm, device_rows(ix), 0, qf, nq, k, dD, dI, id_offset, f, flags, st));
  if (out_kind == OM_HOST) {
    OM_CUDA(cudaMemcpyAsync(D, dD, static_cast<size_t>(nq) * k * 4, cudaMemcpyDeviceToHost, st));
    OM_CUDA(cudaMemcpyAsync(I, dI, static_cast<size_t>(nq) * k * 8, cudaMemcpyDeviceToHost, st));
  }
  OM_CUDA(cudaStreamSynchronize(st));
  if (ix->profile) collect_profile(ix);
  return 0;
}

// ---- range search ---------------------------------------------------------------------------------------------------
// A list count starts a round at most kRangeMaxList (its fill) and a round adds at most kRangeRound: 2^30 + 2^29 < 2^31, so
// the scans' int counters cannot wrap.
constexpr int64_t kRangeRound = int64_t(1) << 29;  // rows per scan round
constexpr int kRangeMaxList = 1 << 30;             // longest candidate list of one query

// Grows b to `need` bytes, keeping its first `keep` bytes.
int grow_keep(DevBuf& b, size_t keep, size_t need, cudaStream_t st) {
  if (need <= b.bytes) return 0;
  need = std::max(need, b.bytes + b.bytes / 2);
  void* p = nullptr;
  if (dev_malloc(&p, need) != cudaSuccess) {
    cudaGetLastError();
    return fail(OM_ENOMEM, "range search: cannot allocate %zu bytes of results", need);
  }
  if (keep) OM_CUDA(cudaMemcpyAsync(p, b.p, keep, cudaMemcpyDeviceToDevice, st));
  OM_CUDA(cudaStreamSynchronize(st));
  b.release();
  b.p = p;
  b.bytes = need;
  return 0;
}

// Per query of one range sweep: the candidates the scans counted, the rows above rho among them (when they fit) and
// whether the query needs the exact scan.
struct RangeSweep {
  std::vector<long long> total;
  std::vector<int> surv, to_exact;
};

// One sweep of a range search over queries list[0, m) (rows of qf / rho) with lists of C keys: mode 0 the tensor-core
// scan at t(q), mode 1 the exact scan at rho; then re-score, cut and sort of every list that holds all its query's
// candidates.  One host synchronisation; the answered queries' sorted keys are appended to ix->rkeys at *stored, and
// src[g] / cnt[g] record where and how many for query g.  f: nullptr, or a checked filter with at least one part; the
// scans then store allowed rows only (the exact scan also drops excluded ids), and the re-score drops excluded ids.
// Exclusions are read through the uploaded list (qmap: sweep query i is the caller's query list[i]), as ids id_offset + row.
int range_sweep(om_index* ix, const float* qf, const float* rho, const std::vector<int>& list, int mode, int C, int sms,
                const om_search_filter* f, int64_t id_offset, int64_t* stored, std::vector<int64_t>& src,
                std::vector<int64_t>& cnt, RangeSweep& r, cudaStream_t st) {
  const int m = static_cast<int>(list.size()), d = ix->d;
  const size_t M = m;
  const bool long_lists = C > kRangeSortKeys;
  Level L;
  Layout lay{level_layout(L, nullptr, M, M, C, ix->dpad)};
  const size_t o_list = lay.add(M * 4), o_q = lay.add(M * d * 4), o_rho = lay.add(M * 4),
               o_alt = lay.add(long_lists ? M * C * 8 : 0), o_filled = lay.add(M * 4), o_total = lay.add(M * 8),
               o_surv = lay.add(M * 4), o_exact = lay.add(M * 4), o_off = lay.add(M * 8);
  if (C == ix->range_list) ix->r_keep_ws = std::max(ix->r_keep_ws, lay.bytes);  // a first sweep's workspace
  if (ix->ws.reserve(lay.bytes) != 0) {
    cudaGetLastError();
    return fail(OM_ENOMEM, "range search: cannot allocate candidate lists of %d queries x %d rows", m, C);
  }
  void* b = ix->ws.p;
  level_layout(L, b, M, M, C, ix->dpad);
  int* dlist = region<int>(b, o_list);
  float* q = region<float>(b, o_q);
  float* rq = region<float>(b, o_rho);
  int* filled = region<int>(b, o_filled);
  long long* total = region<long long>(b, o_total);
  int* surv = region<int>(b, o_surv);
  int* to_exact = region<int>(b, o_exact);
  long long* doff = region<long long>(b, o_off);
  unsigned long long* alt = region<unsigned long long>(b, o_alt);
  L.X = device_rows(ix);
  L.nq = m;
  L.C = C;
  L.mode = mode;
  L.qf = q;
  if (f) {
    L.allow = f->allow_bits;
    L.ex = Excluded{f->exclude_offsets, f->exclude_ids, dlist, 0, id_offset};
  }
  const bool exclude = L.ex.off != nullptr;
  OM_TRY(gather_listed(list, dlist, qf, d, q, st));
  gather_rows_kernel<<<grid_for(m, 256), 256, 0, st>>>(rho, dlist, m, 1, rq);
  OM_CUDA(cudaGetLastError());
  if (mode == 0) OM_TRY(convert_queries(ix, L, st));
  range_threshold_kernel<<<(m + 255) / 256, 256, 0, st>>>(rq, L.hn, L.en, ix->gstats, d, m, mode, L.thr, to_exact);
  OM_CUDA(cudaMemsetAsync(L.count, 0, M * 4, st));
  OM_CUDA(cudaMemsetAsync(filled, 0, M * 4, st));
  OM_CUDA(cudaMemsetAsync(total, 0, M * 8, st));
  OM_CUDA(cudaMemsetAsync(surv, 0, M * 4, st));
  OM_CUDA(cudaMemsetAsync(L.status, 0, 32, st));
  ix->st_launches += 4;
  // the sweep: one pass over the shard at the fixed thresholds, in rounds only to keep the column counts in an int
  for (int64_t pos = 0; pos < L.X.n; pos += kRangeRound) {
    OM_TRY(scan_round(ix, L, 0, m, pos, std::min(L.X.n - pos, kRangeRound), false, sms, st));
    range_fold_kernel<<<(m + 255) / 256, 256, 0, st>>>(L.count, filled, total, C, m);
    OM_CUDA(cudaGetLastError());
    ix->st_rounds++;
    ix->st_launches += 2;
  }
  {
    Timed t(ix, st, 2);
    with_rows(ix, L.X, [&](const auto* xs) {
      using RowT = std::decay_t<decltype(*xs)>;
      // at least 32 CTAs per query, more when few queries would leave SMs idle (a handful of long lists)
      const int gx = std::min((C + 63) / 64, std::max(32, (8 * sms + m - 1) / m));
      const auto kernel = exclude ? range_rescore_kernel<RowT, true> : range_rescore_kernel<RowT>;
      kernel<<<dim3(gx, m), 256, static_cast<size_t>(d) * 4 + (exclude ? kMaxExcluded * 4 : 0), st>>>(
          L.cand, L.count, total, C, q, xs, d, rq, surv, exclude ? L.ex : Excluded{});
    });
    int P = 2;
    while (P < std::min(C, kRangeSortKeys)) P <<= 1;
    range_sort_kernel<<<dim3((C + kRangeSortKeys - 1) / kRangeSortKeys, m), 512, static_cast<size_t>(P) * 8, st>>>(L.cand, L.count,
                                                                                                                  total, C);
    ix->st_launches += 2;
  }
  OM_CUDA(cudaGetLastError());
  unsigned long long *from = L.cand, *to = alt;
  int merges = 0;
  for (int w = kRangeSortKeys; w < C; w <<= 1, ++merges) {
    range_merge_kernel<<<dim3(std::min((C + 255) / 256, 4096), m), 256, 0, st>>>(from, to, L.count, total, C, w);
    std::swap(from, to);
    ix->st_launches += 1;
  }
  OM_CUDA(cudaGetLastError());
  r.total.resize(m);
  r.surv.resize(m);
  r.to_exact.resize(m);
  OM_CUDA(cudaMemcpyAsync(r.total.data(), total, M * 8, cudaMemcpyDeviceToHost, st));
  OM_CUDA(cudaMemcpyAsync(r.surv.data(), surv, M * 4, cudaMemcpyDeviceToHost, st));
  OM_CUDA(cudaMemcpyAsync(r.to_exact.data(), to_exact, M * 4, cudaMemcpyDeviceToHost, st));
  OM_CUDA(cudaStreamSynchronize(st));
  const unsigned int fault = read_clear_dev_fault();
  if (fault) return fail(OM_EFAULT, "scan kernel pipeline fault 0x%08x", fault);
  // the queries this sweep answered: their keys go to the store, in list order
  std::vector<long long> hoff(m, -1);
  int64_t add = 0;
  for (int i = 0; i < m; ++i) {
    if ((mode == 0 && r.to_exact[i]) || r.total[i] > C) continue;
    hoff[i] = *stored + add;
    src[list[i]] = hoff[i];
    cnt[list[i]] = r.surv[i];
    add += r.surv[i];
    ix->st_range_candidates += r.total[i];
  }
  if (add == 0) return 0;
  OM_TRY(grow_keep(ix->rkeys, static_cast<size_t>(*stored) * 8, static_cast<size_t>(*stored + add) * 8, st));
  OM_CUDA(cudaMemcpyAsync(doff, hoff.data(), M * 8, cudaMemcpyHostToDevice, st));
  range_emit_kernel<<<dim3(std::min((C + 255) / 256, 1024), m), 256, 0, st>>>(
      L.cand, alt, (merges & 1) ? kRangeSortKeys : INT_MAX, L.count, surv, doff, C, static_cast<unsigned long long*>(ix->rkeys.p));
  OM_CUDA(cudaGetLastError());
  ix->st_launches += 1;
  *stored += add;
  return 0;
}

// The range search on this shard: every query swept once with lists of range_list keys; the queries whose candidates
// overflowed their list are swept again in groups that fit the device, with lists sized from their counts (a re-sweep may
// run another scan kernel, whose stage scores can differ in the last bit: hence the head-room and a bounded number of
// attempts); queries without a finite certificate bound are swept by the exact scan.  cnt[g] rows above rho for query g
// end sorted at ix->rkeys + src[g]; *stored keys in all.  f: as for range_sweep, every sweep's.
int range_local(om_index* ix, const float* qf, const float* rho, int nq, const om_search_filter* f, int64_t id_offset,
                std::vector<int64_t>& src, std::vector<int64_t>& cnt, int64_t* stored, cudaStream_t st) {
  const int sms = device_sm_count();
  if (sms < 0) return sms;
  struct Job {
    std::vector<int> qs;
    int mode, C;
  };
  std::vector<Job> jobs;
  auto add_chunks = [&](const std::vector<int>& qs, int mode) {
    for (size_t i = 0; i < qs.size(); i += kQueryChunk)
      jobs.push_back({std::vector<int>(qs.begin() + i, qs.begin() + std::min(qs.size(), i + kQueryChunk)), mode, ix->range_list});
  };
  src.assign(nq, -1);
  cnt.assign(nq, 0);
  *stored = 0;
  std::vector<int> all(nq), tries(nq, 0);
  for (int i = 0; i < nq; ++i) all[i] = i;
  add_chunks(all, ix->exact_only ? 1 : 0);
  ix->st_exact = ix->exact_only ? nq : 0;
  for (size_t j = 0; j < jobs.size(); ++j) {
    const Job job = jobs[j];  // a copy: jobs grows below
    RangeSweep r;
    OM_TRY(range_sweep(ix, qf, rho, job.qs, job.mode, job.C, sms, f, id_offset, stored, src, cnt, r, st));
    std::vector<int> exact;
    std::vector<std::pair<long long, int>> over;  // (candidates, query)
    for (size_t i = 0; i < job.qs.size(); ++i) {
      if (job.mode == 0 && r.to_exact[i])
        exact.push_back(job.qs[i]);
      else if (r.total[i] > job.C)
        over.push_back({r.total[i], job.qs[i]});
    }
    ix->st_exact += static_cast<int64_t>(exact.size());
    add_chunks(exact, 1);
    if (over.empty()) continue;
    ix->st_range_resweeps += static_cast<int64_t>(over.size());
    std::sort(over.begin(), over.end(), std::greater<std::pair<long long, int>>());
    size_t free_b = 0, total_b = 0;
    OM_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const size_t budget = (free_b + ix->ws.bytes) / 2;
    for (size_t i = 0; i < over.size();) {
      // the group's lists: the longest count of the group (the first) + 1/8 + 1024 of head-room
      const long long cap = round_up(over[i].first + over[i].first / 8 + 1024, 256);
      if (cap > kRangeMaxList)
        return fail(OM_ENOMEM, "range search: query %d has %lld candidates; a list holds at most %d", over[i].second,
                    over[i].first, kRangeMaxList);
      const size_t per = static_cast<size_t>(cap) * 8 * (cap > kRangeSortKeys ? 2 : 1) + static_cast<size_t>(ix->d) * 8 + 256;
      Job g{{}, job.mode, static_cast<int>(cap)};
      do {
        if (++tries[over[i].second] > 3) return fail(OM_EFAULT, "range search: a candidate list did not converge (bug)");
        g.qs.push_back(over[i++].second);
      } while (i < over.size() && g.qs.size() < static_cast<size_t>(kQueryChunk) && (g.qs.size() + 1) * per <= budget);
      jobs.push_back(std::move(g));
    }
  }
  return 0;
}

// The whole range search, unsharded or this rank's part of a sharded one: argument rules (a NaN radius, fp16 / int8 rows
// holding inf or NaN) checked before anything is written, the shard's results, then with several ranks one all-gather of
// the per-query counts, one all-gather of every shard's sorted results (padded to the largest) and the merge.  The lims
// go to the caller, the results stay in the index (rout).  f: nullptr, or a checked filter with at least one part.
int range_impl(om_index* ix, om_comm* comm, const void* q, om_memkind q_kind, int nq, const float* radius, int64_t* lims,
               om_memkind out_kind, int64_t id_offset, const om_search_filter* f, cudaStream_t st) {
  NvtxRange nvtx("om.range_search");
  // the sharded entry runs the exchange at every world size, one rank included
  const bool sharded = comm != nullptr;
  const int W = sharded ? comm->world : 1;
  const int sms = device_sm_count();
  if (sms < 0) return sms;
  // What only long lists grow is returned when the call ends, however it ends: the level workspace beyond what it held
  // before and what a first sweep needs (re-sweeps, the exchange), and a key store beyond 64 MB.  Smaller scratch stays
  // for the next call; the results (rout) stay until the next search, range search, reset or destroy.
  struct Scratch {
    om_index* ix;
    size_t ws0;
    ~Scratch() {
      if (ix->rkeys.bytes > (size_t(64) << 20)) ix->rkeys.release();
      if (ix->ws.bytes > std::max(ws0, ix->r_keep_ws)) ix->ws.release();
    }
  } scratch{ix, ix->ws.bytes};
  ix->r_keep_ws = 0;
  ix->st_range_candidates = ix->st_range_resweeps = 0;
  Layout ows;
  const float *qf = nullptr, *rho = nullptr;
  OM_TRY(call_prologue(ix, comm, "om_index_range_search", q, q_kind, nq, radius, ows, &qf, &rho, st));

  std::vector<int64_t> src, cnt;
  int64_t stored = 0;
  int rc = range_local(ix, qf, rho, nq, f, id_offset, src, cnt, &stored, st);
  // Every rank takes the same decision after a step that can fail on one rank alone (a re-sweep, an allocation): the
  // largest error code of all ranks, through one all-reduce, before the next collective.
  auto agree = [&](int rc_local) -> int {
    if (!sharded) return rc_local;
    cudaGetLastError();
    fill_i32<<<1, 1, 0, st>>>(ix->scratch(), rc_local < 0 ? -rc_local : 0, 1);
    OM_TRY(read_decision(ix, comm, ix->scratch(), 1, kNcclMax, 0, st));
    if (rc_local == 0 && ix->h_status[0]) return fail(-ix->h_status[0], "om_index_range_search_sharded: another rank failed");
    return rc_local;
  };

  std::vector<long long> ll(nq + 1, 0);  // this shard's lims
  for (int i = 0; i < nq && rc == 0; ++i) ll[i + 1] = ll[i] + cnt[i];
  const size_t NQ1 = static_cast<size_t>(nq) + 1;
  std::vector<long long> plims, glims;  // every part's lims [W][nq + 1], the merged lims
  Layout lay;
  const size_t o_src = lay.add(nq * 8), o_ll = lay.add(NQ1 * 8), o_plims = lay.add(W * NQ1 * 8), o_glims = lay.add(NQ1 * 8),
               o_cnt = lay.add(nq * 8), o_all = lay.add(static_cast<size_t>(W) * nq * 8);
  if (rc == 0 && ix->ws.reserve(lay.bytes) != 0) {
    cudaGetLastError();
    rc = fail(OM_ENOMEM, "range search: cannot allocate the lims of %d queries", nq);
  }
  OM_TRY(agree(rc));
  void* b = ix->ws.p;
  const unsigned long long* keys = static_cast<const unsigned long long*>(ix->rkeys.p);
  auto outputs = [&](int64_t T, float** D, int64_t** I) -> int {
    if (ix->rout.reserve(round_up(T * 4, 256) + T * 8 + 256) != 0) {
      cudaGetLastError();
      return fail(OM_ENOMEM, "range search: cannot allocate %lld results", (long long)T);
    }
    *D = static_cast<float*>(ix->rout.p);
    *I = reinterpret_cast<int64_t*>(static_cast<uint8_t*>(ix->rout.p) + round_up(T * 4, 256));
    return 0;
  };
  // this shard's results in query order: one CTA row per query, enough CTAs per query to fill the device when few
  // queries hold long lists
  const long long cmax = nq > 0 ? *std::max_element(cnt.begin(), cnt.end()) : 0;
  const dim3 gather_grid(static_cast<unsigned>(nq),
                         static_cast<unsigned>(std::max<long long>(1, std::min<long long>({(cmax + 255) / 256,
                                                                                          (8LL * sms + nq - 1) / nq, 65535}))));
  auto gather = [&](float* D, int64_t* I) -> int {
    OM_CUDA(cudaMemcpyAsync(region<long long>(b, o_src), src.data(), nq * 8, cudaMemcpyHostToDevice, st));
    OM_CUDA(cudaMemcpyAsync(region<long long>(b, o_ll), ll.data(), NQ1 * 8, cudaMemcpyHostToDevice, st));
    if (cmax > 0)
      range_gather_kernel<<<gather_grid, 256, 0, st>>>(keys, region<long long>(b, o_src),
                                                       region<long long>(b, o_ll), id_offset, D, I);
    OM_CUDA(cudaGetLastError());
    ix->st_launches += 1;
    return 0;
  };
  int64_t T = ll[nq];
  if (!sharded) {
    float* D;
    int64_t* I;
    OM_TRY(outputs(T, &D, &I));
    OM_TRY(gather(D, I));
    glims = ll;
  } else {
    NcclApi& nc = nccl_api();
    Timed t(ix, st, 3);
    // counts of every shard
    OM_CUDA(cudaMemcpyAsync(region<long long>(b, o_cnt), cnt.data(), nq * 8, cudaMemcpyHostToDevice, st));
    OM_NCCL(nc.AllGather(region<long long>(b, o_cnt), region<long long>(b, o_all), static_cast<size_t>(nq) * 8, kNcclInt8, comm->nccl, st));
    std::vector<long long> all(static_cast<size_t>(W) * nq);
    OM_CUDA(cudaMemcpyAsync(all.data(), region<long long>(b, o_all), all.size() * 8, cudaMemcpyDeviceToHost, st));
    OM_CUDA(cudaStreamSynchronize(st));
    plims.assign(W * NQ1, 0);
    glims.assign(NQ1, 0);
    long long tmax = 0;
    for (int p = 0; p < W; ++p) {
      for (int i = 0; i < nq; ++i) plims[p * NQ1 + i + 1] = plims[p * NQ1 + i] + all[static_cast<size_t>(p) * nq + i];
      tmax = std::max(tmax, plims[p * NQ1 + nq]);
    }
    for (int i = 0; i < nq; ++i) {
      long long c = 0;
      for (int p = 0; p < W; ++p) c += all[static_cast<size_t>(p) * nq + i];
      glims[i + 1] = glims[i] + c;
    }
    T = glims[nq];
    // every shard's sorted results, padded to the longest: [D f32 tmax | I i64 tmax], and the merged results; both
    // allocated, and the outcome agreed, before the results' all-gather
    const size_t o_i = round_up(tmax * 4, 256), blk = o_i + round_up(tmax * 8, 256) + 256;
    const size_t o_send = lay.add(blk), o_recv = lay.add(blk * W);
    float* D = nullptr;
    int64_t* I = nullptr;
    int rc2 = 0;
    if (ix->ws.reserve(lay.bytes) != 0) {
      cudaGetLastError();
      rc2 = fail(OM_ENOMEM, "range search: cannot allocate the exchange of %lld results per shard", tmax);
    }
    if (rc2 == 0) rc2 = outputs(T, &D, &I);
    OM_TRY(agree(rc2));
    b = ix->ws.p;  // possibly a new buffer: the uploads above were read by the all-gather already
    OM_CUDA(cudaMemcpyAsync(region<long long>(b, o_plims), plims.data(), W * NQ1 * 8, cudaMemcpyHostToDevice, st));
    OM_CUDA(cudaMemcpyAsync(region<long long>(b, o_glims), glims.data(), NQ1 * 8, cudaMemcpyHostToDevice, st));
    OM_TRY(gather(region<float>(b, o_send), region<int64_t>(b, o_send + o_i)));
    OM_NCCL(nc.AllGather(region<uint8_t>(b, o_send), region<uint8_t>(b, o_recv), blk, kNcclInt8, comm->nccl, st));
    if (tmax > 0)
      range_merge_parts_kernel<<<dim3(static_cast<unsigned>(std::min<long long>((tmax + 255) / 256, 4096)), W), 256, 0, st>>>(
          region<const float>(b, o_recv), region<const int64_t>(b, o_recv + o_i),
          static_cast<int64_t>(blk / 4), static_cast<int64_t>(blk / 8), region<const long long>(b, o_plims), W, nq,
          region<const long long>(b, o_glims), D, I);
    OM_CUDA(cudaGetLastError());
    ix->st_launches += 3;
  }
  if (out_kind == OM_HOST)
    memcpy(lims, glims.data(), NQ1 * 8);
  else
    OM_CUDA(cudaMemcpyAsync(lims, glims.data(), NQ1 * 8, cudaMemcpyHostToDevice, st));
  OM_CUDA(cudaStreamSynchronize(st));
  if (ix->profile) collect_profile(ix);
  ix->r_total = T;
  return 0;
}

// The eight exported searches: a top-k search or a range search (range), sharded (the entries that take a
// communicator, required) or not, filtered (the _filtered entries) or not.  The filter is checked before the search when
// it has a part and, through a sharded filtered entry with more than one rank, always: every rank checks the filters
// together (one all-reduce), also a rank whose filter is null or empty, so the ranks' collectives stay in step when only
// some pass a filter.  Any other call is the unfiltered search, and its messages name the unfiltered entry.  What differs
// by kind: a top-k search refuses a host-resident index only as a shard, before the communicator is read, needs k > 0,
// ends the last range search's results and drops a one-rank communicator (no collective); a range search refuses a
// host-resident index always, needs lims and the radii, writes lims = {0} for nq = 0 and keeps its collectives at every
// world size.
int search_entry(bool range, bool sharded, bool filtered, om_index* ix, om_comm* comm, const void* q, om_memkind q_kind,
                 int nq, int k, float* D, int64_t* I, const float* radius, int64_t* lims, om_memkind out_kind,
                 int64_t id_offset, const om_search_filter* filter, void* stream) {
  static const char* const kNames[2][2][2] = {  // [range][sharded][filtered]
      {{"om_index_search", "om_index_search_filtered"}, {"om_index_search_sharded", "om_index_search_sharded_filtered"}},
      {{"om_index_range_search", "om_index_range_search_filtered"},
       {"om_index_range_search_sharded", "om_index_range_search_sharded_filtered"}}};
  if (!range && sharded && ix && ix->window)  // refused before the communicator is read
    return fail(OM_EINVAL, "%s: a host-resident index cannot be a shard of a sharded search", kNames[0][1][filtered]);
  const bool local = filter && (filter->allow_bits || filter->exclude_offsets);
  const bool check = local || (filtered && comm && comm->world > 1);
  const char* who = kNames[range][sharded][check];
  const bool bad = range ? !lims || (nq > 0 && (!q || !radius)) : k <= 0 || (nq > 0 && (!q || !D || !I));
  if (!ix || (sharded && !comm) || nq < 0 || bad)
    return range ? fail(OM_EINVAL, "%s: bad arguments (nq=%d)", who, nq)
                 : fail(OM_EINVAL, "%s: bad arguments (nq=%d k=%d)", who, nq, k);
  if (range && ix->window) return fail(OM_EINVAL, "%s: range search is not available on a host-resident index", who);
  ix->r_total = -1;  // the last range search's results end here
  if (!range) {      // a search frees their buffer too; a range search reuses it
    ix->rout.release();
    if (nq == 0) return 0;
  }
  OM_TRY(device_sm_count());
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (nq == 0) {  // a range search: lims = {0}, no results
    if (out_kind == OM_HOST) {
      lims[0] = 0;
    } else {
      OM_CUDA(cudaMemsetAsync(lims, 0, 8, st));
      OM_CUDA(cudaStreamSynchronize(st));
    }
    ix->r_total = 0;
    return 0;
  }
  OM_TRY(settle_reset(ix, st));
  if (!range && comm && comm->world == 1) comm = nullptr;  // one rank: no collective, the single-shard search
  if (check) OM_TRY(check_filter(ix, comm, filter, nq, st));
  const om_search_filter* f = local ? filter : nullptr;
  return range ? range_impl(ix, comm, q, q_kind, nq, radius, lims, out_kind, id_offset, f, st)
               : search_impl(ix, comm, q, q_kind, nq, k, D, I, out_kind, id_offset, f, st);
}

}  // namespace

extern "C" int om_index_range_search(om_index* ix, const void* q, om_memkind q_kind, int nq, const float* radius,
                                     int64_t* lims, om_memkind out_kind, int64_t id_offset, void* stream) {
  return search_entry(true, false, false, ix, nullptr, q, q_kind, nq, 0, nullptr, nullptr, radius, lims, out_kind, id_offset,
                      nullptr, stream);
}

extern "C" int om_index_range_search_filtered(om_index* ix, const void* q, om_memkind q_kind, int nq, const float* radius,
                                              int64_t* lims, om_memkind out_kind, int64_t id_offset,
                                              const om_search_filter* filter, void* stream) {
  return search_entry(true, false, true, ix, nullptr, q, q_kind, nq, 0, nullptr, nullptr, radius, lims, out_kind, id_offset,
                      filter, stream);
}

extern "C" int om_index_range_search_sharded(om_index* ix, om_comm* comm, const void* q, om_memkind q_kind, int nq,
                                             const float* radius, int64_t* lims, om_memkind out_kind, int64_t id_offset,
                                             void* stream) {
  return search_entry(true, true, false, ix, comm, q, q_kind, nq, 0, nullptr, nullptr, radius, lims, out_kind, id_offset,
                      nullptr, stream);
}

extern "C" int om_index_range_search_sharded_filtered(om_index* ix, om_comm* comm, const void* q, om_memkind q_kind, int nq,
                                                      const float* radius, int64_t* lims, om_memkind out_kind,
                                                      int64_t id_offset, const om_search_filter* filter, void* stream) {
  return search_entry(true, true, true, ix, comm, q, q_kind, nq, 0, nullptr, nullptr, radius, lims, out_kind, id_offset,
                      filter, stream);
}

extern "C" int om_index_range_results(const om_index* ix, float* D, int64_t* I, om_memkind out_kind, void* stream) {
  if (!ix) return fail(OM_EINVAL, "om_index_range_results: null index");
  if (ix->r_total < 0) return fail(OM_ESTATE, "om_index_range_results: no range search result on this index");
  const int64_t T = ix->r_total;
  if (T == 0) return 0;
  if (!D || !I) return fail(OM_EINVAL, "om_index_range_results: null output");
  OM_TRY(device_sm_count());
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const cudaMemcpyKind kind = out_kind == OM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  const uint8_t* p = static_cast<const uint8_t*>(ix->rout.p);
  OM_CUDA(cudaMemcpyAsync(D, p, T * 4, kind, st));
  OM_CUDA(cudaMemcpyAsync(I, p + round_up(T * 4, 256), T * 8, kind, st));
  OM_CUDA(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int om_index_search(om_index* ix, const void* q, om_memkind q_kind, int nq, int k, float* D, int64_t* I,
                               om_memkind out_kind, int64_t id_offset, void* stream) {
  return search_entry(false, false, false, ix, nullptr, q, q_kind, nq, k, D, I, nullptr, nullptr, out_kind, id_offset,
                      nullptr, stream);
}

extern "C" int om_index_search_filtered(om_index* ix, const void* q, om_memkind q_kind, int nq, int k, float* D,
                                        int64_t* I, om_memkind out_kind, int64_t id_offset, const om_search_filter* filter,
                                        void* stream) {
  return search_entry(false, false, true, ix, nullptr, q, q_kind, nq, k, D, I, nullptr, nullptr, out_kind, id_offset,
                      filter, stream);
}

// ---- row-sharded search with the exchange inside the library (NCCL over NVLink) -----------------------------------
extern "C" int om_comm_unique_id(char* out128) {
  if (!out128) return fail(OM_EINVAL, "om_comm_unique_id: null buffer");
  NcclApi& nc = nccl_api();
  if (!nc.handle) return fail(OM_ESTATE, "NCCL unavailable: %s", nc.why ? nc.why : "?");
  NcclUid id;
  OM_NCCL(nc.GetUniqueId(&id));
  memcpy(out128, id.internal, 128);
  return 0;
}

extern "C" int om_comm_init(const char* unique_id, int rank, int world, om_comm** out) {
  if (!unique_id || !out || world <= 0 || rank < 0 || rank >= world) return fail(OM_EINVAL, "om_comm_init: bad arguments");
  OM_TRY(device_sm_count());
  NcclApi& nc = nccl_api();
  if (!nc.handle) return fail(OM_ESTATE, "NCCL unavailable: %s", nc.why ? nc.why : "?");
  om_comm* c = new (std::nothrow) om_comm();
  if (!c) return fail(OM_ENOMEM, "om_comm_init: out of host memory");
  c->rank = rank;
  c->world = world;
  NcclUid id;
  memcpy(id.internal, unique_id, 128);
  const int r = nc.CommInitRank(&c->nccl, world, id, rank);
  if (r != 0) {
    delete c;
    return fail(OM_ECUDA, "ncclCommInitRank failed: %s", nc.GetErrorString(r));
  }
  *out = c;
  return 0;
}

extern "C" void om_comm_destroy(om_comm* c) {
  if (!c) return;
  if (c->nccl) nccl_api().CommDestroy(c->nccl);
  delete c;
}

extern "C" int om_index_search_sharded(om_index* ix, om_comm* comm, const void* q, om_memkind q_kind, int nq, int k,
                                       float* D, int64_t* I, om_memkind out_kind, int64_t id_offset, void* stream) {
  return search_entry(false, true, false, ix, comm, q, q_kind, nq, k, D, I, nullptr, nullptr, out_kind, id_offset,
                      nullptr, stream);
}

extern "C" int om_index_search_sharded_filtered(om_index* ix, om_comm* comm, const void* q, om_memkind q_kind, int nq,
                                                int k, float* D, int64_t* I, om_memkind out_kind, int64_t id_offset,
                                                const om_search_filter* filter, void* stream) {
  return search_entry(false, true, true, ix, comm, q, q_kind, nq, k, D, I, nullptr, nullptr, out_kind, id_offset,
                      filter, stream);
}

extern "C" int om_topk_merge_n(const float* D_parts, const int64_t* I_parts, int nparts, int nq, int k_in, int k_out,
                               float* D, int64_t* I, void* stream) {
  if (nparts <= 0 || nq < 0 || k_in <= 0 || k_out <= 0 || !D_parts || !I_parts || !D || !I)
    return fail(OM_EINVAL, "om_topk_merge_n: bad arguments");
  if (nq == 0) return 0;
  OM_TRY(device_sm_count());
  const int64_t stride = static_cast<int64_t>(nq) * k_in;
  return merge_parts(D_parts, I_parts, stride, stride, nparts, nq, k_in, k_out, D, I, static_cast<cudaStream_t>(stream));
}
