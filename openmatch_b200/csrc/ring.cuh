// The shared-memory ring of the TMA -> wgmma pipelines (GEMM core, wide search scan, fused loss): STAGES slots, each
// with a full barrier (one arrival: the producer's expect_tx, completed by the TMA bytes) and an empty barrier (one
// arrival per consumer warp that reads the slot).  Producer and consumers walk the slots in the same order and keep
// their own Ring position.
//
// A consumer keeps one wgmma group in flight: the slot of k block kb is released once the group of k block kb + 1 has
// been issued and the group of kb has completed (wgmma_wait<1>), so each slot is released one group late.
//
// What stays with each kernel: which TMA loads fill a slot, which wgmma instructions consume it, what releasing it
// means (one local arrive, or also remote arrives to the cluster peers that fill it), the accumulators and the
// fault-site codes of its waits.
#pragma once
#include "ptx.cuh"

namespace om {

// Per-thread position in a ring of STAGES slots.
template <int STAGES>
struct Ring {
  uint32_t stage = 0, phase = 0;
  __device__ __forceinline__ void advance() {
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1u;
    }
  }
};

// One thread initialises the barriers of a ring; the caller fences and synchronises before first use.
__device__ __forceinline__ void ring_init(uint64_t* full, uint64_t* empty, int stages, uint32_t empty_arrivals) {
  for (int i = 0; i < stages; ++i) {
    mbar_init(&full[i], 1);
    mbar_init(&empty[i], empty_arrivals);
  }
}

// Producer: wait until slot r.stage has been released by every consumer of its previous fill.
template <int STAGES>
__device__ __forceinline__ void ring_wait_free(uint64_t* empty, const Ring<STAGES>& r, uint32_t site) {
  mbar_wait(&empty[r.stage], r.phase ^ 1u, site);
}

// Producer of a TMA slot: wait until it is free and arm its full barrier for `bytes`.  Returns that barrier; the caller
// issues the loads that complete it into slot r.stage and then advances r.
template <int STAGES>
__device__ __forceinline__ uint64_t* ring_acquire_tx(uint64_t* full, uint64_t* empty, const Ring<STAGES>& r,
                                                     uint32_t bytes, uint32_t site) {
  ring_wait_free(empty, r, site);
  mbar_arrive_expect_tx(&full[r.stage], bytes);
  return &full[r.stage];
}

// Consumer warp of a warpgroup: k blocks [kb_begin, kb_end), one per slot.  issue(stage, accumulate) issues the
// wgmma instructions of a k block (accumulate == 0 for the first: it overwrites the accumulators); release(stage)
// releases a slot.  Returns with every wgmma group complete and every consumed slot released; the caller then fences
// its accumulator registers (wgmma_fence_regs).
template <int STAGES, class Issue, class Release>
__device__ __forceinline__ void ring_consume(uint64_t* full, Ring<STAGES>& r, int kb_begin, int kb_end, uint32_t site,
                                             Issue&& issue, Release&& release) {
  uint32_t prev_stage = 0;
  for (int kb = kb_begin; kb < kb_end; ++kb) {
    mbar_wait_warp(&full[r.stage], r.phase, site);
    wgmma_fence();
    issue(r.stage, kb != kb_begin ? 1u : 0u);
    wgmma_commit();
    if (kb != kb_begin) {
      wgmma_wait<1>();
      release(prev_stage);
    }
    prev_stage = r.stage;
    r.advance();
  }
  wgmma_wait<0>();
  if (kb_end > kb_begin) release(prev_stage);
}

}  // namespace om
