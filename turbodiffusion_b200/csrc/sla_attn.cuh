// Shared by the SLA attention kernels (sla_attn.cu, sla_attn_bwd.cu): the release of a ring slot, and the entry-split
// schedule of the 64-row-query-block kernels with the hand-off between their two consumer warpgroups.
//
// Entry split.  CTA = a producer warpgroup (one warp issues the TMA loads; setmaxnreg gives its registers to the consumers) and
// two consumer warpgroups on the same 64 query rows, which take alternate LUT entries: warpgroup g consumes entries j = g mod 2,
// while the producer streams every entry through one K ring and one V ring of kStages slots.
// Ring slot st serves entries st, st + 3, st + 6, ..., which alternate between the two warpgroups.  One full barrier per slot
// would let a warpgroup skip a phase (the other warpgroup's entry), and try_wait.parity cannot tell phase n from phase n - 2, so
// the wait could pass while the skipped entry's load is still landing.  Each slot therefore has one full barrier per warpgroup:
// entry j completes phase j / 6 of barrier (j % 3, j % 2), and warpgroup j % 2 consumes that barrier's phases in order.  The
// empty barriers stay per slot: the producer waits on every phase in order, and the four warps of the entry's warpgroup arrive
// only after its load, i.e. after the previous phase completed.
#pragma once
#include "common.cuh"

namespace tdb {

// the calling warp is done reading a ring slot: one arrival on the slot's empty barrier, after every lane's reads
__device__ __forceinline__ void warp_release(uint64_t* empty, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(empty);
}

namespace split {
constexpr int kThreads = 3 * 128;
constexpr uint32_t kProducerRegs = 40, kConsumerRegs = 232;   // 128 * 40 + 256 * 232 <= 65536
constexpr int kStages = 3;
// the resident tiles' barrier, then per ring the full barriers [slot][warpgroup] and the empty barriers [slot]
enum Bar { kQFull = 0, kKFull = 1 /*3 x 2*/, kKEmpty = 7 /*3*/, kVFull = 10 /*3 x 2*/, kVEmpty = 16 /*3*/, kNumBars = 19 };

// the full barrier of entry j in the ring whose full barriers start at `base`, and the phase the consumer waits for
__device__ __forceinline__ int full(int base, int j) { return base + 2 * (j % kStages) + (j & 1); }
__device__ __forceinline__ uint32_t full_phase(int j) { return (j / (2 * kStages)) & 1; }

__device__ __forceinline__ void init_barriers(uint64_t* bars) {
  mbar_init(&bars[kQFull], 1);
  for (int i = 0; i < kStages; ++i) {  // each use of a ring slot is consumed by the four warps of one warpgroup
    for (int g = 0; g < 2; ++g) {
      mbar_init(&bars[kKFull + 2 * i + g], 1);
      mbar_init(&bars[kVFull + 2 * i + g], 1);
    }
    mbar_init(&bars[kKEmpty + i], 4);
    mbar_init(&bars[kVEmpty + i], 4);
  }
  mbar_fence_init();
}
}  // namespace split

// Hand-off from consumer warpgroup 1 to consumer warpgroup 0 once both have drained the ring, so that `ring` (shared memory the
// ring's tiles occupied) is free.  Thread t of warpgroup 1 stores value v at x[v], which is float v * 128 + t: thread t of
// warpgroup 0 holds the same fragment positions, and the [value][thread] layout is conflict-free.  `put` runs on warpgroup 1
// only; after the call warpgroup 1 is done and warpgroup 0 reads x[v].  `bar` is a named barrier the kernel uses for nothing else.
struct Handoff {
  float* base;
  __device__ __forceinline__ float& operator[](int v) const { return base[v * 128]; }
};
template <typename Put>
__device__ __forceinline__ Handoff handoff_wg1_to_wg0(uint8_t* ring, int wg, uint32_t bar, Put&& put) {
  const Handoff x{reinterpret_cast<float*>(ring) + (threadIdx.x & 127)};
  named_bar_sync(bar, 256);
  if (wg == 1) put(x);
  named_bar_sync(bar, 256);
  return x;
}

}  // namespace tdb
