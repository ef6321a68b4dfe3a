// Shared-memory staging for the HBM-bound elementwise / reduction kernels.
//
// A plain "load a few 16-byte vectors, compute, store" loop keeps only (resident threads x loads in
// flight x 16 B) bytes in flight per SM, and the per-(image, channel) coefficient registers of the
// SK kernels cap the residency at 512 threads: ~64 KiB in flight, gone to zero between trips, far
// from what HBM needs.  Here one thread per CTA streams the operand rows of the
// next trips into a ring of shared-memory stages with bulk asynchronous copies (cp.async.bulk,
// completion on an mbarrier) while all threads compute on the current stage: the bytes in flight are
// (stages - 1) x stage size x resident CTAs (~100-150 KiB per SM), independent of register use.
#pragma once
#include "ptx.cuh"

namespace acnn {

// global -> shared bulk copy of `bytes` (multiple of 16, both addresses 16-byte aligned)
__device__ __forceinline__ void bulk_load(uint32_t smem_dst, const void* gsrc, uint32_t bytes,
                                          uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::
          "r"(smem_dst),
      "l"(gsrc), "r"(bytes), "r"(bar)
      : "memory");
}

// Ring of kStages stages; every trip of the CTA consumes one stage.  Usage:
//   RowPipe<S> pipe(bars);  pipe.init();           (all threads; contains a __syncthreads)
//   pipe.prologue(trips, issue);                    (issue(trip, stage, bar) called by thread 0)
//   for t: pipe.acquire(t, trips, issue); ...compute on stage pipe.stage(t)...; pipe.release();
template <int kStages>
struct RowPipe {
  uint32_t bar0;   // shared-window address of the first of kStages mbarriers

  __device__ __forceinline__ explicit RowPipe(uint64_t* bars) : bar0(smem_u32(bars)) {}

  __device__ __forceinline__ void init(uint64_t* bars) {
    if (threadIdx.x == 0) {
      for (int s = 0; s < kStages; ++s) mbar_init(&bars[s], 1);
      fence_barrier_init();
    }
    __syncthreads();
  }
  template <class Issue>
  __device__ __forceinline__ void prologue(int trips, Issue issue) {
    if (threadIdx.x == 0) {
      const int n = trips < kStages - 1 ? trips : kStages - 1;
      for (int t = 0; t < n; ++t) issue(t, t % kStages, bar0 + (t % kStages) * 8);
    }
  }
  // start the copy of trip t + kStages - 1 (its stage was released at the end of trip t - 1), then
  // wait for the data of trip t
  template <class Issue>
  __device__ __forceinline__ void acquire(int t, int trips, Issue issue) {
    const int ahead = t + kStages - 1;
    if (threadIdx.x == 0 && ahead < trips) issue(ahead, ahead % kStages, bar0 + (ahead % kStages) * 8);
    mbar_wait_a(bar0 + (t % kStages) * 8, (t / kStages) & 1);
  }
  __device__ __forceinline__ int stage(int t) const { return t % kStages; }
  // all threads are done reading the stage of this trip
  __device__ __forceinline__ void release() { __syncthreads(); }
};

}  // namespace acnn
