// One-shot all-reduce of a small fp64 vector over NVLink peer memory — the statistics exchange
// of synchronised batch norm (reference: torch.nn.SyncBatchNorm behind
// MinkowskiEngine/MinkowskiNormalization.py:101-192; NCCL all-reduce per layer there).
//
// A SyncBN exchange moves 2C+1 doubles (<= 4 KB) per layer, forward and backward: ~140 latency-
// bound NCCL launches per MinkUNet34C step, each with two cross-stream hand-offs (a visible
// share of a 2-GPU step).  Here every rank keeps a buffer in
// symmetric memory (same layout on every GPU, peers' base pointers known); the LAST CTA of the
// batch-norm reduction (csrc/batchnorm.cu, BnTail)
//   1. publishes "my slot for call #seq is complete" by storing seq into each peer's flag word
//      for this rank (st.release.sys after a system-scope fence),
//   2. spins until every peer has published seq in this rank's flag words (ld.acquire.sys),
//   3. sums the ranks' slots in rank order with system-scope loads — every rank adds the same
//      numbers in the same order, so all ranks hold bitwise identical totals.
// Slots rotate (kPeerSlots): a rank can run at most one call ahead of the slowest peer (it needs
// that peer's flag for the call it is in), so a slot is never overwritten while still being read.
//
// Buffer layout, identical on every rank (all offsets in bytes from the symmetric base):
//   [0, 1024)                     flags: uint32 flag[r] = last call for which rank r's slot is ready
//   1024 + s * slot_bytes         slot s, s in [0, kPeerSlots)
// (Round 2 first ran this as a separate single-CTA kernel per exchange; fused into the reduction
// it costs no launch at all.)
#pragma once
#include "common.cuh"

namespace meb200 {

__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ double ld_relaxed_sys_f64(const double *p) {
  double v;
  asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
constexpr uint64_t kPeerTimeoutNs = 30ull * 1000 * 1000 * 1000;   // 30 s


// Publish "my slot for call #seq is complete" to every peer and wait for theirs.  Called by ALL
// threads of one CTA (blockDim.x >= world) after they have written the slot.
__device__ __forceinline__ void peer_publish_and_wait(uint8_t *const *bases, uint32_t seq,
                                                      uint32_t rank, uint32_t world) {
  __threadfence_system();
  __syncthreads();
  const uint32_t tid = threadIdx.x;
  if (tid < world) {
    st_release_sys(reinterpret_cast<uint32_t *>(bases[tid]) + rank, seq);       // tell peer `tid`
    const uint32_t *mine = reinterpret_cast<const uint32_t *>(bases[rank]) + tid;
    const uint64_t t0 = globaltimer_ns();
    while ((int32_t)(ld_acquire_sys(mine) - seq) < 0) {                         // hear from it
      __nanosleep(100);
      // a peer that died or skipped the call must not hang this GPU for ever: fail loudly
      if (globaltimer_ns() - t0 > kPeerTimeoutNs) __trap();
    }
  }
  __syncthreads();
}

}  // namespace meb200
