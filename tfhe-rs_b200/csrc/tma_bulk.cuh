// tma_bulk.cuh -- 1-D bulk asynchronous copies global -> shared memory through
// the TMA unit (cp.async.bulk, SASS UBLKCP) with mbarrier completion.
//
// Used where a CTA streams a contiguous, per-step block of key material that
// it can request a whole step ahead: the per-sample key bundle of the
// low-latency multi-bit kernel and (optionally) the Fourier key block of the
// classic kernel at one CTA per SM.  One elected thread arms the mbarrier with
// the byte count and issues the copies; every consumer thread waits on the
// barrier's phase parity before reading the ring slot.  Reuse of a slot (WAR:
// generic-proxy reads, then an async-proxy write) is ordered by the CTA
// barrier that separates the consumers' last read from the producer's next
// issue.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace b200 {

__device__ __forceinline__ uint32_t smem_addr_u32(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(unsigned long long *bar,
                                          uint32_t arrivals) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(
                   smem_addr_u32(bar)),
               "r"(arrivals)
               : "memory");
}
// make the initialised barriers visible to the async proxy
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long *bar,
                                                      uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(
                   smem_addr_u32(bar)),
               "r"(bytes)
               : "memory");
}
// plain arrival (consumer release of a ring slot)
__device__ __forceinline__ void mbar_arrive(unsigned long long *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(
                   smem_addr_u32(bar))
               : "memory");
}
// consumer release of a ring slot that this thread has read with plain loads,
// arriving on the slot's barrier itself: the next async-proxy (TMA) write into
// the slot must not overtake those reads.  The proxy fence makes the thread's
// shared-memory reads complete first (MEMBAR.CTA + FENCE.VIEW.ASYNC.S); a bare
// arrive may issue while the loads are still in flight.
__device__ __forceinline__ void mbar_arrive_after_reads(unsigned long long *bar) {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  mbar_arrive(bar);
}
__device__ __forceinline__ void mbar_wait_parity(unsigned long long *bar,
                                                 uint32_t parity) {
  asm volatile("{\n\t"
               ".reg .pred p;\n\t"
               "MBAR_WAIT_%=:\n\t"
               "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
               "@p bra MBAR_DONE_%=;\n\t"
               "bra MBAR_WAIT_%=;\n\t"
               "MBAR_DONE_%=:\n\t"
               "}" ::"r"(smem_addr_u32(bar)),
               "r"(parity)
               : "memory");
}
// bytes: multiple of 16; both addresses 16-byte aligned
__device__ __forceinline__ void tma_bulk_g2s(void *smem_dst,
                                             const void *gmem_src,
                                             uint32_t bytes,
                                             unsigned long long *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::"
               "bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_addr_u32(bar))
               : "memory");
}

} // namespace b200
