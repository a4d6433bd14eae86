// 1-D TMA bulk copies from global into shared memory, completed through mbarriers (sm_90).
// K1 stages its PCM tiles and K2 its column ring with these; the protocol per buffer is
//   mbar_init (once, one thread) -> bulk_copy_g2s (one thread) -> mbar_wait (every consumer)
// with the barrier's phase parity flipping on every completed copy.
#pragma once

#include <stdint.h>

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// N consecutive barriers, each completed by one arrival (the issuing thread's expect_tx) plus
// the copy's bytes.  One thread calls this; a CTA or warp barrier must follow before any other
// thread waits on them.
template <int N>
__device__ __forceinline__ void mbar_init(unsigned long long* bar) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bar + i)));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// Copy `bytes` (a multiple of 16; both addresses 16-byte aligned) from src to dst; completes
// the current phase of `bar`.  One thread issues it.
__device__ __forceinline__ void bulk_copy_g2s(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
  // order earlier generic-proxy accesses of this buffer before the async-proxy write
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// Spin until the phase of `bar` with the given parity has completed.
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
}
