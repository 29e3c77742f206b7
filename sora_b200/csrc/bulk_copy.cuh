// sora_b200 — the PTX of the 1-D bulk asynchronous copy (cp.async.bulk, the TMA unit: SASS UBLKCP) global -> shared memory and of the
// mbarrier it completes on (sm_90a).  A copy is: one thread initialises the barrier (arrival count 1), arms it with the bytes to come and
// issues the copies; every waiting thread spins on the barrier's phase.  Copy sources, destinations and sizes are 16-byte multiples.
// Shared memory goes by its 32-bit shared-window address (smem_addr), as the instructions take it, so that the caller decides where a
// barrier's address is computed: converting a generic pointer inside each wrapper changed the code ptxas made for k_channel_sim and
// k_combine.
#pragma once
#include <cstdint>

namespace sb {

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// n consecutive barriers from bar, each with an arrival count of 1, made visible to the copy engine
__device__ __forceinline__ void mbar_init(uint32_t bar, int n = 1) {
#pragma unroll
    for (int i = 0; i < n; i++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bar + 8u * i));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// the one arrival of the barrier's current phase, which also makes the phase wait for `bytes` bytes of copies
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}

// `bytes` bytes from global src to shared dst, counted against the barrier's expected bytes as they land
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// returns once the barrier's phase of the given parity (0 for its first phase) has completed
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok = 0;
    while (!ok) asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
}

} // namespace sb
