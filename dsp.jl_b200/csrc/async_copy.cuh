// dspb200 -- TMA bulk (1-D) global -> shared copies completed through an mbarrier, and per-thread cp.async copies (sm_90a
// PTX).  SASS: UBLKCP (cp.async.bulk), SYNCS.ARRIVE.TRANS64 (expect_tx), SYNCS.PHASECHK.TRANS64.TRYWAIT (try_wait), LDGSTS.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dspb200 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// make the barrier initialisation visible to the async proxy (TMA) before the first copy is issued
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// expect `bytes` more in the current phase without arriving: a phase fed by several copies issued at different times
// posts this for all but the last one, then mbar_expect_tx
__device__ __forceinline__ void mbar_expect_tx_noarrive(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.expect_tx.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

// order the CTA's earlier generic-proxy accesses of shared memory (made visible to this thread by a barrier) before the
// async-proxy writes of a bulk copy issued after it: a buffer that was just read can be refilled by TMA
__device__ __forceinline__ void fence_proxy_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// one elected thread: bytes must be a multiple of 16, src and dst 16-byte aligned
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// L2 prefetch of a contiguous global range (no shared-memory destination): bytes multiple of 16, src 16-byte aligned
__device__ __forceinline__ void tma_prefetch_l2(const void* gmem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes) : "memory");
}

// Per-thread asynchronous copies (cp.async, LDGSTS) of one naturally aligned 8- or 16-byte element: for staging tiles whose
// rows start at any element, where a bulk copy's 16-byte alignment does not hold.  cp_async_commit closes the calling
// thread's group of copies; cp_async_wait<N> waits until at most N of its groups are still in flight.
template <int BYTES> __device__ __forceinline__ void cp_async(void* smem_dst, const void* gmem_src) {
    static_assert(BYTES == 8 || BYTES == 16, "cp.async.ca copies 4, 8 or 16 bytes");
    asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity)
        : "memory");
}

}  // namespace dspb200
