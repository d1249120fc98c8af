// seaweedfs_b200/csrc/tma_fetch.cuh — one TMA bulk copy of a table from global into a CTA's shared memory, for the
// table-driven kernels (swec_table_kernel in kernels.cu, needle_crc_kernel in needles.cu).
// Not part of device_common.cuh: that file is the NVRTC prelude and keys the on-disk cubin cache.
#pragma once
#include "apply_params.h"

__device__ __forceinline__ u32 smem_u32(const void* p) { return (u32)__cvta_generic_to_shared(p); }

// Every thread of the CTA calls this once; it returns when `bytes` (a multiple of 16, both addresses 16-byte aligned)
// from global `src` have landed at shared `dst`.  Thread 0 issues one cp.async.bulk (SASS UBLKCP) that completes on
// `mbar`, a shared word the CTA uses for this one copy (phase 0).
__device__ __forceinline__ void tma_fetch(void* dst, const void* src, u32 bytes, u64* mbar) {
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(mbar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(mbar)), "r"(bytes)
                     : "memory");
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                smem_u32(dst)),
            "l"(src), "r"(bytes), "r"(smem_u32(mbar))
            : "memory");
    }
    u32 done = 0;
    while (!done) {
        asm volatile(
            "{ .reg .pred q; mbarrier.try_wait.parity.shared::cta.b64 q, [%1], 0; selp.u32 %0, 1, 0, q; }"
            : "=r"(done)
            : "r"(smem_u32(mbar))
            : "memory");
    }
}
