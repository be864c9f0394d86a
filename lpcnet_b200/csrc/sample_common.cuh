// sample_common.cuh — what the three per-sample kernels (sample_kernel.cu, sample_kernel_f32.cu, sample_kernel_f32n.cu) share:
// the PTX wrappers of their named barriers, mbarriers and TMA bulk copies, and the staging of the constant shared-memory image.
#pragma once
#include <cstdint>
#include "engine.h"
#include "devmath.cuh"

namespace lpcnet_b200 {

// ---- named barriers, mbarriers, TMA bulk copy global -> shared ----
__device__ __forceinline__ void bar_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}

// One thread: copy the constant image (`bytes` from global `src`) to shared address `dst` in 16 KB bulk copies that complete
// on the mbarrier `bar` (armed here for all of them; the readers wait for phase 0).
__device__ __forceinline__ void stage_image(uint32_t dst, const uint8_t *src, uint32_t bytes, uint32_t bar)
{
    mbar_expect_tx(bar, bytes);
    const uint32_t CH = 16384;
    for (uint32_t o = 0; o < bytes; o += CH) bulk_g2s(dst + o, src + o, min(CH, bytes - o), bar);
}

}  // namespace lpcnet_b200
