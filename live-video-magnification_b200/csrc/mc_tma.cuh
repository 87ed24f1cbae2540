// TMA (cp.async.bulk.tensor) + mbarrier primitives shared by the kernels that stage their tiles with the copy engine
// (fused Laplace level kernel, 9x9 Riesz analysis / collapse).  Device-only; included by .cu files.
#pragma once
#include <cuda.h>   // CUtensorMap (types only; the encoder is fetched through cudaGetDriverEntryPoint)
#include <cstdint>

namespace mc {
namespace {

// ---- TMA (cp.async.bulk.tensor) + mbarrier primitives -------------------------------------------
#if defined(MC_CUDA_EMU)   // CPU logic emulation for GPU-less CI (tests/cuda_emu): same calls, emulated copy engine
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) { cuda_emu::mbar_init(bar, count); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) { cuda_emu::mbar_expect_tx(bar, bytes); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) { cuda_emu::mbar_wait(bar, parity); }
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* tm, int x, int y, int z, uint64_t* bar) {
    const int c[3] = {x, y, z};
    cuda_emu::tma_load(dst, tm, c, bar);
}
__device__ __forceinline__ void fence_proxy_async_shared() {}
#else
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");   // make the init visible to the async proxy
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
    // try_wait suspends the thread for a hardware-defined time slice per attempt; a copy that has not landed after
    // 2^22 attempts (seconds) never will — trap so a bad descriptor surfaces as a launch error, not as a hung GPU.
    unsigned ok = 0;
    for (unsigned spin = 0; spin < (1u << 22); ++spin) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
        if (ok) return;
    }
    __trap();
}
// 3-D tiled load {x, y, plane} -> shared; out-of-bounds elements are zero-filled by the TMA unit
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* tm, int x, int y, int z, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(tm), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z) : "memory");
}
// orders this thread's generic-proxy accesses to shared memory before later async-proxy (bulk copy) accesses
__device__ __forceinline__ void fence_proxy_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

#endif


}  // namespace
}  // namespace mc
