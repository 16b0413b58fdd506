// Shared device-side building blocks for the sm_90a kernels of atlas_b200:
// mbarrier, TMA (cp.async.bulk.tensor) and register re-partitioning (setmaxnreg).  Hand-written inline
// PTX; the warpgroup MMA wrappers live in wgmma.cuh.
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace ab {

// ---------------------------------------------------------------------------------------------
// generic helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "elect.sync _|P, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

// Two fp32 -> packed 16-bit (lo = a, hi = b), round-to-nearest-even.  One F2FP instruction on the ALU pipe; the
// scalar __float2bfloat16_rn / __float2half_rn compile to F2F on the (16 lanes/clk) XU pipe that MUFU.EX2 also needs.
template <bool kBF16>
__device__ __forceinline__ uint32_t pack2_rn(float a, float b) {
    uint32_t d;
    if constexpr (kBF16) {
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(b), "f"(a));
    } else {
        asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(b), "f"(a));
    }
    return d;
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}

__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}

// non-blocking probe (try_wait may suspend the thread for a while before it reports false)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}

// Bounded spin: a protocol bug must surface as a trapped launch with a diagnostic, not as a hung GPU.
// ~2^28 failed probes is several seconds; every wait site passes a distinct `tag`.
#ifndef AB_WATCHDOG_SPINS
#define AB_WATCHDOG_SPINS (1u << 28)
#endif
static __device__ __noinline__ void mbar_watchdog_fire(int tag, uint32_t parity) {
    printf("atlas_b200 watchdog: mbarrier wait timed out (tag %d, parity %u) block %d thread %d\n", tag, parity,
           static_cast<int>(blockIdx.x), static_cast<int>(threadIdx.x));
    __trap();
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag = 0) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins == AB_WATCHDOG_SPINS) mbar_watchdog_fire(tag, parity);
    }
}

// Call-free variant for kernels that re-partition registers with setmaxnreg: a function call (the printf diagnostic
// above) makes ptxas allocate EVERY region of such a kernel under the smallest setmaxnreg value.  Same bounded spin,
// the trap carries no message.
__device__ __forceinline__ void mbar_wait_nocall(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins == AB_WATCHDOG_SPINS) __trap();
    }
}

// ---------------------------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// L2 cache-policy words (createpolicy.fractional encodings used by CUTLASS' TMA::CacheHintSm90)
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* smem_dst, int32_t c0,
                                            int32_t c1, uint64_t cache_hint) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "l"(cache_hint)
        : "memory");
}

// TMA store of a shared-memory box (written by this CTA's threads with generic stores: fence_proxy_async_smem first) to
// global memory through a tensor map; bulk-group completion (commit + wait_group[.read]) by the issuing thread.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem_src, int32_t c0, int32_t c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(map)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the source shared memory of every committed store may be overwritten / all committed stores are complete
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// L2 prefetch of a tensor-map box (no shared-memory destination, no barrier)
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* map, int32_t c0, int32_t c1) {
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0),
                 "r"(c1)
                 : "memory");
}

// ---------------------------------------------------------------------------------------------
// named CTA barriers (ids 1..15; 0 is __syncthreads): `count` threads take part, a multiple of 32.  The non-aligned
// forms, so a warp that just left a single-thread branch may execute them.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) {
    asm volatile("barrier.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t count) {
    asm volatile("barrier.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ---------------------------------------------------------------------------------------------
// register re-partitioning between warpgroups (every warp of a warpgroup executes it)
// ---------------------------------------------------------------------------------------------
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }

}  // namespace ab
