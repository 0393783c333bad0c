// common.cuh -- small sm_90a device helpers shared by the kernels (mbarrier, TMA bulk copy,
// warp reductions).  Inline PTX.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
namespace umr {
extern std::atomic<unsigned long long> g_launches;  // c_api.cu; read through umr_launch_count()
inline void count_launch(int n = 1) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// make the barrier initialisation visible to the async (TMA) proxy
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!ok);
}
// 1-D TMA bulk copy global -> shared (SASS: UBLKCP), completion signalled on an mbarrier.
// dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                             uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// Ampere-style 16-byte async copy global -> shared (SASS: LDGSTS), L2-only caching
__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src_gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// Fire-and-forget float reductions (SASS: RED / ATOMS without return).  Written as PTX on purpose: nvcc
// expands a plain atomicAdd(float*) whose result is unused into a warp-aggregation loop (match.any +
// shuffles) that cost a large share of the backward kernel's instructions.
__device__ __forceinline__ void red_add_global(float* addr, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
// Three consecutive floats (an RGB texel gradient, 12-byte stride) with TWO reductions instead of three: whichever of
// (p, p+1) / (p+1, p+2) is 8-byte aligned goes out as one vector RED (REDG.E.ADD.F32x2, sm_90+), the odd one as a scalar.
// Selected by address parity, no divergence.  The texel REDs are a large part of the streaming backward's memory traffic.
__device__ __forceinline__ void red_add3_global(float* p, float a, float b, float c) {
    const bool mis = (reinterpret_cast<uintptr_t>(p) & 4u) != 0;  // p itself is not 8-byte aligned -> (p+1, p+2) is the pair
    float* pv = p + (mis ? 1 : 0);
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(pv), "f"(mis ? b : a), "f"(mis ? c : b) : "memory");
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p + (mis ? 0 : 2)), "f"(mis ? a : c) : "memory");
}
// four floats of a 16-byte aligned slot in ONE reduction (REDG.E.ADD.F32x4)
__device__ __forceinline__ void red_add4_global(float* p, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void red_add_shared(float* addr, float v) {
    asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(smem_u32(addr)), "f"(v) : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}
// p[0] + p[1] + ... + p[n-1], left to right in float: the fixed order of the deterministic reductions' finalize kernels,
// which sum per-CTA partials stored in workspace slots instead of adding them with atomics
__device__ __forceinline__ float sum_ascending(const float* p, int n) {
    float t = 0.f;
    for (int k = 0; k < n; ++k) t += p[k];
    return t;
}
__device__ __forceinline__ float warp_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 16));
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 8));
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return v;
}

}  // namespace umr
