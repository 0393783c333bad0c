// common.cuh -- small sm_90a device helpers shared by the kernels (mbarrier, TMA bulk copy,
// warp reductions; inline PTX), and the counted kernel launch of every C entry point.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <utility>
namespace umr {
extern std::atomic<unsigned long long> g_launches;  // c_api.cu; read through umr_launch_count()

// Launches kernel(args...) with the given grid, block, dynamic shared memory and stream, counted in umr_launch_count().
// Every kernel of the library is launched here, so the count is one per kernel launch by construction; memsets and event
// records are not counted.
template <typename... P, typename... A>
inline void launch(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, A&&... args) {
    kernel<<<grid, block, smem, stream>>>(std::forward<A>(args)...);
    g_launches.fetch_add(1, std::memory_order_relaxed);
}

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

// warp_sum and sum_ascending serve float and double alike
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}
// p[0] + p[1] + ... + p[n-1], left to right: the fixed order of the deterministic reductions' finalize kernels, which sum
// per-CTA partials stored in workspace slots instead of adding them with atomics
template <typename T>
__device__ __forceinline__ T sum_ascending(const T* p, int n) {
    T t = 0;
    for (int k = 0; k < n; ++k) t += p[k];
    return t;
}
// deterministic finalize of a per-row reduction: out[r] = the row's n slots summed in ascending order
template <typename T>
__global__ void k_sum_slot_rows(const T* __restrict__ slots, T* __restrict__ out, int rows, int n) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < rows) out[r] = sum_ascending(slots + (size_t)r * n, n);
}
// grad[b][v] = v's 3-vectors of terms[b] ([width][3] per batch item) summed over a transposed table (vrowptr [V+1], vinc
// listing term indices in ascending order, so the sum order is fixed); a vertex with no entry gets 0.  Serves the flatten
// backward (width 4E: edge * 4 + role) and CorrLossChamfer's (width NS: the selection index j).
template <typename T>
__global__ void __launch_bounds__(256) k_gather3(const T* __restrict__ terms, const int32_t* __restrict__ vrowptr,
                                                 const int32_t* __restrict__ vinc, T* __restrict__ gverts, int V,
                                                 int64_t width) {
    const int b = blockIdx.y;
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const T* tb = terms + (size_t)b * width * 3;
    T g0 = 0, g1 = 0, g2 = 0;
    for (int k = __ldg(vrowptr + v); k < __ldg(vrowptr + v + 1); ++k) {
        const T* t = tb + (size_t)__ldg(vinc + k) * 3;
        g0 += t[0]; g1 += t[1]; g2 += t[2];
    }
    T* o = gverts + ((size_t)b * V + v) * 3;
    o[0] = g0; o[1] = g1; o[2] = g2;
}

// Operations rounded once and never contracted to FMA, whatever the compile flags, for float and double
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }

// float2 / double2 by scalar type
template <typename T> struct Vec2;
template <> struct Vec2<float> { using type = float2; };
template <> struct Vec2<double> { using type = double2; };
template <typename T> using vec2_t = typename Vec2<T>::type;
__device__ __forceinline__ float2 make_vec2(float x, float y) { return make_float2(x, y); }
__device__ __forceinline__ double2 make_vec2(double x, double y) { return make_double2(x, y); }
__device__ __forceinline__ float warp_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 16));
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 8));
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return v;
}

}  // namespace umr
