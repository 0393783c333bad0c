// voxel.cu -- mesh voxelisation, the fourth SoftRas native (external/SoftRas/soft_renderer/cuda/voxelization_cuda_kernel.cu,
// functional/voxelization.py).  Compiled with -fmad=false: the surface test is an arithmetic twin of `voxelize_sub1`
// (same operation order, float or double like AT_DISPATCH_FLOATING_TYPES), so the occupancy is bit-exact.
// Contract and error bound: DESIGN.md §8.
//
//   k_vox_surface<T>  one warp per (batch item, face): the three projections of voxelize_sub1 and the vertex marks of
//                     voxelize_sub2 in one pass, each projection over the face's column box only (whole grid for faces
//                     whose conditioning does not bound the rounding), atomicOr into a z-packed occupancy bitmap
//   k_vox_fill<SMEM>  one CTA per batch item: the "outside" set of voxelize_sub3/sub4 (empty voxels 6-connected through
//                     empty voxels to the boundary) as an on-device fixed point -- run fill along z by word arithmetic,
//                     OR of the 4 neighbouring rows, __syncthreads_or convergence, hard sweep cap.  Volumes in shared
//                     memory for vs <= 64, in the (L2-resident) workspace above
//   k_vox_unpack      result = 1 - visible -> int32 [B,vs,vs,vs], 128-bit stores
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "umr_b200.h"

namespace umr {

constexpr int VOX_SURF_WARPS = 8;
constexpr int VOX_FILL_THREADS = 1024;
constexpr int VOX_SMEM_MAX_VS = 64;  // 2 volumes x 64^3 bits = 64 KB of shared memory per CTA
constexpr size_t VOX_HEADER = 256;   // status word(s) in front of the bitmaps

inline size_t vox_words(int B, int vs) { return (size_t)B * vs * vs * ((vs + 31) / 32); }
inline size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

template <typename T> struct VoxEps;
template <> struct VoxEps<float> { static constexpr double u = 5.9604644775390625e-08; };      // 2^-24
template <> struct VoxEps<double> { static constexpr double u = 1.1102230246251565e-16; };     // 2^-53

__device__ __forceinline__ void vox_set(uint32_t* occ, int vs, int W, int c0, int c1, int c2) {
    atomicOr(occ + ((size_t)c0 * vs + c1) * W + (c2 >> 5), 1u << (c2 & 31));
}

// One projection of voxelize_sub1: column slots (y, x) = coordinates (ys, xs), depth slot zs.  A column passing the
// reference's float test marks (y, x, zi), (y-1, x, zi), (y, x-1, zi), (y-1, x-1, zi) where they lie in the grid.
template <typename T, int ys, int xs, int zs>
__device__ __forceinline__ void vox_axis(const T (&f)[9], uint32_t* occ, int vs, int W, int lane) {
    const T y1d = f[3 + ys] - f[ys], x1d = f[3 + xs] - f[xs], z1d = f[3 + zs] - f[zs];
    const T y2d = f[6 + ys] - f[ys], x2d = f[6 + xs] - f[xs], z2d = f[6 + zs] - f[zs];
    const T det = x1d * y2d - x2d * y1d;
    if (det == 0) return;  // the reference skips the face for every column
    // Column box (DESIGN.md §8): for a face with gamma2 * L^2 / |det| <= 2^-10 a passing column lies within
    // 1 + L/32 of the face's projected bounding box; any other face (thin, huge, non-finite) scans the whole grid.
    int ylo = 0, yhi = vs - 1, xlo = 0, xhi = vs - 1;
    {
        const double L2 = fmax((double)y1d * (double)y1d + (double)x1d * (double)x1d,
                               (double)y2d * (double)y2d + (double)x2d * (double)x2d);
        const double gamma2 = 2.0 * VoxEps<T>::u / (1.0 - 2.0 * VoxEps<T>::u);
        if (gamma2 * L2 <= 0x1p-10 * fabs((double)det) && L2 <= 1e30) {  // false for NaN / inf
            const double m = 1.0 + sqrt(L2) * (1.0 / 32.0);
            const double a0 = f[ys], a1 = f[3 + ys], a2 = f[6 + ys];
            const double b0 = f[xs], b1 = f[3 + xs], b2 = f[6 + xs];
            const double lo_y = floor(fmin(a0, fmin(a1, a2)) - m), hi_y = ceil(fmax(a0, fmax(a1, a2)) + m);
            const double lo_x = floor(fmin(b0, fmin(b1, b2)) - m), hi_x = ceil(fmax(b0, fmax(b1, b2)) + m);
            if (hi_y < 0 || lo_y > vs - 1 || hi_x < 0 || lo_x > vs - 1) return;
            ylo = (int)fmax(lo_y, 0.0); yhi = (int)fmin(hi_y, (double)(vs - 1));
            xlo = (int)fmax(lo_x, 0.0); xhi = (int)fmin(hi_x, (double)(vs - 1));
        }
    }
    const int nx = xhi - xlo + 1;
    const int n = (yhi - ylo + 1) * nx;
    for (int i = lane; i < n; i += 32) {
        const int y = ylo + i / nx, x = xlo + i % nx;
        const T ypd = (T)y - f[ys];
        const T xpd = (T)x - f[xs];
        const T t1 = (y2d * xpd - x2d * ypd) / det;
        const T t2 = (-y1d * xpd + x1d * ypd) / det;
        if (t1 < 0) continue;
        if (t2 < 0) continue;
        if (1 < t1 + t2) continue;
        const T zf = floor(t1 * z1d + t2 * z2d + f[zs]);
        if (!(zf >= 0 && zf < (T)vs)) continue;  // NaN / inf / out of grid: nothing
        const int zi = (int)zf;
        int idx[3];
        idx[zs] = zi;
#pragma unroll
        for (int d = 0; d < 4; ++d) {
            const int yy = y - (d & 1), xx = x - (d >> 1);
            if (yy < 0 || xx < 0) continue;
            idx[ys] = yy;
            idx[xs] = xx;
            vox_set(occ, vs, W, idx[0], idx[1], idx[2]);
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(VOX_SURF_WARPS * 32) k_vox_surface(const T* __restrict__ faces, uint32_t* __restrict__ occ,
                                                                     int64_t nfaces_total, int F, int vs, int W, T scale) {
    const int64_t g = (int64_t)blockIdx.x * VOX_SURF_WARPS + (threadIdx.x >> 5);
    if (g >= nfaces_total) return;
    const int lane = threadIdx.x & 31;
    const int64_t b = g / F;
    T f[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) f[k] = faces[g * 9 + k] * scale;  // `faces *= size` (functional/voxelization.py:44)
    uint32_t* o = occ + (size_t)b * vs * vs * W;
    // voxelize_sub2: floor of each vertex
    if (lane < 3) {
        const T* v = faces + g * 9 + 3 * lane;  // re-read rather than index f[] by lane (keeps f[] in registers)
        const T c0 = floor(v[0] * scale), c1 = floor(v[1] * scale), c2 = floor(v[2] * scale);
        if (c0 >= 0 && c0 < (T)vs && c1 >= 0 && c1 < (T)vs && c2 >= 0 && c2 < (T)vs)
            vox_set(o, vs, W, (int)c0, (int)c1, (int)c2);
    }
    // voxelize_sub1 with the faces permuted [2,1,0], [0,2,1] and unpermuted (voxelization.py:12-17, 47-49)
    vox_axis<T, 2, 1, 0>(f, o, vs, W, lane);
    vox_axis<T, 0, 2, 1>(f, o, vs, W, lane);
    vox_axis<T, 0, 1, 2>(f, o, vs, W, lane);
}

// Run fill toward the high bits: every bit of `e` (empty voxels) in a run of set bits at or above a seed of s (s ⊆ e).
// e + s carries from the lowest seed of each run through the run's remaining set bits, clearing them, and stops at the
// run's end (a clear bit of e), so e & ~(e + s) is the run from the lowest seed up, minus the seeds themselves.
__device__ __forceinline__ uint32_t fill_up(uint32_t s, uint32_t e) { return (e & ~(e + s)) | s; }
__device__ __forceinline__ uint32_t fill_down(uint32_t s, uint32_t e) { return __brev(fill_up(__brev(s), __brev(e))); }

template <bool SMEM>
__global__ void __launch_bounds__(VOX_FILL_THREADS) k_vox_fill(const uint32_t* __restrict__ occ_g, uint32_t* vis_g,
                                                               uint32_t* status, int vs, int W) {
    extern __shared__ uint32_t s_vol[];
    __shared__ unsigned long long s_runs;
    const int R = vs * vs;
    const size_t nw = (size_t)R * W;
    const uint32_t* occ = occ_g + blockIdx.x * nw;
    volatile uint32_t* vis = vis_g + blockIdx.x * nw;
    if (SMEM) {
        uint32_t* so = s_vol;
        for (size_t i = threadIdx.x; i < nw; i += blockDim.x) so[i] = occ[i];
        occ = so;
        vis = s_vol + nw;
    }
    if (threadIdx.x == 0) s_runs = 0;
    __syncthreads();
    const uint32_t top = (vs & 31) ? (1u << (vs & 31)) - 1u : ~0u;  // grid bits of the last word
    auto empty = [&](size_t r, int w) -> uint32_t { return ~occ[r * W + w] & (w == W - 1 ? top : ~0u); };
    const uint32_t last_bit = 1u << ((vs - 1) & 31);

    // seeds: every empty voxel on the boundary.  Rows on the y / x faces of the cube are wholly boundary; other rows
    // are seeded at z = 0 and z = vs-1 and run-filled.  The empty runs are counted for the sweep cap.
    unsigned long long runs = 0;
    for (int r = threadIdx.x; r < R; r += blockDim.x) {
        const int y = r / vs, x = r % vs;
        const bool bnd = y == 0 || y == vs - 1 || x == 0 || x == vs - 1;
        uint32_t carry = 0, prev_top = 0;
        for (int w = 0; w < W; ++w) {
            const uint32_t e = empty(r, w);
            runs += __popc(e & ~((e << 1) | prev_top));
            prev_top = e >> 31;
            uint32_t s = bnd ? e : ((w == 0 ? (e & 1u) : 0u) | (w == W - 1 ? (e & last_bit) : 0u));
            s |= carry & e;
            const uint32_t u = fill_up(s, e);
            carry = u >> 31;
            vis[(size_t)r * W + w] = u;
        }
        carry = 0;
        for (int w = W - 1; w >= 0; --w) {
            const uint32_t e = empty(r, w);
            const uint32_t d = fill_down(vis[(size_t)r * W + w] | ((carry << 31) & e), e);
            carry = d & 1u;
            vis[(size_t)r * W + w] = d;
        }
    }
    atomicAdd(&s_runs, runs);
    __syncthreads();
    // Every productive sweep makes at least one more whole run visible, so runs + 1 sweeps always reach the fixed
    // point.  Hitting the cap means a bug: stop and report it rather than spin on a shared GPU.
    const unsigned long long cap = s_runs + 1;
    for (unsigned long long sweep = 0;; ++sweep) {
        if (sweep >= cap) {
            if (threadIdx.x == 0) atomicOr(status, 1u);
            break;
        }
        int changed = 0;
        for (int r = threadIdx.x; r < R; r += blockDim.x) {
            const int y = r / vs, x = r % vs;
            if (y == 0 || y == vs - 1 || x == 0 || x == vs - 1) continue;  // final since the seeding
            // neighbours' words are read while their owners may be writing them: every value ever stored is a subset
            // of the outside set and a superset of the previous one, so a racy read is only ever a slower read
            uint32_t carry = 0;
            const size_t o = (size_t)r * W;
            for (int w = 0; w < W; ++w) {
                const uint32_t e = empty(r, w);
                const uint32_t old = vis[o + w];
                const uint32_t s = ((old | vis[o + w - W] | vis[o + w + W] | vis[o + w - (size_t)vs * W] |
                                     vis[o + w + (size_t)vs * W]) & e) | (carry & e);
                const uint32_t u = fill_up(s, e);
                carry = u >> 31;
                if (u != old) { vis[o + w] = u; changed = 1; }
            }
            carry = 0;
            for (int w = W - 1; w >= 0; --w) {
                const uint32_t e = empty(r, w);
                const uint32_t old = vis[o + w];
                const uint32_t d = fill_down(old | ((carry << 31) & e), e);
                carry = d & 1u;
                if (d != old) { vis[o + w] = d; changed = 1; }
            }
        }
        if (!__syncthreads_or(changed)) break;
    }
    if (SMEM) {
        uint32_t* out = vis_g + blockIdx.x * nw;
        for (size_t i = threadIdx.x; i < nw; i += blockDim.x) out[i] = vis[i];
    }
}

// voxels = 1 - visible; one thread per 4 consecutive voxels of a row (one int4 store when rows are 16-byte aligned)
__global__ void __launch_bounds__(256) k_vox_unpack(const uint32_t* __restrict__ vis, int32_t* __restrict__ out, int64_t nrows,
                                                    int vs, int W) {
    const int q = (vs + 3) / 4;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nrows * q) return;
    const int64_t r = i / q;
    const int z = (int)(i % q) * 4;
    const uint32_t v = ~(vis[r * W + (z >> 5)] >> (z & 31));
    int32_t* o = out + r * vs + z;
    if ((vs & 3) == 0) {
        *reinterpret_cast<int4*>(o) = make_int4((int)(v & 1u), (int)((v >> 1) & 1u), (int)((v >> 2) & 1u), (int)((v >> 3) & 1u));
    } else {
        for (int k = 0; k < 4 && z + k < vs; ++k) o[k] = (int)((v >> k) & 1u);
    }
}

}  // namespace umr

using namespace umr;

extern "C" size_t umr_voxelize_workspace_bytes(int32_t B, int32_t vs) {
    if (B <= 0 || vs <= 0 || (double)B * vs * vs * vs >= 2147483648.0) return 0;  // umr_voxelize refuses these
    return VOX_HEADER + 2 * align256(vox_words(B, vs) * sizeof(uint32_t));
}

extern "C" int umr_voxelize(const void* faces, int32_t dtype, int32_t* voxels, int32_t B, int32_t F, int32_t vs, double scale,
                            void* workspace, void* stream_) {
    if (B <= 0 || F < 0 || vs < 1 || (dtype != UMR_DTYPE_FLOAT32 && dtype != UMR_DTYPE_FLOAT64)) return UMR_ERR_BAD_ARG;
    if ((double)B * vs * vs * vs >= 2147483648.0) return UMR_ERR_TOO_LARGE;  // the reference's int32 voxel index
    if ((!faces && F > 0) || !voxels || !workspace || ((uintptr_t)voxels & 15) || ((uintptr_t)workspace & 255))
        return UMR_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream_;
    const int W = (vs + 31) / 32;
    const size_t wbytes = align256(vox_words(B, vs) * sizeof(uint32_t));
    uint32_t* status = (uint32_t*)workspace;
    uint32_t* occ = (uint32_t*)((char*)workspace + VOX_HEADER);
    uint32_t* vis = (uint32_t*)((char*)occ + wbytes);
    cudaError_t e = cudaMemsetAsync(workspace, 0, VOX_HEADER + wbytes, st);  // status word + occupancy
    if (e != cudaSuccess) return (int)e;
    const int64_t nf = (int64_t)B * F;
    if (nf > 0) {
        const unsigned blocks = (unsigned)((nf + VOX_SURF_WARPS - 1) / VOX_SURF_WARPS);
        if (dtype == UMR_DTYPE_FLOAT32)
            launch(k_vox_surface<float>, blocks, VOX_SURF_WARPS * 32, 0, st, (const float*)faces, occ, nf, F, vs, W, (float)scale);
        else
            launch(k_vox_surface<double>, blocks, VOX_SURF_WARPS * 32, 0, st, (const double*)faces, occ, nf, F, vs, W, scale);
    }
    if (vs <= VOX_SMEM_MAX_VS) {
        const size_t smem = 2 * (size_t)vs * vs * W * sizeof(uint32_t);
        e = cudaFuncSetAttribute(k_vox_fill<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
        launch(k_vox_fill<true>, B, VOX_FILL_THREADS, smem, st, occ, vis, status, vs, W);
    } else {
        launch(k_vox_fill<false>, B, VOX_FILL_THREADS, 0, st, occ, vis, status, vs, W);
    }
    const int64_t n = (int64_t)B * vs * vs * ((vs + 3) / 4);
    launch(k_vox_unpack, (unsigned)((n + 255) / 256), 256, 0, st, vis, voxels, (int64_t)B * vs * vs, vs, W);
    return (int)cudaGetLastError();
}
