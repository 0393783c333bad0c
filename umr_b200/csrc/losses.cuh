// losses.cuh -- the loss kernels shared by float32 and float64, each written once on the scalar type T, with the host
// launchers that the deterministic float32 entry points and the float64 ones have in common.
//
// losses.cu instantiates T = float (built with FMA contraction, as the float32 kernels always were) and keeps the float32
// entry points; losses_f64.cu instantiates T = double in a -fmad=false unit (every double operation rounded once, in the
// written order) and keeps the `umr_*_f64` entry points.  Where the two precisions compute differently on purpose (the IoU
// partial's CTA shape, the sampler's float-only image-gradient atomics) the body says so.  The reductions store one
// partial per CTA into workspace slots in deterministic mode and in float64 (DESIGN.md §2, §10); only float32's default
// mode adds them with atomics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <climits>
#include <type_traits>

#include "common.cuh"
#include "umr_b200.h"

namespace umr {

// ---------------------------------------------------------------------------------------------
// bilinear sampler: grid_sample(bilinear, zeros padding) with the torch-1.1 coordinate map
// (== align_corners=True): ix = (x + 1) / 2 * (W - 1), in T as torch computes it for T.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool inb(int x, int y, int W, int H) { return x >= 0 && x < W && y >= 0 && y < H; }

// One sample's bilinear tap: its top-left corner (x0, y0), the weights of the corners nw = (x0, y0), ne = (x0+1, y0),
// sw = (x0, y0+1), se = (x0+1, y0+1), and which of them lie in the H x W image.  Shared with kp_transfer.cu, which
// samples its keypoint heat maps and the identity grid in exactly this arithmetic.
template <typename T>
struct BilinearTap {
    int x0, y0;
    T nw, ne, sw, se;
    bool v00, v10, v01, v11;
};
template <typename T>
__device__ __forceinline__ BilinearTap<T> bilinear_tap(vec2_t<T> xy, int H, int W) {
    BilinearTap<T> t;
    const T ix = ((xy.x + T(1)) / T(2)) * (T)(W - 1);
    const T iy = ((xy.y + T(1)) / T(2)) * (T)(H - 1);
    const T fx = floor(ix), fy = floor(iy);
    t.x0 = (int)fx;
    t.y0 = (int)fy;
    const int x1 = t.x0 + 1, y1 = t.y0 + 1;
    t.nw = ((T)x1 - ix) * ((T)y1 - iy);
    t.ne = (ix - (T)t.x0) * ((T)y1 - iy);
    t.sw = ((T)x1 - ix) * (iy - (T)t.y0);
    t.se = (ix - (T)t.x0) * (iy - (T)t.y0);
    t.v00 = inb(t.x0, t.y0, W, H);
    t.v10 = inb(x1, t.y0, W, H);
    t.v01 = inb(t.x0, y1, W, H);
    t.v11 = inb(x1, y1, W, H);
    return t;
}
// The sampled value: pixel(x, y) times its weight, summed over the in-image corners in the order nw, ne, sw, se
template <typename T, typename Pixel>
__device__ __forceinline__ T bilinear_value(const BilinearTap<T>& t, Pixel pixel) {
    T acc = 0;
    if (t.v00) acc += pixel(t.x0, t.y0) * t.nw;
    if (t.v10) acc += pixel(t.x0 + 1, t.y0) * t.ne;
    if (t.v01) acc += pixel(t.x0, t.y0 + 1) * t.sw;
    if (t.v11) acc += pixel(t.x0 + 1, t.y0 + 1) * t.se;
    return acc;
}

template <typename T, int C>
__global__ void __launch_bounds__(256) k_sample_fwd(const T* __restrict__ image, const vec2_t<T>* __restrict__ flow,
                                                    T* __restrict__ out, int H, int W, int N) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= N) return;
    const BilinearTap<T> tap = bilinear_tap<T>(__ldg(flow + (size_t)b * N + n), H, W);
    const T* img = image + (size_t)b * C * H * W;
    T* o = out + ((size_t)b * N + n) * C;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const T* p = img + (size_t)c * H * W;
        o[c] = bilinear_value(tap, [&](int x, int y) { return __ldg(p + (size_t)y * W + x); });
    }
}

// grad_flow, one writer per sample.  float32 only: with gimage != NULL the image gradient is also scattered with float
// atomics (the default, non-deterministic path); the deterministic and float64 image gradients are the gather below.
template <typename T, int C>
__global__ void __launch_bounds__(256) k_sample_bwd(const T* __restrict__ image, const vec2_t<T>* __restrict__ flow,
                                                    const T* __restrict__ gout, vec2_t<T>* __restrict__ gflow,
                                                    T* __restrict__ gimage, int H, int W, int N) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= N) return;
    const vec2_t<T> xy = __ldg(flow + (size_t)b * N + n);
    const T ix = ((xy.x + T(1)) / T(2)) * (T)(W - 1);
    const T iy = ((xy.y + T(1)) / T(2)) * (T)(H - 1);
    const T fx = floor(ix), fy = floor(iy);
    const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
    const T wx1 = (T)x1 - ix, wx0 = ix - (T)x0, wy1 = (T)y1 - iy, wy0 = iy - (T)y0;
    const bool v00 = inb(x0, y0, W, H), v10 = inb(x1, y0, W, H), v01 = inb(x0, y1, W, H), v11 = inb(x1, y1, W, H);
    const T* img = image + (size_t)b * C * H * W;
    const T* go = gout + ((size_t)b * N + n) * C;
    T gix = 0, giy = 0;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const T* p = img + (size_t)c * H * W;
        const T g = __ldg(go + c);
        const T a00 = v00 ? __ldg(p + (size_t)y0 * W + x0) : T(0);
        const T a10 = v10 ? __ldg(p + (size_t)y0 * W + x1) : T(0);
        const T a01 = v01 ? __ldg(p + (size_t)y1 * W + x0) : T(0);
        const T a11 = v11 ? __ldg(p + (size_t)y1 * W + x1) : T(0);
        gix += g * ((a10 - a00) * wy1 + (a11 - a01) * wy0);
        giy += g * ((a01 - a00) * wx1 + (a11 - a10) * wx0);
        if constexpr (std::is_same<T, float>::value) {
            if (gimage != nullptr) {
                float* q = gimage + ((size_t)b * C + c) * H * W;
                if (v00) atomicAdd(q + (size_t)y0 * W + x0, g * wx1 * wy1);
                if (v10) atomicAdd(q + (size_t)y0 * W + x1, g * wx0 * wy1);
                if (v01) atomicAdd(q + (size_t)y1 * W + x0, g * wx1 * wy0);
                if (v11) atomicAdd(q + (size_t)y1 * W + x1, g * wx0 * wy0);
            }
        }
    }
    gflow[(size_t)b * N + n] = make_vec2(gix * ((T)(W - 1) / T(2)), giy * ((T)(H - 1) / T(2)));
}

// Deterministic image gradient of the sampler.  Samples are keyed by the cell (y0, x0) of their top-left corner,
// shifted by one so that every cell with an in-bounds corner is in [0, H] x [0, W]: key = b * (H+1)(W+1) +
// (y0+1)(W+1) + (x0+1), from k_sample_bwd's own expressions (so a non-finite coordinate reaches the same pixels);
// a sample with no in-bounds corner gets the drop key B * (H+1)(W+1).
template <typename T>
__global__ void __launch_bounds__(256) k_sample_cells(const vec2_t<T>* __restrict__ flow, int32_t* __restrict__ cells, int B,
                                                      int H, int W, int N) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= N) return;
    const vec2_t<T> xy = __ldg(flow + (size_t)b * N + n);
    const T ix = ((xy.x + T(1)) / T(2)) * (T)(W - 1);
    const T iy = ((xy.y + T(1)) / T(2)) * (T)(H - 1);
    const T fx = floor(ix), fy = floor(iy);
    const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
    const bool any = inb(x0, y0, W, H) || inb(x1, y0, W, H) || inb(x0, y1, W, H) || inb(x1, y1, W, H);
    const int cell = (H + 1) * (W + 1);
    cells[(size_t)b * N + n] = any ? b * cell + (y0 + 1) * (W + 1) + (x0 + 1) : B * cell;
}

// grad_image[b][c][y][x], one thread per (image, pixel): the terms of the four roles the pixel plays, in the order
// 00 of cell (y,x), 10 of cell (y,x-1), 01 of cell (y-1,x), 11 of cell (y-1,x-1); within a role the samples of the
// cell table (rowptr [B(H+1)(W+1)+1], samples: flat sample indices b * N + n) in ascending order.  Each term is
// k_sample_bwd's product, rounded as there.  A pixel no sample touches gets 0.
template <typename T, int C>
__global__ void __launch_bounds__(256) k_sample_bwd_image_gather(const vec2_t<T>* __restrict__ flow, const T* __restrict__ gout,
                                                                 const int32_t* __restrict__ rowptr,
                                                                 const int32_t* __restrict__ samples,
                                                                 T* __restrict__ gimage, int H, int W) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (p >= H * W) return;
    const int y = p / W, x = p - y * W;
    const size_t c0 = (size_t)b * (H + 1) * (W + 1);
    const size_t cell[4] = {c0 + (size_t)(y + 1) * (W + 1) + (x + 1), c0 + (size_t)(y + 1) * (W + 1) + x,
                            c0 + (size_t)y * (W + 1) + (x + 1), c0 + (size_t)y * (W + 1) + x};
    T acc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] = 0;
#pragma unroll
    for (int role = 0; role < 4; ++role) {
        const int k1 = __ldg(rowptr + cell[role] + 1);
        for (int k = __ldg(rowptr + cell[role]); k < k1; ++k) {
            const int s = __ldg(samples + k);
            const vec2_t<T> xy = __ldg(flow + s);
            const T ix = ((xy.x + T(1)) / T(2)) * (T)(W - 1);
            const T iy = ((xy.y + T(1)) / T(2)) * (T)(H - 1);
            const T fx = floor(ix), fy = floor(iy);
            const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
            const T wx1 = (T)x1 - ix, wx0 = ix - (T)x0, wy1 = (T)y1 - iy, wy0 = iy - (T)y0;
            const T wa = (role & 1) ? wx0 : wx1, wb = (role & 2) ? wy0 : wy1;
            const T* go = gout + (size_t)s * C;
#pragma unroll
            for (int c = 0; c < C; ++c) acc[c] = add_rn(acc[c], mul_rn(mul_rn(__ldg(go + c), wa), wb));
        }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) gimage[((size_t)b * C + c) * H * W + p] = acc[c];
}

// ---------------------------------------------------------------------------------------------
// IoU.  The CTA shape differs by precision: float32 512 threads, float4 loads when aligned, 16384 elements per CTA;
// float64 256 threads, scalar loads, 2048 elements per CTA (so the summation orders and workspace sizes differ too).
// ---------------------------------------------------------------------------------------------
template <typename T> constexpr int IOU_THREADS = std::is_same<T, float>::value ? 512 : 256;
template <typename T> constexpr int IOU_PER_CTA = IOU_THREADS<T> * (std::is_same<T, float>::value ? 4 * 8 : 8);

// DET: `inter` / `uni` are the workspace slots [B][gridDim.x]; the CTA stores its partial instead of adding it
template <typename T, bool DET>
__global__ void __launch_bounds__(IOU_THREADS<T>) k_iou_partial(const T* __restrict__ p, const T* __restrict__ t,
                                                                T* __restrict__ inter, T* __restrict__ uni,
                                                                int64_t N, int64_t p_bstride) {
    constexpr int THREADS = IOU_THREADS<T>, PER_CTA = IOU_PER_CTA<T>;
    const int b = blockIdx.y;
    const T* pb = p + (size_t)b * p_bstride;
    const T* tb = t + (size_t)b * N;
    const int64_t begin = (int64_t)blockIdx.x * PER_CTA;
    const int64_t end = min(N, begin + PER_CTA);
    T si = 0, su = 0;
    bool vec = false;
    if constexpr (std::is_same<T, float>::value) {
        vec = ((N & 3) == 0) && ((((uintptr_t)pb | (uintptr_t)tb) & 15) == 0);
        if (vec) {
            for (int64_t i = begin + (int64_t)threadIdx.x * 4; i < end; i += THREADS * 4) {
                const float4 a = __ldg(reinterpret_cast<const float4*>(pb + i));
                const float4 c = __ldg(reinterpret_cast<const float4*>(tb + i));
                si += a.x * c.x; su += a.x + c.x - a.x * c.x;
                si += a.y * c.y; su += a.y + c.y - a.y * c.y;
                si += a.z * c.z; su += a.z + c.z - a.z * c.z;
                si += a.w * c.w; su += a.w + c.w - a.w * c.w;
            }
        }
    }
    if (!vec) {
        for (int64_t i = begin + threadIdx.x; i < end; i += THREADS) {
            const T a = __ldg(pb + i), c = __ldg(tb + i);
            si += a * c; su += a + c - a * c;
        }
    }
    __shared__ T s_i[THREADS / 32], s_u[THREADS / 32];
    si = warp_sum(si); su = warp_sum(su);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s_i[warp] = si; s_u[warp] = su; }
    __syncthreads();
    if (warp == 0) {
        si = lane < THREADS / 32 ? s_i[lane] : T(0);
        su = lane < THREADS / 32 ? s_u[lane] : T(0);
        si = warp_sum(si); su = warp_sum(su);
        if (DET) {
            if (lane == 0) {
                const size_t slot = (size_t)b * gridDim.x + blockIdx.x;
                inter[slot] = si; uni[slot] = su;
            }
        } else {
            if (lane == 0) { atomicAdd(inter + b, si); atomicAdd(uni + b, su); }
        }
    }
}
// deterministic finalize: image b's slots summed in ascending CTA order, then k_iou_finalize's arithmetic
template <typename T>
__global__ void k_iou_finalize_det(const T* __restrict__ si, const T* __restrict__ su, T* __restrict__ inter,
                                   T* __restrict__ uni, T* __restrict__ loss, int B, int nslot) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const T I = sum_ascending(si + (size_t)b * nslot, nslot);
    const T u = sum_ascending(su + (size_t)b * nslot, nslot) + T(1e-6);
    inter[b] = I;
    uni[b] = u;
    loss[b] = T(1) - I / u;
}
template <typename T>
__global__ void __launch_bounds__(256) k_iou_bwd(const T* __restrict__ t, const T* __restrict__ inter,
                                                 const T* __restrict__ uni, const T* __restrict__ gl,
                                                 T* __restrict__ gp, int64_t N) {
    const int b = blockIdx.y;
    const T I = __ldg(inter + b), U = __ldg(uni + b), g = __ldg(gl + b);
    const T k = -g / (U * U);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
        const T tt = __ldg(t + (size_t)b * N + i);
        gp[(size_t)b * N + i] = k * (tt * U - I * (T(1) - tt));
    }
}

// ---------------------------------------------------------------------------------------------
// chamfer: one warp per query point, lanes stride over the key set; lexicographic (value, index)
// minimum => lowest index wins ties, like torch.min.
// ---------------------------------------------------------------------------------------------
// Defined operation order (never contracted to FMA, whatever the compile flags):
//   |p|^2 = ((p0*p0 + p1*p1) + p2*p2),  a.b = ((a0*b0 + a1*b1) + a2*b2),  P = (|q|^2 + |k|^2) - 2*(q.k)
// -- chamfer_python.py:58-63 with every product and sum rounded once.  oracle/losses.py::dist_chamfer_np
// restates exactly this sequence, so distances AND argmins are bit-exact against it.  kp_transfer.cu's nearest-vertex
// and nearest-pixel searches use the same distance and the same warp minimum.
template <typename T, int D>
__device__ __forceinline__ T chamfer_sqnorm(const T (&v)[D]) {
    T s = mul_rn(v[0], v[0]);
#pragma unroll
    for (int d = 1; d < D; ++d) s = add_rn(s, mul_rn(v[d], v[d]));
    return s;
}
// P between a query qv (|q|^2 = qq) and a key kv
template <typename T, int D>
__device__ __forceinline__ T chamfer_dist(const T (&qv)[D], T qq, const T (&kv)[D]) {
    T kk = mul_rn(kv[0], kv[0]), zz = mul_rn(qv[0], kv[0]);
#pragma unroll
    for (int d = 1; d < D; ++d) {
        kk = add_rn(kk, mul_rn(kv[d], kv[d]));
        zz = add_rn(zz, mul_rn(qv[d], kv[d]));
    }
    return sub_rn(add_rn(qq, kk), mul_rn(T(2), zz));  // chamfer_python.py:63 expanded form
}
// every lane of the warp ends with the lexicographic (value, index) minimum of the lanes' (best, bi)
template <typename T>
__device__ __forceinline__ void warp_argmin(T& best, int& bi) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const T ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
}

template <typename T, int D>
__global__ void __launch_bounds__(256) k_chamfer_nn(const T* __restrict__ q, const T* __restrict__ k,
                                                    T* __restrict__ dist, int32_t* __restrict__ idx, int NQ, int NK) {
    const int lane = threadIdx.x & 31;
    const int qi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int b = blockIdx.y;
    if (qi >= NQ) return;
    const T* qp = q + ((size_t)b * NQ + qi) * D;
    T qv[D];
#pragma unroll
    for (int d = 0; d < D; ++d) { qv[d] = __ldg(qp + d); }
    const T qq = chamfer_sqnorm(qv);
    T best = (T)INFINITY;
    int bi = 0x7fffffff;
    const T* kb = k + (size_t)b * NK * D;
    for (int j = lane; j < NK; j += 32) {
        T kv[D];
#pragma unroll
        for (int d = 0; d < D; ++d) kv[d] = __ldg(kb + (size_t)j * D + d);
        const T P = chamfer_dist(qv, qq, kv);
        if (P < best) { best = P; bi = j; }
    }
    warp_argmin(best, bi);
    if (lane == 0) {
        dist[(size_t)b * NQ + qi] = best;
        idx[(size_t)b * NQ + qi] = bi;
    }
}

// Deterministic backward as a gather, one warp per output point i of `q` (no atomics, no workspace):
//   gq[i] = own term (gd_q[i], idx_q[i]) + sum over j with idx_k[j] == i of the j terms (gd_k[j])
// with k_chamfer_bwd's per-term arithmetic.  Lane l owns the j = l (mod 32) in ascending order; the ballot skips the
// 32-wide chunks with no match; the lanes' sums meet in warp_sum's fixed tree.  gd_q / gd_k may be NULL (no term).
template <typename T, int D>
__global__ void __launch_bounds__(256) k_chamfer_bwd_gather(const T* __restrict__ q, const T* __restrict__ k,
                                                            const int32_t* __restrict__ idx_q, const int32_t* __restrict__ idx_k,
                                                            const T* __restrict__ gd_q, const T* __restrict__ gd_k,
                                                            T* __restrict__ gq, int NQ, int NK) {
    const int lane = threadIdx.x & 31;
    const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int b = blockIdx.y;
    if (i >= NQ) return;
    T qv[D], acc[D];
#pragma unroll
    for (int d = 0; d < D; ++d) { qv[d] = __ldg(q + ((size_t)b * NQ + i) * D + d); acc[d] = 0; }
    if (gd_k != nullptr) {
        const int32_t* ik = idx_k + (size_t)b * NK;
        for (int j0 = 0; j0 < NK; j0 += 32) {
            const int j = j0 + lane;
            const bool hit = j < NK && __ldg(ik + j) == i;
            if (__ballot_sync(0xffffffffu, hit) == 0u) continue;
            if (hit) {
                const T g = __ldg(gd_k + (size_t)b * NK + j);
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    const T diff = __ldg(k + ((size_t)b * NK + j) * D + d) - qv[d];
                    acc[d] += T(-2) * g * diff;
                }
            }
        }
#pragma unroll
        for (int d = 0; d < D; ++d) acc[d] = warp_sum(acc[d]);
    }
    if (lane != 0) return;
    T own[D];
#pragma unroll
    for (int d = 0; d < D; ++d) own[d] = 0;
    if (gd_q != nullptr) {
        const T g = __ldg(gd_q + (size_t)b * NQ + i);
        const int j = __ldg(idx_q + (size_t)b * NQ + i);
#pragma unroll
        for (int d = 0; d < D; ++d) own[d] = T(2) * g * (qv[d] - __ldg(k + ((size_t)b * NK + j) * D + d));
    }
#pragma unroll
    for (int d = 0; d < D; ++d) gq[((size_t)b * NQ + i) * D + d] = own[d] + acc[d];
}

// ---------------------------------------------------------------------------------------------
// texture cycle
// ---------------------------------------------------------------------------------------------
// losses.cu: the face-visibility bitmap of the float32 face-id plane, shared by both precisions
__global__ void k_visible(const float* __restrict__ ids, uint8_t* __restrict__ vis, int F, int64_t P);

// DET: `loss` is the workspace slot array [gridDim.x]; every CTA stores its scaled partial
template <typename T, bool DET>
__global__ void __launch_bounds__(256) k_texcycle_fwd(const vec2_t<T>* __restrict__ flow, const vec2_t<T>* __restrict__ prob,
                                                      const uint8_t* __restrict__ vis, T* __restrict__ loss, int n,
                                                      int T2, T scale) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;  // (b, f)
    T acc = 0;
    if (i < n && vis[i]) {
        T sx = 0, sy = 0;
        for (int t = 0; t < T2; ++t) {
            const vec2_t<T> v = __ldg(flow + (size_t)i * T2 + t);
            sx += v.x; sy += v.y;
        }
        const vec2_t<T> p = __ldg(prob + i);
        const T dx = sx / (T)T2 - p.x, dy = sy / (T)T2 - p.y;
        acc = dx * dx + dy * dy;
    }
    acc = warp_sum(acc);
    __shared__ T s[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s[warp] = acc;
    __syncthreads();
    if (warp == 0) {
        acc = lane < 8 ? s[lane] : T(0);
        acc = warp_sum(acc);
        if (DET) {
            if (lane == 0) loss[blockIdx.x] = acc * scale;
        } else {
            if (lane == 0 && acc != 0.f) atomicAdd(loss, acc * scale);
        }
    }
}
template <typename T>
__global__ void __launch_bounds__(256) k_texcycle_bwd(const vec2_t<T>* __restrict__ flow, const vec2_t<T>* __restrict__ prob,
                                                      const uint8_t* __restrict__ vis, const T* __restrict__ gl,
                                                      vec2_t<T>* __restrict__ gflow, int n, int T2, T scale) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    T gx = 0, gy = 0;
    if (vis[i]) {
        T sx = 0, sy = 0;
        for (int t = 0; t < T2; ++t) {
            const vec2_t<T> v = __ldg(flow + (size_t)i * T2 + t);
            sx += v.x; sy += v.y;
        }
        const vec2_t<T> p = __ldg(prob + i);
        const T k = T(2) * __ldg(gl) * scale / (T)T2;
        gx = k * (sx / (T)T2 - p.x);
        gy = k * (sy / (T)T2 - p.y);
    }
    for (int t = 0; t < T2; ++t) gflow[(size_t)i * T2 + t] = make_vec2(gx, gy);
}

// ---------------------------------------------------------------------------------------------
// masked L1 texture loss: nnutils/loss_utils.py:103-116 `texture_loss_masks`
//   per image: sum_{c,h,w} | pred[c]*mask_pred - gt[c]*mask_gt | / (C*H*W)
// pred / mask_pred may be strided views of the renderer's RGBA output (batch strides passed in).
// ---------------------------------------------------------------------------------------------
constexpr int ML1_THREADS = 256;
constexpr int ML1_PER_CTA = ML1_THREADS * 8;  // pixels per CTA

// DET: `loss` is the workspace slot array [B][gridDim.x]; every CTA stores its scaled partial
template <typename T, int C, bool DET>
__global__ void __launch_bounds__(ML1_THREADS) k_masked_l1_fwd(const T* __restrict__ pred, int64_t pred_bs,
                                                              const T* __restrict__ mpred, int64_t mpred_bs,
                                                              const T* __restrict__ gt, const T* __restrict__ mgt,
                                                              T* __restrict__ loss, int64_t HW, T inv_n) {
    const int b = blockIdx.y;
    const T* p = pred + (size_t)b * pred_bs;
    const T* mp = mpred + (size_t)b * mpred_bs;
    const T* g = gt + (size_t)b * C * HW;
    const T* mg = mgt + (size_t)b * HW;
    const int64_t begin = (int64_t)blockIdx.x * ML1_PER_CTA;
    const int64_t end = min(HW, begin + ML1_PER_CTA);
    T acc = 0;
    for (int64_t i = begin + threadIdx.x; i < end; i += ML1_THREADS) {
        const T a = __ldg(mp + i), m = __ldg(mg + i);
#pragma unroll
        for (int c = 0; c < C; ++c) acc += fabs(__ldg(p + (size_t)c * HW + i) * a - __ldg(g + (size_t)c * HW + i) * m);
    }
    acc = warp_sum(acc);
    __shared__ T s[ML1_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s[warp] = acc;
    __syncthreads();
    if (warp == 0) {
        acc = lane < ML1_THREADS / 32 ? s[lane] : T(0);
        acc = warp_sum(acc);
        if (DET) {
            if (lane == 0) loss[(size_t)b * gridDim.x + blockIdx.x] = acc * inv_n;
        } else {
            if (lane == 0) atomicAdd(loss + b, acc * inv_n);
        }
    }
}

template <typename T, int C>
__global__ void __launch_bounds__(ML1_THREADS) k_masked_l1_bwd(const T* __restrict__ pred, int64_t pred_bs,
                                                              const T* __restrict__ mpred, int64_t mpred_bs,
                                                              const T* __restrict__ gt, const T* __restrict__ mgt,
                                                              const T* __restrict__ gl, T* __restrict__ gpred,
                                                              T* __restrict__ gmask, int64_t HW, T inv_n) {
    const int b = blockIdx.y;
    const T* p = pred + (size_t)b * pred_bs;
    const T* mp = mpred + (size_t)b * mpred_bs;
    const T* g = gt + (size_t)b * C * HW;
    const T* mg = mgt + (size_t)b * HW;
    const T k = __ldg(gl + b) * inv_n;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (int64_t)gridDim.x * blockDim.x) {
        const T a = __ldg(mp + i), m = __ldg(mg + i);
        T gm = 0;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const T pv = __ldg(p + (size_t)c * HW + i);
            const T d = pv * a - __ldg(g + (size_t)c * HW + i) * m;
            const T sg = d > T(0) ? k : (d < T(0) ? -k : T(0));  // torch: grad * sign(d), sign(0) = 0
            if (gpred) gpred[((size_t)b * C + c) * HW + i] = sg * a;
            gm += sg * pv;
        }
        if (gmask) gmask[(size_t)b * HW + i] = gm;
    }
}

// ---------------------------------------------------------------------------------------------
// fused loss head:  w_iou * mean_b neg_iou(alpha, mask)  +  w_tex * mean_b masked_L1(rgb, gt, mask, alpha)
// (loss_utils.py:41-48 and :103-116 evaluated on the SAME RGBA render, as train_s1.py:211-215 / the bench step do):
// the RGBA image is read once, forward = one reduction + a one-warp finalize, backward = one kernel that writes the
// complete [B,4,HW] image gradient (round 1: 2 + 2 kernels plus ~20 torch elementwise / fill / add launches).
// ---------------------------------------------------------------------------------------------
constexpr int LH_THREADS = 256;
constexpr int LH_PER_CTA = LH_THREADS * 8;  // pixels per CTA

// acc [B][3] += (sum alpha*m, sum alpha + m - alpha*m, sum_c |rgb_c*alpha - gt_c*m|)
// DET: `acc` is the workspace slot array [B][gridDim.x][3]; every CTA stores its three partials
template <typename T, bool DET>
__global__ void __launch_bounds__(LH_THREADS) k_losshead_partial(const T* __restrict__ rgba, const T* __restrict__ gt,
                                                                const T* __restrict__ mgt, T* __restrict__ acc,
                                                                int64_t HW) {
    const int b = blockIdx.y;
    const T* im = rgba + (size_t)b * 4 * HW;
    const T* g = gt + (size_t)b * 3 * HW;
    const T* mg = mgt + (size_t)b * HW;
    const int64_t begin = (int64_t)blockIdx.x * LH_PER_CTA;
    const int64_t end = min(HW, begin + LH_PER_CTA);
    T si = 0, su = 0, sl = 0;
    for (int64_t i = begin + threadIdx.x; i < end; i += LH_THREADS) {
        const T a = __ldg(im + 3 * HW + i), m = __ldg(mg + i);
        si += a * m;
        su += a + m - a * m;
#pragma unroll
        for (int c = 0; c < 3; ++c) sl += fabs(__ldg(im + (size_t)c * HW + i) * a - __ldg(g + (size_t)c * HW + i) * m);
    }
    si = warp_sum(si); su = warp_sum(su); sl = warp_sum(sl);
    __shared__ T s[3][LH_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s[0][warp] = si; s[1][warp] = su; s[2][warp] = sl; }
    __syncthreads();
    if (warp == 0) {
        si = lane < LH_THREADS / 32 ? s[0][lane] : T(0);
        su = lane < LH_THREADS / 32 ? s[1][lane] : T(0);
        sl = lane < LH_THREADS / 32 ? s[2][lane] : T(0);
        si = warp_sum(si); su = warp_sum(su); sl = warp_sum(sl);
        if (DET) {
            if (lane == 0) {
                T* o = acc + ((size_t)b * gridDim.x + blockIdx.x) * 3;
                o[0] = si; o[1] = su; o[2] = sl;
            }
        } else {
            if (lane == 0) { atomicAdd(acc + b * 3 + 0, si); atomicAdd(acc + b * 3 + 1, su); atomicAdd(acc + b * 3 + 2, sl); }
        }
    }
}
// deterministic pre-pass of k_losshead_finalize: stats[b][k] = image b's slots [nslot][3] summed in ascending CTA order
template <typename T>
__global__ void k_losshead_sum(const T* __restrict__ slots, T* __restrict__ stats, int B, int nslot) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;  // (b, k)
    if (r >= B * 3) return;
    const T* s = slots + (size_t)(r / 3) * nslot * 3 + r % 3;
    T t = 0;
    for (int c = 0; c < nslot; ++c) t += s[(size_t)c * 3];
    stats[r] = t;
}
// one warp: stats[b] = (I, U + 1e-6, per-image L1 mean); per_image[b] = (1 - I/U, L1 mean); loss = weighted batch means
template <typename T>
__global__ void k_losshead_finalize(T* __restrict__ acc, T* __restrict__ per_image, T* __restrict__ loss, int B,
                                    T inv_n, T w_iou, T w_tex) {
    T t_iou = 0, t_tex = 0;
    for (int b = threadIdx.x; b < B; b += 32) {
        const T I = acc[b * 3 + 0], U = acc[b * 3 + 1] + T(1e-6), L = acc[b * 3 + 2] * inv_n;
        acc[b * 3 + 1] = U;
        const T li = T(1) - I / U;
        per_image[b * 2 + 0] = li;
        per_image[b * 2 + 1] = L;
        t_iou += li;
        t_tex += L;
    }
    t_iou = warp_sum(t_iou); t_tex = warp_sum(t_tex);
    if (threadIdx.x == 0) loss[0] = w_iou * (t_iou / B) + w_tex * (t_tex / B);
}
template <typename T>
__global__ void __launch_bounds__(256) k_losshead_bwd(const T* __restrict__ rgba, const T* __restrict__ gt,
                                                      const T* __restrict__ mgt, const T* __restrict__ acc,
                                                      const T* __restrict__ gloss, T* __restrict__ grgba, int64_t HW,
                                                      int B, T inv_n, T w_iou, T w_tex) {
    const int b = blockIdx.y;
    const T* im = rgba + (size_t)b * 4 * HW;
    const T* g = gt + (size_t)b * 3 * HW;
    const T* mg = mgt + (size_t)b * HW;
    T* go = grgba + (size_t)b * 4 * HW;
    const T gl = __ldg(gloss);
    const T I = __ldg(acc + b * 3 + 0), U = __ldg(acc + b * 3 + 1);
    const T ki = -(gl * w_iou / B) / (U * U);  // d(1 - I/U)/dalpha = -(m*U - I*(1-m)) / U^2
    const T kt = gl * w_tex / B * inv_n;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (int64_t)gridDim.x * blockDim.x) {
        const T a = __ldg(im + 3 * HW + i), m = __ldg(mg + i);
        T ga = ki * (m * U - I * (T(1) - m));
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const T pv = __ldg(im + (size_t)c * HW + i);
            const T d = pv * a - __ldg(g + (size_t)c * HW + i) * m;
            const T sg = d > T(0) ? kt : (d < T(0) ? -kt : T(0));  // torch: grad * sign(d), sign(0) = 0
            go[(size_t)c * HW + i] = sg * a;
            ga += sg * pv;
        }
        go[3 * HW + i] = ga;
    }
}

// ---------------------------------------------------------------------------------------------
// part_matching_loss head (nnutils/loss_utils.py, everything after the part render; DESIGN.md §13).  Per image b, with
// proj = (c0, P_1..P_4) and Q the five part_segs channels, S = softmax_c(proj), R = softmax_c(Q), x/y the float32
// coordinate maps of `_coordinate_maps`:
//   terms[b][0] = sum_{c=1..4, d} (C_cd - CQ_cd)^2,  C_c = (sum m x, sum m y) / sum m,  m = S_c + 1e-3 (CQ likewise from R)
//   terms[b][1] = mse: sum_c w_c sum_p (proj_c / mp_c - Q_c / mq_c)^2,  mp_c = clamp_min(max_p proj_c, 1e-5) (mq_c of Q)
//                 kld: sum_{c,p} xlogy(R, R) - R log_softmax_c(proj)
// Forward: a per-CTA partial pass (centroid sums of S and R, the KL sum, max and arg-max of all ten channels) into
// workspace slots, a per-image finalize that sums the slots in ascending order, and for mse a second partial pass (the
// terms and, per channel, sum_p d_c proj_c for the max's adjoint) with its finalize.  Backward: one elementwise pass from
// per-image adjoints of the two terms.  No atomics: every output is bitwise reproducible.
// ---------------------------------------------------------------------------------------------
constexpr int PH_THREADS = 256;
constexpr int PH_PER_CTA = PH_THREADS * 8;  // pixels per CTA
constexpr int PH_SUMS = 25;                 // (Z, X, Y) of S_1..S_4, then of R_1..R_4, then the KL sum
constexpr int PH_MAX = 10;                  // max of proj_0..4, then of Q_0..4
constexpr int PH_MSE = 5;                   // E, then G_1..G_4 = sum_p d_c proj_c
constexpr int PH_SLOT = PH_SUMS + PH_MAX + PH_MSE;
// per-image stats: Z_1..4 [0,4), C [4,12), CQ [12,20), mp [20,25), mq [25,30), raw max of proj [30,35), G [35,40)
constexpr int PH_STATS = 40;
constexpr int PH_IDX = 8;                   // per-image int32: arg-max of proj_0..4 (3 unused)

template <typename T>
struct PartHeadIn {
    const T* map[4];
    int64_t map_bs[4];
    const T* c0;
    int64_t c0_bs;
    const T* q;
    int64_t q_bs;
};

__device__ __forceinline__ float ph_exp(float v) { return expf(v); }
__device__ __forceinline__ double ph_exp(double v) { return exp(v); }
__device__ __forceinline__ float ph_log(float v) { return logf(v); }
__device__ __forceinline__ double ph_log(double v) { return log(v); }

// `_coordinate_maps`: k / n * 2 - 1 evaluated in double and rounded to float32 (widened again for T = double)
template <typename T>
__device__ __forceinline__ T ph_coord(int k, int n) { return (T)(float)((double)k / (double)n * 2.0 - 1.0); }

// torch.max's choice: NaN wins, then the larger value, then the lower flat index (a total order, so any reduction tree
// picks the same element)
template <typename T>
__device__ __forceinline__ bool ph_beats(T a, int ia, T b, int ib) {
    const bool na = a != a, nb = b != b;
    if (na || nb) return na && (!nb || ia < ib);
    return a > b || (a == b && ia < ib);
}

template <typename T>
__device__ __forceinline__ void ph_load(const PartHeadIn<T>& in, int b, int64_t HW, int p, T v[5], T q[5]) {
    v[0] = __ldg(in.c0 + (size_t)b * in.c0_bs + p);
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k + 1] = __ldg(in.map[k] + (size_t)b * in.map_bs[k] + p);
    const T* qb = in.q + (size_t)b * in.q_bs;
#pragma unroll
    for (int c = 0; c < 5; ++c) q[c] = __ldg(qb + (size_t)c * HW + p);
}

// s[c] = softmax over the five channels; returns log of the sum of exp(v - max), with `mx` the max
template <typename T>
__device__ __forceinline__ void ph_softmax(const T v[5], T s[5], T& mx, T& sum) {
    mx = v[0];
#pragma unroll
    for (int c = 1; c < 5; ++c) mx = v[c] > mx ? v[c] : mx;
    sum = 0;
#pragma unroll
    for (int c = 0; c < 5; ++c) { s[c] = ph_exp(v[c] - mx); sum += s[c]; }
#pragma unroll
    for (int c = 0; c < 5; ++c) s[c] = s[c] / sum;
}

template <typename T>
__global__ void __launch_bounds__(PH_THREADS) k_part_head_partial(const PartHeadIn<T> in, T* __restrict__ slots,
                                                                  int32_t* __restrict__ slot_idx, int H, int kld) {
    const int b = blockIdx.y;
    const int64_t HW = (int64_t)H * H;
    const int begin = blockIdx.x * PH_PER_CTA;
    const int end = (int)min(HW, (int64_t)begin + PH_PER_CTA);
    T acc[PH_SUMS];
#pragma unroll
    for (int k = 0; k < PH_SUMS; ++k) acc[k] = 0;
    T mv[PH_MAX];
    int mi[PH_MAX];
#pragma unroll
    for (int c = 0; c < PH_MAX; ++c) { mv[c] = -(T)INFINITY; mi[c] = INT_MAX; }
    for (int p = begin + threadIdx.x; p < end; p += PH_THREADS) {
        const int i = p / H, j = p - i * H;
        const T x = ph_coord<T>(j, H), y = ph_coord<T>(i, H);
        T v[5], q[5], s[5], r[5], mx, sum, qmx, qsum;
        ph_load(in, b, HW, p, v, q);
#pragma unroll
        for (int c = 0; c < 5; ++c) {
            if (ph_beats(v[c], p, mv[c], mi[c])) { mv[c] = v[c]; mi[c] = p; }
            if (ph_beats(q[c], p, mv[5 + c], mi[5 + c])) { mv[5 + c] = q[c]; mi[5 + c] = p; }
        }
        ph_softmax(v, s, mx, sum);
        ph_softmax(q, r, qmx, qsum);
#pragma unroll
        for (int c = 1; c < 5; ++c) {
            const T m = s[c] + T(1e-3), mr = r[c] + T(1e-3);
            acc[3 * (c - 1) + 0] += m;
            acc[3 * (c - 1) + 1] += m * x;
            acc[3 * (c - 1) + 2] += m * y;
            acc[12 + 3 * (c - 1) + 0] += mr;
            acc[12 + 3 * (c - 1) + 1] += mr * x;
            acc[12 + 3 * (c - 1) + 2] += mr * y;
        }
        if (kld) {
            const T lse = mx + ph_log(sum);
#pragma unroll
            for (int c = 0; c < 5; ++c) acc[24] += (r[c] == T(0) ? T(0) : r[c] * ph_log(r[c])) - r[c] * (v[c] - lse);  // xlogy(R, R) - R logS
        }
    }
    __shared__ T s_sum[PH_THREADS / 32][PH_SUMS];
    __shared__ T s_mv[PH_THREADS / 32][PH_MAX];
    __shared__ int s_mi[PH_THREADS / 32][PH_MAX];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < PH_SUMS; ++k) {
        const T t = warp_sum(acc[k]);
        if (lane == 0) s_sum[warp][k] = t;
    }
#pragma unroll
    for (int c = 0; c < PH_MAX; ++c) {
        T a = mv[c];
        int ia = mi[c];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const T ob = __shfl_xor_sync(0xffffffffu, a, o);
            const int oi = __shfl_xor_sync(0xffffffffu, ia, o);
            if (ph_beats(ob, oi, a, ia)) { a = ob; ia = oi; }
        }
        if (lane == 0) { s_mv[warp][c] = a; s_mi[warp][c] = ia; }
    }
    __syncthreads();
    const size_t slot = (size_t)b * gridDim.x + blockIdx.x;
    const int t = threadIdx.x;
    if (t < PH_SUMS) {
        T tot = 0;
        for (int w = 0; w < PH_THREADS / 32; ++w) tot += s_sum[w][t];
        slots[slot * PH_SLOT + t] = tot;
    } else if (t >= 32 && t < 32 + PH_MAX) {
        const int c = t - 32;
        T a = s_mv[0][c];
        int ia = s_mi[0][c];
        for (int w = 1; w < PH_THREADS / 32; ++w)
            if (ph_beats(s_mv[w][c], s_mi[w][c], a, ia)) { a = s_mv[w][c]; ia = s_mi[w][c]; }
        slots[slot * PH_SLOT + PH_SUMS + c] = a;
        slot_idx[slot * PH_MAX + c] = ia;
    }
}

// one CTA per image: the slots summed / reduced in ascending CTA order, then the centroids, lmeqv and the clamped maxima
template <typename T>
__global__ void __launch_bounds__(64) k_part_head_finalize(const T* __restrict__ slots, const int32_t* __restrict__ slot_idx,
                                                           T* __restrict__ stats, int32_t* __restrict__ idx,
                                                           T* __restrict__ terms, int nslot, int kld) {
    const int b = blockIdx.x, t = threadIdx.x;
    __shared__ T tot[PH_SUMS];
    const T* sl = slots + (size_t)b * nslot * PH_SLOT;
    T* st = stats + (size_t)b * PH_STATS;
    if (t < PH_SUMS) {
        T a = 0;
        for (int k = 0; k < nslot; ++k) a += sl[(size_t)k * PH_SLOT + t];
        tot[t] = a;
    } else if (t >= 32 && t < 32 + PH_MAX) {
        const int c = t - 32;
        const int32_t* si = slot_idx + (size_t)b * nslot * PH_MAX;
        T a = sl[PH_SUMS + c];
        int ia = si[c];
        for (int k = 1; k < nslot; ++k) {
            const T o = sl[(size_t)k * PH_SLOT + PH_SUMS + c];
            const int oi = si[(size_t)k * PH_MAX + c];
            if (ph_beats(o, oi, a, ia)) { a = o; ia = oi; }
        }
        const T clamped = a < T(1e-5) ? T(1e-5) : a;   // clamp_min keeps a NaN
        if (c < 5) {
            st[20 + c] = clamped;
            st[30 + c] = a;
            idx[(size_t)b * PH_IDX + c] = ia;
        } else {
            st[25 + c - 5] = clamped;
        }
    }
    __syncthreads();
    if (t == 0) {
        T L = 0;
        for (int c = 0; c < 4; ++c) {
            const T z = tot[3 * c], zq = tot[12 + 3 * c];
            st[c] = z;
            for (int d = 0; d < 2; ++d) {
                const T cc = tot[3 * c + 1 + d] / z, cq = tot[12 + 3 * c + 1 + d] / zq;
                st[4 + 2 * c + d] = cc;
                st[12 + 2 * c + d] = cq;
                L += (cc - cq) * (cc - cq);
            }
        }
        terms[2 * b] = L;
        if (kld) terms[2 * b + 1] = tot[24];
    }
}

// mse: E and G_1..G_4 partials once the maxima are known
template <typename T>
__global__ void __launch_bounds__(PH_THREADS) k_part_head_mse(const PartHeadIn<T> in, const T* __restrict__ w,
                                                              const T* __restrict__ stats, T* __restrict__ slots, int H) {
    const int b = blockIdx.y;
    const int64_t HW = (int64_t)H * H;
    const int begin = blockIdx.x * PH_PER_CTA;
    const int end = (int)min(HW, (int64_t)begin + PH_PER_CTA);
    const T* st = stats + (size_t)b * PH_STATS;
    T mp[5], mq[5], wc[5], acc[PH_MSE];
#pragma unroll
    for (int c = 0; c < 5; ++c) { mp[c] = st[20 + c]; mq[c] = st[25 + c]; wc[c] = __ldg(w + c); acc[c] = 0; }
    for (int p = begin + threadIdx.x; p < end; p += PH_THREADS) {
        T v[5], q[5];
        ph_load(in, b, HW, p, v, q);
#pragma unroll
        for (int c = 0; c < 5; ++c) {
            const T d = v[c] / mp[c] - q[c] / mq[c];
            acc[0] += (d * d) * wc[c];
            if (c > 0) acc[c] += d * v[c];
        }
    }
    __shared__ T s[PH_THREADS / 32][PH_MSE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < PH_MSE; ++k) {
        const T t = warp_sum(acc[k]);
        if (lane == 0) s[warp][k] = t;
    }
    __syncthreads();
    if (threadIdx.x < PH_MSE) {
        T tot = 0;
        for (int w2 = 0; w2 < PH_THREADS / 32; ++w2) tot += s[w2][threadIdx.x];
        slots[((size_t)b * gridDim.x + blockIdx.x) * PH_SLOT + PH_SUMS + PH_MAX + threadIdx.x] = tot;
    }
}
template <typename T>
__global__ void __launch_bounds__(32) k_part_head_mse_finalize(const T* __restrict__ slots, T* __restrict__ stats,
                                                               T* __restrict__ terms, int nslot) {
    const int b = blockIdx.x, t = threadIdx.x;
    if (t >= PH_MSE) return;
    const T* sl = slots + (size_t)b * nslot * PH_SLOT + PH_SUMS + PH_MAX + t;
    T a = 0;
    for (int k = 0; k < nslot; ++k) a += sl[(size_t)k * PH_SLOT];
    if (t == 0) terms[2 * b + 1] = a;
    else stats[(size_t)b * PH_STATS + 35 + t] = a;
}

// grad_maps [B,4,HW] from the per-image adjoints grad_terms [B,2]
template <typename T>
__global__ void __launch_bounds__(256) k_part_head_bwd(const PartHeadIn<T> in, const T* __restrict__ w,
                                                       const T* __restrict__ stats, const int32_t* __restrict__ idx,
                                                       const T* __restrict__ gterms, T* __restrict__ gmaps, int H, int kld) {
    const int b = blockIdx.y;
    const int64_t HW = (int64_t)H * H;
    const T* st = stats + (size_t)b * PH_STATS;
    const T aL = __ldg(gterms + 2 * b), aE = __ldg(gterms + 2 * b + 1);
    T cx[4], cy[4], kx[4], ky[4], kd[4], km[4], wc[4], mp[4];
    int im[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const T z = st[c];
        cx[c] = st[4 + 2 * c];
        cy[c] = st[5 + 2 * c];
        kx[c] = aL * (T(2) * (cx[c] - st[12 + 2 * c])) / z;   // d terms[0] / d m_c = aL * 2 (C - CQ) . (xy - C) / Z_c
        ky[c] = aL * (T(2) * (cy[c] - st[13 + 2 * c])) / z;
        mp[c] = st[21 + c];
        wc[c] = __ldg(w + 1 + c);
        kd[c] = aE * T(2) * wc[c] / mp[c];
        km[c] = st[31 + c] >= T(1e-5) ? aE * (T(-2) * wc[c] * st[36 + c] / (mp[c] * mp[c])) : T(0);  // clamped: none
        im[c] = idx[(size_t)b * PH_IDX + 1 + c];
    }
    T mq[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) mq[c] = st[26 + c];
    T* gb = gmaps + (size_t)b * 4 * HW;
    for (int64_t pp = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pp < HW; pp += (int64_t)gridDim.x * blockDim.x) {
        const int p = (int)pp;
        const int i = p / H, j = p - i * H;
        const T x = ph_coord<T>(j, H), y = ph_coord<T>(i, H);
        T v[5], q[5], s[5], mx, sum;
        ph_load(in, b, HW, p, v, q);
        ph_softmax(v, s, mx, sum);
        T gs[4], dot = 0;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            gs[c] = kx[c] * (x - cx[c]) + ky[c] * (y - cy[c]);
            dot += s[c + 1] * gs[c];
        }
        T r[5], rsum = 0;
        if (kld) {
            T qmx, qsum;
            ph_softmax(q, r, qmx, qsum);
#pragma unroll
            for (int c = 0; c < 5; ++c) rsum += r[c];
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            T g = s[c + 1] * (gs[c] - dot);
            if (kld) {
                g += aE * (s[c + 1] * rsum - r[c + 1]);
            } else {
                g += kd[c] * (v[c + 1] / mp[c] - q[c + 1] / mq[c]);
                if (p == im[c]) g += km[c];
            }
            gb[(size_t)c * HW + p] = g;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Host launchers shared by the deterministic float32 entry points (losses.cu) and the float64 ones (losses_f64.cu).
// Each validates as both entry points do; where their checks differ, the entry points check and call the launcher.
// ---------------------------------------------------------------------------------------------
template <typename T> static unsigned iou_slots(int64_t N) { return (unsigned)((N + IOU_PER_CTA<T> - 1) / IOU_PER_CTA<T>); }
static inline unsigned ml1_slots(int64_t HW) { return (unsigned)((HW + ML1_PER_CTA - 1) / ML1_PER_CTA); }
static inline unsigned lh_slots(int64_t HW) { return (unsigned)((HW + LH_PER_CTA - 1) / LH_PER_CTA); }

static inline bool cells_too_large(int32_t B, int32_t H, int32_t W) {
    return B > 65535 || (int64_t)B * ((int64_t)H + 1) * ((int64_t)W + 1) > INT_MAX;
}

// The sampler's flow and TexCycle's flow / prob / grad_flow are read and written as vec2_t<T> (float2 / double2), which
// needs an address aligned to 2 * sizeof(T); a misaligned one would fault on the device.  NULL passes.
template <typename T>
static inline bool vec2_misaligned(const T* p) {
    return ((uintptr_t)p & (2 * sizeof(T) - 1)) != 0;
}

// f(std::integral_constant<int, C>{}) for the channel count C of the sampler kernels; 1 <= C <= 4
template <typename Fn>
static void with_channels(int32_t C, Fn&& f) {
    switch (C) {
        case 1: f(std::integral_constant<int, 1>{}); break;
        case 2: f(std::integral_constant<int, 2>{}); break;
        case 3: f(std::integral_constant<int, 3>{}); break;
        default: f(std::integral_constant<int, 4>{}); break;
    }
}

template <typename T>
static int sample_forward(const T* image, const T* flow, T* out, int32_t B, int32_t C, int32_t H, int32_t W, int32_t N,
                          void* stream_) {
    if (!image || !flow || !out || B <= 0 || C <= 0 || H <= 0 || W <= 0 || N <= 0 || vec2_misaligned(flow))
        return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (C > 4) return UMR_ERR_UNSUPPORTED;
    with_channels(C, [&](auto c) {
        launch(k_sample_fwd<T, c>, dim3((N + 255) / 256, B), 256, 0, (cudaStream_t)stream_, image,
               reinterpret_cast<const vec2_t<T>*>(flow), out, H, W, N);
    });
    return (int)cudaGetLastError();
}

template <typename T>
static int sample_cells(const T* flow, int32_t* cells, int32_t B, int32_t H, int32_t W, int32_t N, void* stream_) {
    if (!flow || !cells || B <= 0 || H <= 0 || W <= 0 || N <= 0 || vec2_misaligned(flow)) return UMR_ERR_BAD_ARG;
    if (cells_too_large(B, H, W)) return UMR_ERR_TOO_LARGE;
    launch(k_sample_cells<T>, dim3((N + 255) / 256, B), 256, 0, (cudaStream_t)stream_,
           reinterpret_cast<const vec2_t<T>*>(flow), cells, B, H, W, N);
    return (int)cudaGetLastError();
}

// grad_flow from k_sample_bwd (no image gradient there), the image gradient from the per-pixel gather over the cell table
template <typename T>
static int sample_backward_gather(const T* image, const T* flow, const T* grad_out, T* grad_flow, T* grad_image, int32_t B,
                                  int32_t C, int32_t H, int32_t W, int32_t N, const int32_t* cell_rowptr,
                                  const int32_t* cell_samples, void* stream_) {
    if (!image || !flow || !grad_out || !grad_flow || B <= 0 || C <= 0 || H <= 0 || W <= 0 || N <= 0 ||
        vec2_misaligned(flow) || vec2_misaligned(grad_flow))
        return UMR_ERR_BAD_ARG;
    if (grad_image && (!cell_rowptr || !cell_samples)) return UMR_ERR_BAD_ARG;
    if (cells_too_large(B, H, W)) return UMR_ERR_TOO_LARGE;
    if (C > 4) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const vec2_t<T>* fl = reinterpret_cast<const vec2_t<T>*>(flow);
    with_channels(C, [&](auto c) {
        launch(k_sample_bwd<T, c>, dim3((N + 255) / 256, B), 256, 0, st, image, fl, grad_out,
               reinterpret_cast<vec2_t<T>*>(grad_flow), nullptr, H, W, N);
        if (grad_image)
            launch(k_sample_bwd_image_gather<T, c>, dim3((H * W + 255) / 256, B), 256, 0, st, fl, grad_out, cell_rowptr,
                   cell_samples, grad_image, H, W);
    });
    return (int)cudaGetLastError();
}

template <typename T>
static size_t iou_workspace_bytes(int32_t B, int64_t N) {
    if (B <= 0 || N <= 0) return 0;
    return (size_t)2 * B * iou_slots<T>(N) * sizeof(T);
}
template <typename T>
static int iou_forward_slots(const T* predict, int64_t predict_bstride, const T* target, T* inter, T* uni, T* loss, int32_t B,
                             int64_t N, void* workspace, void* stream_) {
    if (!predict || !target || !inter || !uni || !loss || !workspace || B <= 0 || N <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const unsigned gx = iou_slots<T>(N);
    T* si = (T*)workspace;
    T* su = si + (size_t)B * gx;
    launch(k_iou_partial<T, true>, dim3(gx, B), IOU_THREADS<T>, 0, st, predict, target, si, su, N, predict_bstride);
    launch(k_iou_finalize_det<T>, (B + 127) / 128, 128, 0, st, si, su, inter, uni, loss, B, (int)gx);
    return (int)cudaGetLastError();
}
template <typename T>
static int iou_backward(const T* target, const T* inter, const T* uni, const T* grad_loss, T* grad_predict, int32_t B,
                        int64_t N, void* stream_) {
    if (!target || !inter || !uni || !grad_loss || !grad_predict || B <= 0 || N <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    const unsigned gx = (unsigned)std::min<int64_t>((N + 1023) / 1024, 1024);
    launch(k_iou_bwd<T>, dim3(gx, B), 256, 0, (cudaStream_t)stream_, target, inter, uni, grad_loss, grad_predict, N);
    return (int)cudaGetLastError();
}

template <typename T>
static int chamfer_forward(const T* a, const T* b, T* dist_ab, T* dist_ba, int32_t* idx_ab, int32_t* idx_ba, int32_t B,
                           int32_t N, int32_t M, int32_t D, void* stream_) {
    if (!a || !b || !dist_ab || !dist_ba || !idx_ab || !idx_ba || B <= 0 || N <= 0 || M <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (D != 2 && D != 3) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const dim3 g1((N + 7) / 8, B), g2((M + 7) / 8, B);
    auto nn = D == 2 ? k_chamfer_nn<T, 2> : k_chamfer_nn<T, 3>;
    launch(nn, g1, 256, 0, st, a, b, dist_ab, idx_ab, N, M);
    launch(nn, g2, 256, 0, st, b, a, dist_ba, idx_ba, M, N);
    return (int)cudaGetLastError();
}
template <typename T>
static int chamfer_backward_gather(const T* a, const T* b, const int32_t* idx_ab, const int32_t* idx_ba, const T* grad_dist_ab,
                                   const T* grad_dist_ba, T* grad_a, T* grad_b, int32_t B, int32_t N, int32_t M, int32_t D,
                                   void* stream_) {
    if (!a || !b || !grad_a || !grad_b || B <= 0 || N <= 0 || M <= 0) return UMR_ERR_BAD_ARG;
    if ((grad_dist_ab && !idx_ab) || (grad_dist_ba && !idx_ba)) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (D != 2 && D != 3) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const dim3 g1((N + 7) / 8, B), g2((M + 7) / 8, B);  // one warp per output point
    auto gather = D == 2 ? k_chamfer_bwd_gather<T, 2> : k_chamfer_bwd_gather<T, 3>;
    launch(gather, g1, 256, 0, st, a, b, idx_ab, idx_ba, grad_dist_ab, grad_dist_ba, grad_a, N, M);
    launch(gather, g2, 256, 0, st, b, a, idx_ba, idx_ab, grad_dist_ba, grad_dist_ab, grad_b, M, N);
    return (int)cudaGetLastError();
}

template <typename T>
static size_t texcycle_workspace_bytes(int32_t B, int32_t F) {
    if (B <= 0 || F <= 0) return 0;
    return (size_t)(((int64_t)B * F + 255) / 256) * sizeof(T);
}
// the bitmap of the face-id plane (if given; NULL: `visible` was already filled by umr_raster_visibility), the per-CTA
// slots and their sum
template <typename T>
static int texcycle_forward_slots(const T* flow, const T* prob, const float* face_ids, uint8_t* visible, T* loss, int32_t B,
                                  int32_t F, int32_t T2, int64_t P, void* workspace, void* stream_) {
    if (!flow || !prob || !visible || !loss || !workspace || B <= 0 || F <= 0 || T2 <= 0 || (face_ids && P <= 0) ||
        vec2_misaligned(flow) || vec2_misaligned(prob))
        return UMR_ERR_BAD_ARG;
    if (B > 65535 || (int64_t)B * F > INT_MAX) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    if (face_ids) {   // the bitmap only ever receives 1s: its bytes do not depend on the order of the stores
        cudaError_t e = cudaMemsetAsync(visible, 0, (size_t)B * F, st);
        if (e != cudaSuccess) return (int)e;
        const int64_t blocks = (P / 4 + 255) / 256 + 1;
        launch(k_visible, dim3((unsigned)(blocks > 1024 ? 1024 : blocks), B), 256, 0, st, face_ids, visible, F, P);
    }
    const int n = B * F;
    const int gx = (n + 255) / 256;
    T* slots = (T*)workspace;
    launch(k_texcycle_fwd<T, true>, gx, 256, 0, st, reinterpret_cast<const vec2_t<T>*>(flow),
           reinterpret_cast<const vec2_t<T>*>(prob), visible, slots, n, T2, T(1) / ((T)n * T(2)));  // MSELoss mean over B*F*2
    launch(k_sum_slot_rows<T>, 1, 32, 0, st, slots, loss, 1, gx);
    return (int)cudaGetLastError();
}
// after the entry point's checks
template <typename T>
static int texcycle_backward(const T* flow, const T* prob, const uint8_t* visible, const T* grad_loss, T* grad_flow, int32_t B,
                             int32_t F, int32_t T2, void* stream_) {
    const int n = B * F;
    launch(k_texcycle_bwd<T>, (n + 255) / 256, 256, 0, (cudaStream_t)stream_, reinterpret_cast<const vec2_t<T>*>(flow),
           reinterpret_cast<const vec2_t<T>*>(prob), visible, grad_loss, reinterpret_cast<vec2_t<T>*>(grad_flow), n, T2,
           T(1) / ((T)n * T(2)));
    return (int)cudaGetLastError();
}

template <typename T>
static size_t masked_l1_workspace_bytes(int32_t B, int64_t HW) {
    if (B <= 0 || HW <= 0) return 0;
    return (size_t)B * ml1_slots(HW) * sizeof(T);
}
template <typename T>
static int masked_l1_forward_slots(const T* pred, int64_t pred_bstride, const T* mask_pred, int64_t mask_pred_bstride,
                                   const T* gt, const T* mask_gt, T* loss, int32_t B, int32_t C, int64_t HW, void* workspace,
                                   void* stream_) {
    if (!pred || !mask_pred || !gt || !mask_gt || !loss || !workspace || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (C != 3 && C != 1) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const unsigned gx = ml1_slots(HW);
    const dim3 grid(gx, B);
    const T inv_n = T(1) / ((T)C * (T)HW);
    T* slots = (T*)workspace;
    launch(C == 3 ? k_masked_l1_fwd<T, 3, true> : k_masked_l1_fwd<T, 1, true>, grid, ML1_THREADS, 0, st, pred, pred_bstride,
           mask_pred, mask_pred_bstride, gt, mask_gt, slots, HW, inv_n);
    launch(k_sum_slot_rows<T>, (B + 127) / 128, 128, 0, st, slots, loss, B, (int)gx);
    return (int)cudaGetLastError();
}
template <typename T>
static int masked_l1_backward(const T* pred, int64_t pred_bstride, const T* mask_pred, int64_t mask_pred_bstride, const T* gt,
                              const T* mask_gt, const T* grad_loss, T* grad_pred, T* grad_mask_pred, int32_t B, int32_t C,
                              int64_t HW, void* stream_) {
    if (!pred || !mask_pred || !gt || !mask_gt || !grad_loss || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (C != 3 && C != 1) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const dim3 grid((unsigned)std::min<int64_t>((HW + 1023) / 1024, 1024), B);
    const T inv_n = T(1) / ((T)C * (T)HW);
    launch(C == 3 ? k_masked_l1_bwd<T, 3> : k_masked_l1_bwd<T, 1>, grid, 256, 0, st, pred, pred_bstride, mask_pred,
           mask_pred_bstride, gt, mask_gt, grad_loss, grad_pred, grad_mask_pred, HW, inv_n);
    return (int)cudaGetLastError();
}

template <typename T>
static size_t loss_head_workspace_bytes(int32_t B, int64_t HW) {
    if (B <= 0 || HW <= 0) return 0;
    return (size_t)3 * B * lh_slots(HW) * sizeof(T);
}
template <typename T>
static int loss_head_forward_slots(const T* rgba, const T* gt, const T* mask_gt, T* stats, T* per_image, T* loss, int32_t B,
                                   int64_t HW, T w_iou, T w_tex, void* workspace, void* stream_) {
    if (!rgba || !gt || !mask_gt || !stats || !per_image || !loss || !workspace || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const unsigned gx = lh_slots(HW);
    T* slots = (T*)workspace;
    launch(k_losshead_partial<T, true>, dim3(gx, B), LH_THREADS, 0, st, rgba, gt, mask_gt, slots, HW);
    launch(k_losshead_sum<T>, (3 * B + 127) / 128, 128, 0, st, slots, stats, B, (int)gx);
    launch(k_losshead_finalize<T>, 1, 32, 0, st, stats, per_image, loss, B, T(1) / (T(3) * (T)HW), w_iou, w_tex);
    return (int)cudaGetLastError();
}
template <typename T>
static int loss_head_backward(const T* rgba, const T* gt, const T* mask_gt, const T* stats, const T* grad_loss, T* grad_rgba,
                              int32_t B, int64_t HW, T w_iou, T w_tex, void* stream_) {
    if (!rgba || !gt || !mask_gt || !stats || !grad_loss || !grad_rgba || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    const unsigned gx = (unsigned)std::min<int64_t>((HW + 255) / 256, 1024);
    launch(k_losshead_bwd<T>, dim3(gx, B), 256, 0, (cudaStream_t)stream_, rgba, gt, mask_gt, stats, grad_loss, grad_rgba, HW,
           B, T(1) / (T(3) * (T)HW), w_iou, w_tex);
    return (int)cudaGetLastError();
}

// part_matching_loss head.  Workspace: stats [B][PH_STATS] T | slots [B][nslot][PH_SLOT] T | idx [B][PH_IDX] int32 |
// slot indices [B][nslot][PH_MAX] int32.  The forward fills it; the backward reads stats and idx.
static inline bool ph_too_large(int32_t B, int32_t H) { return B > 65535 || (int64_t)H * H > INT_MAX; }
static inline int64_t ph_slots(int32_t H) { return ((int64_t)H * H + PH_PER_CTA - 1) / PH_PER_CTA; }
template <typename T>
static size_t part_head_workspace_bytes(int32_t B, int32_t H) {
    if (B <= 0 || H <= 0 || ph_too_large(B, H)) return 0;
    const int64_t ns = ph_slots(H);
    return (size_t)B * ((size_t)(ns + 1) * PH_STATS * sizeof(T) + (size_t)(PH_IDX + ns * PH_MAX) * sizeof(int32_t));
}
template <typename T>
static bool ph_misaligned(const void* p) { return ((uintptr_t)p & (sizeof(T) - 1)) != 0; }
// validates the arguments the forward and backward share and fills `in`
template <typename T>
static int part_head_check(const T* const* maps, const int64_t* map_bstrides, const T* c0, int64_t c0_bstride,
                           const T* part_segs, int64_t segs_bstride, const T* weights, const void* workspace, int32_t B,
                           int32_t H, int32_t kld, PartHeadIn<T>& in) {
    if (!maps || !map_bstrides || !c0 || !part_segs || !weights || !workspace || B <= 0 || H <= 0 || (kld != 0 && kld != 1) ||
        c0_bstride < 0 || segs_bstride < 0 || ph_misaligned<T>(c0) || ph_misaligned<T>(part_segs) ||
        ph_misaligned<T>(weights) || ph_misaligned<T>(workspace))
        return UMR_ERR_BAD_ARG;
    for (int k = 0; k < 4; ++k) {
        if (!maps[k] || map_bstrides[k] < 0 || ph_misaligned<T>(maps[k])) return UMR_ERR_BAD_ARG;
        in.map[k] = maps[k];
        in.map_bs[k] = map_bstrides[k];
    }
    if (ph_too_large(B, H)) return UMR_ERR_TOO_LARGE;
    in.c0 = c0;
    in.c0_bs = c0_bstride;
    in.q = part_segs;
    in.q_bs = segs_bstride;
    return UMR_OK;
}
template <typename T>
static int part_head_forward(const T* const* maps, const int64_t* map_bstrides, const T* c0, int64_t c0_bstride,
                             const T* part_segs, int64_t segs_bstride, const T* weights, T* terms, int32_t B, int32_t H,
                             int32_t kld, void* workspace, void* stream_) {
    PartHeadIn<T> in;
    if (!terms || ph_misaligned<T>(terms)) return UMR_ERR_BAD_ARG;
    const int rc = part_head_check(maps, map_bstrides, c0, c0_bstride, part_segs, segs_bstride, weights, workspace, B, H, kld,
                                   in);
    if (rc != UMR_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream_;
    const int ns = (int)ph_slots(H);
    T* stats = (T*)workspace;
    T* slots = stats + (size_t)B * PH_STATS;
    int32_t* idx = (int32_t*)(slots + (size_t)B * ns * PH_SLOT);
    int32_t* slot_idx = idx + (size_t)B * PH_IDX;
    launch(k_part_head_partial<T>, dim3(ns, B), PH_THREADS, 0, st, in, slots, slot_idx, H, kld);
    launch(k_part_head_finalize<T>, B, 64, 0, st, slots, slot_idx, stats, idx, terms, ns, kld);
    if (!kld) {
        launch(k_part_head_mse<T>, dim3(ns, B), PH_THREADS, 0, st, in, weights, stats, slots, H);
        launch(k_part_head_mse_finalize<T>, B, 32, 0, st, slots, stats, terms, ns);
    }
    return (int)cudaGetLastError();
}
template <typename T>
static int part_head_backward(const T* const* maps, const int64_t* map_bstrides, const T* c0, int64_t c0_bstride,
                              const T* part_segs, int64_t segs_bstride, const T* weights, const void* workspace,
                              const T* grad_terms, T* grad_maps, int32_t B, int32_t H, int32_t kld, void* stream_) {
    PartHeadIn<T> in;
    if (!grad_terms || !grad_maps || ph_misaligned<T>(grad_terms) || ph_misaligned<T>(grad_maps)) return UMR_ERR_BAD_ARG;
    const int rc = part_head_check(maps, map_bstrides, c0, c0_bstride, part_segs, segs_bstride, weights, workspace, B, H, kld,
                                   in);
    if (rc != UMR_OK) return rc;
    const int64_t HW = (int64_t)H * H;
    const T* stats = (const T*)workspace;
    const int32_t* idx = (const int32_t*)(stats + (size_t)B * PH_STATS + (size_t)B * ph_slots(H) * PH_SLOT);
    const unsigned gx = (unsigned)std::min<int64_t>((HW + 255) / 256, 1024);
    launch(k_part_head_bwd<T>, dim3(gx, B), 256, 0, (cudaStream_t)stream_, in, weights, stats, idx, grad_terms, grad_maps, H,
           kld);
    return (int)cudaGetLastError();
}
// losses_f64.cu: the double instantiations, reached through the dtype argument of the entry points in losses.cu
int part_head_forward_f64(const void* const* maps, const int64_t* map_bstrides, const void* c0, int64_t c0_bstride,
                          const void* part_segs, int64_t segs_bstride, const void* weights, void* terms, int32_t B, int32_t H,
                          int32_t kld, void* workspace, void* stream_);
int part_head_backward_f64(const void* const* maps, const int64_t* map_bstrides, const void* c0, int64_t c0_bstride,
                           const void* part_segs, int64_t segs_bstride, const void* weights, const void* workspace,
                           const void* grad_terms, void* grad_maps, int32_t B, int32_t H, int32_t kld, void* stream_);

}  // namespace umr
