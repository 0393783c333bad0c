// losses.cu -- geometric-loss kernels around the rasteriser (sm_90a): bilinear texture-flow
// sampler, silhouette IoU, O(N*M) chamfer, texture-cycle.  All HBM/L2-bound gather/reduce work; no
// tensor cores (none of these is a dense contraction -- chamfer's inner dimension is 2 or 3).
//
// Reference entry points replaced (file:line under the reference tree):
//   nnutils/geom_utils.py:41-59 `sample_textures`, nnutils/loss_utils.py:59-64 (texture_dt_loss)
//   nnutils/loss_utils.py:41-48 `neg_iou_loss`
//   nnutils/chamfer_python.py:43-64 `distChamfer`
//   nnutils/loss_utils.py:152-182 `TexCycle.forward`
//
// The reductions and the chamfer backward also have deterministic variants (DET template parameter / gather kernels,
// `*_deterministic` entry points at the end of this file; DESIGN.md §2): no atomics reach their outputs.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <climits>

#include "common.cuh"
#include "umr_b200.h"

namespace umr {

// ---------------------------------------------------------------------------------------------
// bilinear sampler: grid_sample(bilinear, zeros padding) with the torch-1.1 coordinate map
// (== align_corners=True): ix = (x + 1) / 2 * (W - 1).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool inb(int x, int y, int W, int H) { return x >= 0 && x < W && y >= 0 && y < H; }

template <int C>
__global__ void __launch_bounds__(256) k_sample_fwd(const float* __restrict__ image, const float2* __restrict__ flow,
                                                    float* __restrict__ out, int H, int W, int N) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= N) return;
    const float2 xy = __ldg(flow + (size_t)b * N + n);
    const float ix = ((xy.x + 1.f) / 2.f) * (float)(W - 1);
    const float iy = ((xy.y + 1.f) / 2.f) * (float)(H - 1);
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
    const float nw = ((float)x1 - ix) * ((float)y1 - iy), ne = (ix - (float)x0) * ((float)y1 - iy);
    const float sw = ((float)x1 - ix) * (iy - (float)y0), se = (ix - (float)x0) * (iy - (float)y0);
    const bool v00 = inb(x0, y0, W, H), v10 = inb(x1, y0, W, H), v01 = inb(x0, y1, W, H), v11 = inb(x1, y1, W, H);
    const float* img = image + (size_t)b * C * H * W;
    float* o = out + ((size_t)b * N + n) * C;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const float* p = img + (size_t)c * H * W;
        float acc = 0.f;
        if (v00) acc += __ldg(p + (size_t)y0 * W + x0) * nw;
        if (v10) acc += __ldg(p + (size_t)y0 * W + x1) * ne;
        if (v01) acc += __ldg(p + (size_t)y1 * W + x0) * sw;
        if (v11) acc += __ldg(p + (size_t)y1 * W + x1) * se;
        o[c] = acc;
    }
}

template <int C>
__global__ void __launch_bounds__(256) k_sample_bwd(const float* __restrict__ image, const float2* __restrict__ flow,
                                                    const float* __restrict__ gout, float2* __restrict__ gflow,
                                                    float* __restrict__ gimage, int H, int W, int N) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= N) return;
    const float2 xy = __ldg(flow + (size_t)b * N + n);
    const float ix = ((xy.x + 1.f) / 2.f) * (float)(W - 1);
    const float iy = ((xy.y + 1.f) / 2.f) * (float)(H - 1);
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
    const float wx1 = (float)x1 - ix, wx0 = ix - (float)x0, wy1 = (float)y1 - iy, wy0 = iy - (float)y0;
    const bool v00 = inb(x0, y0, W, H), v10 = inb(x1, y0, W, H), v01 = inb(x0, y1, W, H), v11 = inb(x1, y1, W, H);
    const float* img = image + (size_t)b * C * H * W;
    const float* go = gout + ((size_t)b * N + n) * C;
    float gix = 0.f, giy = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const float* p = img + (size_t)c * H * W;
        const float g = __ldg(go + c);
        const float a00 = v00 ? __ldg(p + (size_t)y0 * W + x0) : 0.f;
        const float a10 = v10 ? __ldg(p + (size_t)y0 * W + x1) : 0.f;
        const float a01 = v01 ? __ldg(p + (size_t)y1 * W + x0) : 0.f;
        const float a11 = v11 ? __ldg(p + (size_t)y1 * W + x1) : 0.f;
        gix += g * ((a10 - a00) * wy1 + (a11 - a01) * wy0);
        giy += g * ((a01 - a00) * wx1 + (a11 - a10) * wx0);
        if (gimage != nullptr) {
            float* q = gimage + ((size_t)b * C + c) * H * W;
            if (v00) atomicAdd(q + (size_t)y0 * W + x0, g * wx1 * wy1);
            if (v10) atomicAdd(q + (size_t)y0 * W + x1, g * wx0 * wy1);
            if (v01) atomicAdd(q + (size_t)y1 * W + x0, g * wx1 * wy0);
            if (v11) atomicAdd(q + (size_t)y1 * W + x1, g * wx0 * wy0);
        }
    }
    gflow[(size_t)b * N + n] = make_float2(gix * ((float)(W - 1) / 2.f), giy * ((float)(H - 1) / 2.f));
}

// Deterministic image gradient of the sampler.  Samples are keyed by the cell (y0, x0) of their top-left corner,
// shifted by one so that every cell with an in-bounds corner is in [0, H] x [0, W]: key = b * (H+1)(W+1) +
// (y0+1)(W+1) + (x0+1), from k_sample_bwd's own expressions (so a non-finite coordinate reaches the same pixels);
// a sample with no in-bounds corner gets the drop key B * (H+1)(W+1).
__global__ void __launch_bounds__(256) k_sample_cells(const float2* __restrict__ flow, int32_t* __restrict__ cells, int B,
                                                      int H, int W, int N) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= N) return;
    const float2 xy = __ldg(flow + (size_t)b * N + n);
    const float ix = ((xy.x + 1.f) / 2.f) * (float)(W - 1);
    const float iy = ((xy.y + 1.f) / 2.f) * (float)(H - 1);
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
    const bool any = inb(x0, y0, W, H) || inb(x1, y0, W, H) || inb(x0, y1, W, H) || inb(x1, y1, W, H);
    const int cell = (H + 1) * (W + 1);
    cells[(size_t)b * N + n] = any ? b * cell + (y0 + 1) * (W + 1) + (x0 + 1) : B * cell;
}

// grad_image[b][c][y][x], one thread per (image, pixel): the terms of the four roles the pixel plays, in the order
// 00 of cell (y,x), 10 of cell (y,x-1), 01 of cell (y-1,x), 11 of cell (y-1,x-1); within a role the samples of the
// cell table (rowptr [B(H+1)(W+1)+1], samples: flat sample indices b * N + n) in ascending order.  Each term is
// k_sample_bwd's product, rounded as there.  A pixel no sample touches gets 0.
template <int C>
__global__ void __launch_bounds__(256) k_sample_bwd_image_gather(const float2* __restrict__ flow, const float* __restrict__ gout,
                                                                 const int32_t* __restrict__ rowptr,
                                                                 const int32_t* __restrict__ samples,
                                                                 float* __restrict__ gimage, int H, int W) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (p >= H * W) return;
    const int y = p / W, x = p - y * W;
    const size_t c0 = (size_t)b * (H + 1) * (W + 1);
    const size_t cell[4] = {c0 + (size_t)(y + 1) * (W + 1) + (x + 1), c0 + (size_t)(y + 1) * (W + 1) + x,
                            c0 + (size_t)y * (W + 1) + (x + 1), c0 + (size_t)y * (W + 1) + x};
    float acc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] = 0.f;
#pragma unroll
    for (int role = 0; role < 4; ++role) {
        const int k1 = __ldg(rowptr + cell[role] + 1);
        for (int k = __ldg(rowptr + cell[role]); k < k1; ++k) {
            const int s = __ldg(samples + k);
            const float2 xy = __ldg(flow + s);
            const float ix = ((xy.x + 1.f) / 2.f) * (float)(W - 1);
            const float iy = ((xy.y + 1.f) / 2.f) * (float)(H - 1);
            const float fx = floorf(ix), fy = floorf(iy);
            const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
            const float wx1 = (float)x1 - ix, wx0 = ix - (float)x0, wy1 = (float)y1 - iy, wy0 = iy - (float)y0;
            const float wa = (role & 1) ? wx0 : wx1, wb = (role & 2) ? wy0 : wy1;
            const float* go = gout + (size_t)s * C;
#pragma unroll
            for (int c = 0; c < C; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(__fmul_rn(__ldg(go + c), wa), wb));
        }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) gimage[((size_t)b * C + c) * H * W + p] = acc[c];
}

// ---------------------------------------------------------------------------------------------
// IoU
// ---------------------------------------------------------------------------------------------
constexpr int IOU_THREADS = 512;
constexpr int IOU_PER_CTA = IOU_THREADS * 4 * 8;  // elements per CTA

// DET: `inter` / `uni` are the workspace slots [B][gridDim.x]; the CTA stores its partial instead of adding it
template <bool DET>
__global__ void __launch_bounds__(IOU_THREADS) k_iou_partial(const float* __restrict__ p, const float* __restrict__ t,
                                                             float* __restrict__ inter, float* __restrict__ uni,
                                                             int64_t N, int64_t p_bstride) {
    const int b = blockIdx.y;
    const float* pb = p + (size_t)b * p_bstride;
    const float* tb = t + (size_t)b * N;
    const int64_t begin = (int64_t)blockIdx.x * IOU_PER_CTA;
    const int64_t end = min(N, begin + IOU_PER_CTA);
    float si = 0.f, su = 0.f;
    const bool vec = ((N & 3) == 0) && ((((uintptr_t)pb | (uintptr_t)tb) & 15) == 0);
    if (vec) {
        for (int64_t i = begin + (int64_t)threadIdx.x * 4; i < end; i += IOU_THREADS * 4) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(pb + i));
            const float4 c = __ldg(reinterpret_cast<const float4*>(tb + i));
            si += a.x * c.x; su += a.x + c.x - a.x * c.x;
            si += a.y * c.y; su += a.y + c.y - a.y * c.y;
            si += a.z * c.z; su += a.z + c.z - a.z * c.z;
            si += a.w * c.w; su += a.w + c.w - a.w * c.w;
        }
    } else {
        for (int64_t i = begin + threadIdx.x; i < end; i += IOU_THREADS) {
            const float a = __ldg(pb + i), c = __ldg(tb + i);
            si += a * c; su += a + c - a * c;
        }
    }
    __shared__ float s_i[IOU_THREADS / 32], s_u[IOU_THREADS / 32];
    si = warp_sum(si); su = warp_sum(su);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s_i[warp] = si; s_u[warp] = su; }
    __syncthreads();
    if (warp == 0) {
        si = lane < IOU_THREADS / 32 ? s_i[lane] : 0.f;
        su = lane < IOU_THREADS / 32 ? s_u[lane] : 0.f;
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
__global__ void k_iou_finalize_det(const float* __restrict__ si, const float* __restrict__ su, float* __restrict__ inter,
                                   float* __restrict__ uni, float* __restrict__ loss, int B, int nslot) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float I = sum_ascending(si + (size_t)b * nslot, nslot);
    const float u = sum_ascending(su + (size_t)b * nslot, nslot) + 1e-6f;
    inter[b] = I;
    uni[b] = u;
    loss[b] = 1.f - I / u;
}
__global__ void k_iou_finalize(const float* __restrict__ inter, float* __restrict__ uni, float* __restrict__ loss, int B) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float u = uni[b] + 1e-6f;
    uni[b] = u;
    loss[b] = 1.f - inter[b] / u;
}
__global__ void __launch_bounds__(256) k_iou_bwd(const float* __restrict__ t, const float* __restrict__ inter,
                                                 const float* __restrict__ uni, const float* __restrict__ gl,
                                                 float* __restrict__ gp, int64_t N) {
    const int b = blockIdx.y;
    const float I = __ldg(inter + b), U = __ldg(uni + b), g = __ldg(gl + b);
    const float k = -g / (U * U);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
        const float tt = __ldg(t + (size_t)b * N + i);
        gp[(size_t)b * N + i] = k * (tt * U - I * (1.f - tt));
    }
}

// ---------------------------------------------------------------------------------------------
// chamfer: one warp per query point, lanes stride over the key set; lexicographic (value, index)
// minimum => lowest index wins ties, like torch.min.
// ---------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(256) k_chamfer_nn(const float* __restrict__ q, const float* __restrict__ k,
                                                    float* __restrict__ dist, int32_t* __restrict__ idx, int NQ, int NK) {
    const int lane = threadIdx.x & 31;
    const int qi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int b = blockIdx.y;
    if (qi >= NQ) return;
    const float* qp = q + ((size_t)b * NQ + qi) * D;
    // Defined fp32 operation order (never contracted to FMA, whatever the compile flags):
    //   |p|^2 = ((p0*p0 + p1*p1) + p2*p2),  a.b = ((a0*b0 + a1*b1) + a2*b2),  P = (|q|^2 + |k|^2) - 2*(q.k)
    // -- chamfer_python.py:58-63 with every product and sum rounded once.  oracle/losses.py::dist_chamfer_np
    // restates exactly this sequence, so distances AND argmins are bit-exact against it.
    float qv[D];
#pragma unroll
    for (int d = 0; d < D; ++d) { qv[d] = __ldg(qp + d); }
    float qq = __fmul_rn(qv[0], qv[0]);
#pragma unroll
    for (int d = 1; d < D; ++d) qq = __fadd_rn(qq, __fmul_rn(qv[d], qv[d]));
    float best = __int_as_float(0x7f800000);  // +inf
    int bi = 0x7fffffff;
    const float* kb = k + (size_t)b * NK * D;
    for (int j = lane; j < NK; j += 32) {
        float kv[D];
#pragma unroll
        for (int d = 0; d < D; ++d) kv[d] = __ldg(kb + (size_t)j * D + d);
        float kk = __fmul_rn(kv[0], kv[0]), zz = __fmul_rn(qv[0], kv[0]);
#pragma unroll
        for (int d = 1; d < D; ++d) {
            kk = __fadd_rn(kk, __fmul_rn(kv[d], kv[d]));
            zz = __fadd_rn(zz, __fmul_rn(qv[d], kv[d]));
        }
        const float P = __fsub_rn(__fadd_rn(qq, kk), __fmul_rn(2.f, zz));  // chamfer_python.py:63 expanded form
        if (P < best) { best = P; bi = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) {
        dist[(size_t)b * NQ + qi] = best;
        idx[(size_t)b * NQ + qi] = bi;
    }
}

template <int D>
__global__ void __launch_bounds__(256) k_chamfer_bwd(const float* __restrict__ q, const float* __restrict__ k,
                                                     const int32_t* __restrict__ idx, const float* __restrict__ gd,
                                                     float* __restrict__ gq, float* __restrict__ gk, int NQ, int NK) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (i >= NQ) return;
    const float g = __ldg(gd + (size_t)b * NQ + i);
    const int j = __ldg(idx + (size_t)b * NQ + i);
#pragma unroll
    for (int d = 0; d < D; ++d) {
        const float diff = __ldg(q + ((size_t)b * NQ + i) * D + d) - __ldg(k + ((size_t)b * NK + j) * D + d);
        atomicAdd(gq + ((size_t)b * NQ + i) * D + d, 2.f * g * diff);
        atomicAdd(gk + ((size_t)b * NK + j) * D + d, -2.f * g * diff);
    }
}

// Deterministic backward as a gather, one warp per output point i of `q` (no atomics, no workspace):
//   gq[i] = own term (gd_q[i], idx_q[i]) + sum over j with idx_k[j] == i of the j terms (gd_k[j])
// with k_chamfer_bwd's per-term arithmetic.  Lane l owns the j = l (mod 32) in ascending order; the ballot skips the
// 32-wide chunks with no match; the lanes' sums meet in warp_sum's fixed tree.  gd_q / gd_k may be NULL (no term).
template <int D>
__global__ void __launch_bounds__(256) k_chamfer_bwd_gather(const float* __restrict__ q, const float* __restrict__ k,
                                                            const int32_t* __restrict__ idx_q, const int32_t* __restrict__ idx_k,
                                                            const float* __restrict__ gd_q, const float* __restrict__ gd_k,
                                                            float* __restrict__ gq, int NQ, int NK) {
    const int lane = threadIdx.x & 31;
    const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int b = blockIdx.y;
    if (i >= NQ) return;
    float qv[D], acc[D];
#pragma unroll
    for (int d = 0; d < D; ++d) { qv[d] = __ldg(q + ((size_t)b * NQ + i) * D + d); acc[d] = 0.f; }
    if (gd_k != nullptr) {
        const int32_t* ik = idx_k + (size_t)b * NK;
        for (int j0 = 0; j0 < NK; j0 += 32) {
            const int j = j0 + lane;
            const bool hit = j < NK && __ldg(ik + j) == i;
            if (__ballot_sync(0xffffffffu, hit) == 0u) continue;
            if (hit) {
                const float g = __ldg(gd_k + (size_t)b * NK + j);
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    const float diff = __ldg(k + ((size_t)b * NK + j) * D + d) - qv[d];
                    acc[d] += -2.f * g * diff;
                }
            }
        }
#pragma unroll
        for (int d = 0; d < D; ++d) acc[d] = warp_sum(acc[d]);
    }
    if (lane != 0) return;
    float own[D];
#pragma unroll
    for (int d = 0; d < D; ++d) own[d] = 0.f;
    if (gd_q != nullptr) {
        const float g = __ldg(gd_q + (size_t)b * NQ + i);
        const int j = __ldg(idx_q + (size_t)b * NQ + i);
#pragma unroll
        for (int d = 0; d < D; ++d) own[d] = 2.f * g * (qv[d] - __ldg(k + ((size_t)b * NK + j) * D + d));
    }
#pragma unroll
    for (int d = 0; d < D; ++d) gq[((size_t)b * NQ + i) * D + d] = own[d] + acc[d];
}

// ---------------------------------------------------------------------------------------------
// texture cycle
// ---------------------------------------------------------------------------------------------
// Visibility bitmap of the face-id plane (replaces the per-sample torch.unique + host sync of loss_utils.py:174-179).
// Almost every pixel carries the background id or the id of its neighbour: a thread only touches the bitmap when the id
// differs from the previous pixel it saw AND the byte is not set yet (test-before-set through L2), so the plane is
// streamed at HBM speed instead of serialising millions of stores on a handful of bytes.
__global__ void __launch_bounds__(256) k_visible(const float* __restrict__ ids, uint8_t* __restrict__ vis, int F, int64_t P) {
    const int b = blockIdx.y;
    const float* src = ids + (size_t)b * P;
    uint8_t* v = vis + (size_t)b * F;
    int last = INT_MIN;
    auto mark = [&](float id) {
        int f = (int)id;
        if (f == last) return;
        last = f;
        if (f < 0) f += F;  // python negative index: -1 (background) marks the LAST face (loss_utils.py:175-177)
        if (f >= 0 && f < F && __ldcg(v + f) == 0) v[f] = 1;
    };
    const bool vec = ((P & 3) == 0) && ((((uintptr_t)src) & 15) == 0);
    if (vec) {
        const int64_t n4 = P >> 2;
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(src) + i);
            mark(q.x); mark(q.y); mark(q.z); mark(q.w);
        }
    } else {
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < P; i += (int64_t)gridDim.x * blockDim.x)
            mark(__ldg(src + i));
    }
}
// DET: `loss` is the workspace slot array [gridDim.x]; every CTA stores its scaled partial
template <bool DET>
__global__ void __launch_bounds__(256) k_texcycle_fwd(const float2* __restrict__ flow, const float2* __restrict__ prob,
                                                      const uint8_t* __restrict__ vis, float* __restrict__ loss, int n,
                                                      int T2, float scale) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;  // (b, f)
    float acc = 0.f;
    if (i < n && vis[i]) {
        float sx = 0.f, sy = 0.f;
        for (int t = 0; t < T2; ++t) {
            const float2 v = __ldg(flow + (size_t)i * T2 + t);
            sx += v.x; sy += v.y;
        }
        const float2 p = __ldg(prob + i);
        const float dx = sx / (float)T2 - p.x, dy = sy / (float)T2 - p.y;
        acc = dx * dx + dy * dy;
    }
    acc = warp_sum(acc);
    __shared__ float s[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s[warp] = acc;
    __syncthreads();
    if (warp == 0) {
        acc = lane < 8 ? s[lane] : 0.f;
        acc = warp_sum(acc);
        if (DET) {
            if (lane == 0) loss[blockIdx.x] = acc * scale;
        } else {
            if (lane == 0 && acc != 0.f) atomicAdd(loss, acc * scale);
        }
    }
}
// deterministic finalize of a per-row reduction: out[r] = the row's n slots summed in ascending order
__global__ void k_sum_slot_rows(const float* __restrict__ slots, float* __restrict__ out, int rows, int n) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < rows) out[r] = sum_ascending(slots + (size_t)r * n, n);
}
__global__ void __launch_bounds__(256) k_texcycle_bwd(const float2* __restrict__ flow, const float2* __restrict__ prob,
                                                      const uint8_t* __restrict__ vis, const float* __restrict__ gl,
                                                      float2* __restrict__ gflow, int n, int T2, float scale) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float gx = 0.f, gy = 0.f;
    if (vis[i]) {
        float sx = 0.f, sy = 0.f;
        for (int t = 0; t < T2; ++t) {
            const float2 v = __ldg(flow + (size_t)i * T2 + t);
            sx += v.x; sy += v.y;
        }
        const float2 p = __ldg(prob + i);
        const float k = 2.f * __ldg(gl) * scale / (float)T2;
        gx = k * (sx / (float)T2 - p.x);
        gy = k * (sy / (float)T2 - p.y);
    }
    for (int t = 0; t < T2; ++t) gflow[(size_t)i * T2 + t] = make_float2(gx, gy);
}


// ---------------------------------------------------------------------------------------------
// masked L1 texture loss: nnutils/loss_utils.py:103-116 `texture_loss_masks`
//   per image: sum_{c,h,w} | pred[c]*mask_pred - gt[c]*mask_gt | / (C*H*W)
// pred / mask_pred may be strided views of the renderer's RGBA output (batch strides passed in).
// ---------------------------------------------------------------------------------------------
constexpr int ML1_THREADS = 256;
constexpr int ML1_PER_CTA = ML1_THREADS * 8;  // pixels per CTA

// DET: `loss` is the workspace slot array [B][gridDim.x]; every CTA stores its scaled partial
template <int C, bool DET>
__global__ void __launch_bounds__(ML1_THREADS) k_masked_l1_fwd(const float* __restrict__ pred, int64_t pred_bs,
                                                              const float* __restrict__ mpred, int64_t mpred_bs,
                                                              const float* __restrict__ gt, const float* __restrict__ mgt,
                                                              float* __restrict__ loss, int64_t HW, float inv_n) {
    const int b = blockIdx.y;
    const float* p = pred + (size_t)b * pred_bs;
    const float* mp = mpred + (size_t)b * mpred_bs;
    const float* g = gt + (size_t)b * C * HW;
    const float* mg = mgt + (size_t)b * HW;
    const int64_t begin = (int64_t)blockIdx.x * ML1_PER_CTA;
    const int64_t end = min(HW, begin + ML1_PER_CTA);
    float acc = 0.f;
    for (int64_t i = begin + threadIdx.x; i < end; i += ML1_THREADS) {
        const float a = __ldg(mp + i), m = __ldg(mg + i);
#pragma unroll
        for (int c = 0; c < C; ++c) acc += fabsf(__ldg(p + (size_t)c * HW + i) * a - __ldg(g + (size_t)c * HW + i) * m);
    }
    acc = warp_sum(acc);
    __shared__ float s[ML1_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s[warp] = acc;
    __syncthreads();
    if (warp == 0) {
        acc = lane < ML1_THREADS / 32 ? s[lane] : 0.f;
        acc = warp_sum(acc);
        if (DET) {
            if (lane == 0) loss[(size_t)b * gridDim.x + blockIdx.x] = acc * inv_n;
        } else {
            if (lane == 0) atomicAdd(loss + b, acc * inv_n);
        }
    }
}

template <int C>
__global__ void __launch_bounds__(ML1_THREADS) k_masked_l1_bwd(const float* __restrict__ pred, int64_t pred_bs,
                                                              const float* __restrict__ mpred, int64_t mpred_bs,
                                                              const float* __restrict__ gt, const float* __restrict__ mgt,
                                                              const float* __restrict__ gl, float* __restrict__ gpred,
                                                              float* __restrict__ gmask, int64_t HW, float inv_n) {
    const int b = blockIdx.y;
    const float* p = pred + (size_t)b * pred_bs;
    const float* mp = mpred + (size_t)b * mpred_bs;
    const float* g = gt + (size_t)b * C * HW;
    const float* mg = mgt + (size_t)b * HW;
    const float k = __ldg(gl + b) * inv_n;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (int64_t)gridDim.x * blockDim.x) {
        const float a = __ldg(mp + i), m = __ldg(mg + i);
        float gm = 0.f;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const float pv = __ldg(p + (size_t)c * HW + i);
            const float d = pv * a - __ldg(g + (size_t)c * HW + i) * m;
            const float sg = d > 0.f ? k : (d < 0.f ? -k : 0.f);  // torch: grad * sign(d), sign(0) = 0
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
template <bool DET>
__global__ void __launch_bounds__(LH_THREADS) k_losshead_partial(const float* __restrict__ rgba, const float* __restrict__ gt,
                                                                const float* __restrict__ mgt, float* __restrict__ acc,
                                                                int64_t HW) {
    const int b = blockIdx.y;
    const float* im = rgba + (size_t)b * 4 * HW;
    const float* g = gt + (size_t)b * 3 * HW;
    const float* mg = mgt + (size_t)b * HW;
    const int64_t begin = (int64_t)blockIdx.x * LH_PER_CTA;
    const int64_t end = min(HW, begin + LH_PER_CTA);
    float si = 0.f, su = 0.f, sl = 0.f;
    for (int64_t i = begin + threadIdx.x; i < end; i += LH_THREADS) {
        const float a = __ldg(im + 3 * HW + i), m = __ldg(mg + i);
        si += a * m;
        su += a + m - a * m;
#pragma unroll
        for (int c = 0; c < 3; ++c) sl += fabsf(__ldg(im + (size_t)c * HW + i) * a - __ldg(g + (size_t)c * HW + i) * m);
    }
    si = warp_sum(si); su = warp_sum(su); sl = warp_sum(sl);
    __shared__ float s[3][LH_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s[0][warp] = si; s[1][warp] = su; s[2][warp] = sl; }
    __syncthreads();
    if (warp == 0) {
        si = lane < LH_THREADS / 32 ? s[0][lane] : 0.f;
        su = lane < LH_THREADS / 32 ? s[1][lane] : 0.f;
        sl = lane < LH_THREADS / 32 ? s[2][lane] : 0.f;
        si = warp_sum(si); su = warp_sum(su); sl = warp_sum(sl);
        if (DET) {
            if (lane == 0) {
                float* o = acc + ((size_t)b * gridDim.x + blockIdx.x) * 3;
                o[0] = si; o[1] = su; o[2] = sl;
            }
        } else {
            if (lane == 0) { atomicAdd(acc + b * 3 + 0, si); atomicAdd(acc + b * 3 + 1, su); atomicAdd(acc + b * 3 + 2, sl); }
        }
    }
}
// deterministic pre-pass of k_losshead_finalize: stats[b][k] = image b's slots [nslot][3] summed in ascending CTA order
__global__ void k_losshead_sum_det(const float* __restrict__ slots, float* __restrict__ stats, int B, int nslot) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;  // (b, k)
    if (r >= B * 3) return;
    const float* s = slots + (size_t)(r / 3) * nslot * 3 + r % 3;
    float t = 0.f;
    for (int c = 0; c < nslot; ++c) t += s[(size_t)c * 3];
    stats[r] = t;
}
// one warp: stats[b] = (I, U + 1e-6, per-image L1 mean); per_image[b] = (1 - I/U, L1 mean); loss = weighted batch means
__global__ void k_losshead_finalize(float* __restrict__ acc, float* __restrict__ per_image, float* __restrict__ loss, int B,
                                    float inv_n, float w_iou, float w_tex) {
    float t_iou = 0.f, t_tex = 0.f;
    for (int b = threadIdx.x; b < B; b += 32) {
        const float I = acc[b * 3 + 0], U = acc[b * 3 + 1] + 1e-6f, L = acc[b * 3 + 2] * inv_n;
        acc[b * 3 + 1] = U;
        const float li = 1.f - I / U;
        per_image[b * 2 + 0] = li;
        per_image[b * 2 + 1] = L;
        t_iou += li;
        t_tex += L;
    }
    t_iou = warp_sum(t_iou); t_tex = warp_sum(t_tex);
    if (threadIdx.x == 0) loss[0] = w_iou * (t_iou / B) + w_tex * (t_tex / B);
}
__global__ void __launch_bounds__(256) k_losshead_bwd(const float* __restrict__ rgba, const float* __restrict__ gt,
                                                      const float* __restrict__ mgt, const float* __restrict__ acc,
                                                      const float* __restrict__ gloss, float* __restrict__ grgba, int64_t HW,
                                                      int B, float inv_n, float w_iou, float w_tex) {
    const int b = blockIdx.y;
    const float* im = rgba + (size_t)b * 4 * HW;
    const float* g = gt + (size_t)b * 3 * HW;
    const float* mg = mgt + (size_t)b * HW;
    float* go = grgba + (size_t)b * 4 * HW;
    const float gl = __ldg(gloss);
    const float I = __ldg(acc + b * 3 + 0), U = __ldg(acc + b * 3 + 1);
    const float ki = -(gl * w_iou / B) / (U * U);  // d(1 - I/U)/dalpha = -(m*U - I*(1-m)) / U^2
    const float kt = gl * w_tex / B * inv_n;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (int64_t)gridDim.x * blockDim.x) {
        const float a = __ldg(im + 3 * HW + i), m = __ldg(mg + i);
        float ga = ki * (m * U - I * (1.f - m));
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float pv = __ldg(im + (size_t)c * HW + i);
            const float d = pv * a - __ldg(g + (size_t)c * HW + i) * m;
            const float sg = d > 0.f ? kt : (d < 0.f ? -kt : 0.f);  // torch: grad * sign(d), sign(0) = 0
            go[(size_t)c * HW + i] = sg * a;
            ga += sg * pv;
        }
        go[3 * HW + i] = ga;
    }
}

}  // namespace umr

using namespace umr;

#define UMR_RET_LAST() return (int)cudaGetLastError()

extern "C" int umr_bilinear_sample_forward(const float* image, const float* flow, float* out, int32_t B,
                                           int32_t C, int32_t H, int32_t W, int32_t N, void* stream_) {
    if (!image || !flow || !out || B <= 0 || C <= 0 || H <= 0 || W <= 0 || N <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const dim3 grid((N + 255) / 256, B);
    const float2* fl = reinterpret_cast<const float2*>(flow);
    count_launch();
    switch (C) {
        case 1: k_sample_fwd<1><<<grid, 256, 0, st>>>(image, fl, out, H, W, N); break;
        case 2: k_sample_fwd<2><<<grid, 256, 0, st>>>(image, fl, out, H, W, N); break;
        case 3: k_sample_fwd<3><<<grid, 256, 0, st>>>(image, fl, out, H, W, N); break;
        case 4: k_sample_fwd<4><<<grid, 256, 0, st>>>(image, fl, out, H, W, N); break;
        default: return UMR_ERR_UNSUPPORTED;
    }
    UMR_RET_LAST();
}

extern "C" int umr_bilinear_sample_backward(const float* image, const float* flow, const float* grad_out,
                                            float* grad_flow, float* grad_image, int32_t B, int32_t C,
                                            int32_t H, int32_t W, int32_t N, void* stream_) {
    if (!image || !flow || !grad_out || !grad_flow || B <= 0 || C <= 0 || H <= 0 || W <= 0 || N <= 0)
        return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    if (grad_image) {
        cudaError_t e = cudaMemsetAsync(grad_image, 0, (size_t)B * C * H * W * sizeof(float), st);
        if (e != cudaSuccess) return (int)e;
    }
    const dim3 grid((N + 255) / 256, B);
    const float2* fl = reinterpret_cast<const float2*>(flow);
    float2* gf = reinterpret_cast<float2*>(grad_flow);
    count_launch();
    switch (C) {
        case 1: k_sample_bwd<1><<<grid, 256, 0, st>>>(image, fl, grad_out, gf, grad_image, H, W, N); break;
        case 2: k_sample_bwd<2><<<grid, 256, 0, st>>>(image, fl, grad_out, gf, grad_image, H, W, N); break;
        case 3: k_sample_bwd<3><<<grid, 256, 0, st>>>(image, fl, grad_out, gf, grad_image, H, W, N); break;
        case 4: k_sample_bwd<4><<<grid, 256, 0, st>>>(image, fl, grad_out, gf, grad_image, H, W, N); break;
        default: return UMR_ERR_UNSUPPORTED;
    }
    UMR_RET_LAST();
}

extern "C" int umr_iou_forward(const float* predict, int64_t predict_bstride, const float* target, float* inter,
                               float* uni, float* loss, int32_t B, int64_t N, void* stream_) {
    if (!predict || !target || !inter || !uni || !loss || B <= 0 || N <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(inter, 0, (size_t)B * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    e = cudaMemsetAsync(uni, 0, (size_t)B * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    const dim3 grid((unsigned)((N + IOU_PER_CTA - 1) / IOU_PER_CTA), B);
    count_launch(); k_iou_partial<false><<<grid, IOU_THREADS, 0, st>>>(predict, target, inter, uni, N, predict_bstride);
    count_launch(); k_iou_finalize<<<(B + 127) / 128, 128, 0, st>>>(inter, uni, loss, B);
    UMR_RET_LAST();
}

extern "C" int umr_iou_backward(const float* target, const float* inter, const float* uni, const float* grad_loss,
                                float* grad_predict, int32_t B, int64_t N, void* stream_) {
    if (!target || !inter || !uni || !grad_loss || !grad_predict || B <= 0 || N <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const int64_t blocks = (N + 256 * 4 - 1) / (256 * 4);
    const dim3 grid((unsigned)(blocks < 1 ? 1 : (blocks > 1024 ? 1024 : blocks)), B);
    count_launch(); k_iou_bwd<<<grid, 256, 0, st>>>(target, inter, uni, grad_loss, grad_predict, N);
    UMR_RET_LAST();
}

extern "C" int umr_chamfer_forward(const float* a, const float* b, float* dist_ab, float* dist_ba, int32_t* idx_ab,
                                   int32_t* idx_ba, int32_t B, int32_t N, int32_t M, int32_t D, void* stream_) {
    if (!a || !b || !dist_ab || !dist_ba || !idx_ab || !idx_ba || B <= 0 || N <= 0 || M <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (D != 2 && D != 3) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const dim3 g1((N + 7) / 8, B), g2((M + 7) / 8, B);
    if (D == 2) {
        count_launch(); k_chamfer_nn<2><<<g1, 256, 0, st>>>(a, b, dist_ab, idx_ab, N, M);
        count_launch(); k_chamfer_nn<2><<<g2, 256, 0, st>>>(b, a, dist_ba, idx_ba, M, N);
    } else {
        count_launch(); k_chamfer_nn<3><<<g1, 256, 0, st>>>(a, b, dist_ab, idx_ab, N, M);
        count_launch(); k_chamfer_nn<3><<<g2, 256, 0, st>>>(b, a, dist_ba, idx_ba, M, N);
    }
    UMR_RET_LAST();
}

extern "C" int umr_chamfer_backward(const float* a, const float* b, const int32_t* idx_ab, const int32_t* idx_ba,
                                    const float* grad_dist_ab, const float* grad_dist_ba, float* grad_a, float* grad_b,
                                    int32_t B, int32_t N, int32_t M, int32_t D, void* stream_) {
    if (!a || !b || !grad_a || !grad_b || B <= 0 || N <= 0 || M <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (D != 2 && D != 3) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(grad_a, 0, (size_t)B * N * D * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    e = cudaMemsetAsync(grad_b, 0, (size_t)B * M * D * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    const dim3 g1((N + 255) / 256, B), g2((M + 255) / 256, B);
    if (grad_dist_ab) {
        if (!idx_ab) return UMR_ERR_BAD_ARG;
        count_launch();
        if (D == 2) k_chamfer_bwd<2><<<g1, 256, 0, st>>>(a, b, idx_ab, grad_dist_ab, grad_a, grad_b, N, M);
        else k_chamfer_bwd<3><<<g1, 256, 0, st>>>(a, b, idx_ab, grad_dist_ab, grad_a, grad_b, N, M);
    }
    if (grad_dist_ba) {
        if (!idx_ba) return UMR_ERR_BAD_ARG;
        count_launch();
        if (D == 2) k_chamfer_bwd<2><<<g2, 256, 0, st>>>(b, a, idx_ba, grad_dist_ba, grad_b, grad_a, M, N);
        else k_chamfer_bwd<3><<<g2, 256, 0, st>>>(b, a, idx_ba, grad_dist_ba, grad_b, grad_a, M, N);
    }
    UMR_RET_LAST();
}

extern "C" int umr_texcycle_forward(const float* flow, const float* prob, const float* face_ids, uint8_t* visible,
                                    float* loss, int32_t B, int32_t F, int32_t T2, int64_t P, void* stream_) {
    // face_ids == NULL: `visible` was already filled by umr_raster_visibility (its visible_faces output)
    if (!flow || !prob || !visible || !loss || B <= 0 || F <= 0 || T2 <= 0 || (face_ids && P <= 0)) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(loss, 0, sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    if (face_ids) {
        e = cudaMemsetAsync(visible, 0, (size_t)B * F, st);
        if (e != cudaSuccess) return (int)e;
        const int64_t blocks = (P / 4 + 255) / 256 + 1;
        count_launch(); k_visible<<<dim3((unsigned)(blocks > 1024 ? 1024 : blocks), B), 256, 0, st>>>(face_ids, visible, F, P);
    }
    const int n = B * F;
    const float scale = 1.f / ((float)n * 2.f);  // MSELoss mean over B*F*2 elements
    count_launch(); k_texcycle_fwd<false><<<(n + 255) / 256, 256, 0, st>>>(reinterpret_cast<const float2*>(flow),
                                                    reinterpret_cast<const float2*>(prob), visible, loss, n, T2, scale);
    UMR_RET_LAST();
}

extern "C" int umr_texcycle_backward(const float* flow, const float* prob, const uint8_t* visible, const float* grad_loss,
                                     float* grad_flow, int32_t B, int32_t F, int32_t T2, void* stream_) {
    if (!flow || !prob || !visible || !grad_loss || !grad_flow || B <= 0 || F <= 0 || T2 <= 0) return UMR_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream_;
    const int n = B * F;
    const float scale = 1.f / ((float)n * 2.f);
    count_launch(); k_texcycle_bwd<<<(n + 255) / 256, 256, 0, st>>>(reinterpret_cast<const float2*>(flow),
                                                    reinterpret_cast<const float2*>(prob), visible, grad_loss,
                                                    reinterpret_cast<float2*>(grad_flow), n, T2, scale);
    UMR_RET_LAST();
}

extern "C" int umr_masked_l1_forward(const float* pred, int64_t pred_bstride, const float* mask_pred,
                                     int64_t mask_pred_bstride, const float* gt, const float* mask_gt, float* loss,
                                     int32_t B, int32_t C, int64_t HW, void* stream_) {
    if (!pred || !mask_pred || !gt || !mask_gt || !loss || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (C != 3 && C != 1) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(loss, 0, (size_t)B * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    const dim3 grid((unsigned)((HW + ML1_PER_CTA - 1) / ML1_PER_CTA), B);
    const float inv_n = 1.f / ((float)C * (float)HW);
    count_launch();
    if (C == 3) k_masked_l1_fwd<3, false><<<grid, ML1_THREADS, 0, st>>>(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, loss, HW, inv_n);
    else k_masked_l1_fwd<1, false><<<grid, ML1_THREADS, 0, st>>>(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, loss, HW, inv_n);
    UMR_RET_LAST();
}

extern "C" int umr_masked_l1_backward(const float* pred, int64_t pred_bstride, const float* mask_pred,
                                      int64_t mask_pred_bstride, const float* gt, const float* mask_gt,
                                      const float* grad_loss, float* grad_pred, float* grad_mask_pred, int32_t B,
                                      int32_t C, int64_t HW, void* stream_) {
    if (!pred || !mask_pred || !gt || !mask_gt || !grad_loss || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (C != 3 && C != 1) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const int64_t blocks = (HW + 256 * 4 - 1) / (256 * 4);
    const dim3 grid((unsigned)(blocks < 1 ? 1 : (blocks > 1024 ? 1024 : blocks)), B);
    const float inv_n = 1.f / ((float)C * (float)HW);
    count_launch();
    if (C == 3) k_masked_l1_bwd<3><<<grid, 256, 0, st>>>(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, grad_loss, grad_pred, grad_mask_pred, HW, inv_n);
    else k_masked_l1_bwd<1><<<grid, 256, 0, st>>>(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, grad_loss, grad_pred, grad_mask_pred, HW, inv_n);
    UMR_RET_LAST();
}

extern "C" int umr_loss_head_forward(const float* rgba, const float* gt, const float* mask_gt, float* stats,
                                     float* per_image, float* loss, int32_t B, int64_t HW, float w_iou, float w_tex,
                                     void* stream_) {
    if (!rgba || !gt || !mask_gt || !stats || !per_image || !loss || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(stats, 0, (size_t)B * 3 * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    count_launch(2);
    k_losshead_partial<false><<<dim3((unsigned)((HW + LH_PER_CTA - 1) / LH_PER_CTA), B), LH_THREADS, 0, st>>>(rgba, gt, mask_gt, stats, HW);
    k_losshead_finalize<<<1, 32, 0, st>>>(stats, per_image, loss, B, 1.f / (3.f * (float)HW), w_iou, w_tex);
    return (int)cudaGetLastError();
}

extern "C" int umr_loss_head_backward(const float* rgba, const float* gt, const float* mask_gt, const float* stats,
                                      const float* grad_loss, float* grad_rgba, int32_t B, int64_t HW, float w_iou,
                                      float w_tex, void* stream_) {
    if (!rgba || !gt || !mask_gt || !stats || !grad_loss || !grad_rgba || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    count_launch();
    const unsigned gx = (unsigned)std::min<int64_t>((HW + 255) / 256, 1024);
    k_losshead_bwd<<<dim3(gx, B), 256, 0, st>>>(rgba, gt, mask_gt, stats, grad_loss, grad_rgba, HW, B,
                                                1.f / (3.f * (float)HW), w_iou, w_tex);
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// deterministic mode (include/umr_b200.h, DESIGN.md §2): each reduction CTA stores its partial into a workspace slot
// (grids sized from the shapes only, so the slot layout is fixed) and a finalize kernel sums every image's slots in
// ascending CTA order; the chamfer backward is a gather with one writer per gradient element
// ---------------------------------------------------------------------------------------------
static unsigned iou_slots(int64_t N) { return (unsigned)((N + IOU_PER_CTA - 1) / IOU_PER_CTA); }
static unsigned ml1_slots(int64_t HW) { return (unsigned)((HW + ML1_PER_CTA - 1) / ML1_PER_CTA); }
static unsigned lh_slots(int64_t HW) { return (unsigned)((HW + LH_PER_CTA - 1) / LH_PER_CTA); }

extern "C" size_t umr_iou_workspace_bytes_deterministic(int32_t B, int64_t N) {
    if (B <= 0 || N <= 0) return 0;
    return (size_t)2 * B * iou_slots(N) * sizeof(float);
}
extern "C" int umr_iou_forward_deterministic(const float* predict, int64_t predict_bstride, const float* target, float* inter,
                                             float* uni, float* loss, int32_t B, int64_t N, void* workspace, void* stream_) {
    if (!predict || !target || !inter || !uni || !loss || !workspace || B <= 0 || N <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const unsigned gx = iou_slots(N);
    float* si = (float*)workspace;
    float* su = si + (size_t)B * gx;
    count_launch(); k_iou_partial<true><<<dim3(gx, B), IOU_THREADS, 0, st>>>(predict, target, si, su, N, predict_bstride);
    count_launch(); k_iou_finalize_det<<<(B + 127) / 128, 128, 0, st>>>(si, su, inter, uni, loss, B, (int)gx);
    UMR_RET_LAST();
}

extern "C" int umr_chamfer_backward_deterministic(const float* a, const float* b, const int32_t* idx_ab, const int32_t* idx_ba,
                                                  const float* grad_dist_ab, const float* grad_dist_ba, float* grad_a,
                                                  float* grad_b, int32_t B, int32_t N, int32_t M, int32_t D, void* stream_) {
    if (!a || !b || !grad_a || !grad_b || B <= 0 || N <= 0 || M <= 0) return UMR_ERR_BAD_ARG;
    if ((grad_dist_ab && !idx_ab) || (grad_dist_ba && !idx_ba)) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (D != 2 && D != 3) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const dim3 g1((N + 7) / 8, B), g2((M + 7) / 8, B);   // one warp per output point
    count_launch(2);
    if (D == 2) {
        k_chamfer_bwd_gather<2><<<g1, 256, 0, st>>>(a, b, idx_ab, idx_ba, grad_dist_ab, grad_dist_ba, grad_a, N, M);
        k_chamfer_bwd_gather<2><<<g2, 256, 0, st>>>(b, a, idx_ba, idx_ab, grad_dist_ba, grad_dist_ab, grad_b, M, N);
    } else {
        k_chamfer_bwd_gather<3><<<g1, 256, 0, st>>>(a, b, idx_ab, idx_ba, grad_dist_ab, grad_dist_ba, grad_a, N, M);
        k_chamfer_bwd_gather<3><<<g2, 256, 0, st>>>(b, a, idx_ba, idx_ab, grad_dist_ba, grad_dist_ab, grad_b, M, N);
    }
    UMR_RET_LAST();
}

extern "C" size_t umr_texcycle_workspace_bytes_deterministic(int32_t B, int32_t F) {
    if (B <= 0 || F <= 0) return 0;
    return (size_t)(((int64_t)B * F + 255) / 256) * sizeof(float);
}
extern "C" int umr_texcycle_forward_deterministic(const float* flow, const float* prob, const float* face_ids, uint8_t* visible,
                                                  float* loss, int32_t B, int32_t F, int32_t T2, int64_t P, void* workspace,
                                                  void* stream_) {
    if (!flow || !prob || !visible || !loss || !workspace || B <= 0 || F <= 0 || T2 <= 0 || (face_ids && P <= 0))
        return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    if (face_ids) {   // the bitmap only ever receives 1s: its bytes do not depend on the order of the stores
        cudaError_t e = cudaMemsetAsync(visible, 0, (size_t)B * F, st);
        if (e != cudaSuccess) return (int)e;
        const int64_t blocks = (P / 4 + 255) / 256 + 1;
        count_launch(); k_visible<<<dim3((unsigned)(blocks > 1024 ? 1024 : blocks), B), 256, 0, st>>>(face_ids, visible, F, P);
    }
    const int n = B * F;
    const int gx = (n + 255) / 256;
    const float scale = 1.f / ((float)n * 2.f);
    float* slots = (float*)workspace;
    count_launch(); k_texcycle_fwd<true><<<gx, 256, 0, st>>>(reinterpret_cast<const float2*>(flow),
                                                             reinterpret_cast<const float2*>(prob), visible, slots, n, T2, scale);
    count_launch(); k_sum_slot_rows<<<1, 32, 0, st>>>(slots, loss, 1, gx);
    UMR_RET_LAST();
}

extern "C" size_t umr_masked_l1_workspace_bytes_deterministic(int32_t B, int64_t HW) {
    if (B <= 0 || HW <= 0) return 0;
    return (size_t)B * ml1_slots(HW) * sizeof(float);
}
extern "C" int umr_masked_l1_forward_deterministic(const float* pred, int64_t pred_bstride, const float* mask_pred,
                                                   int64_t mask_pred_bstride, const float* gt, const float* mask_gt, float* loss,
                                                   int32_t B, int32_t C, int64_t HW, void* workspace, void* stream_) {
    if (!pred || !mask_pred || !gt || !mask_gt || !loss || !workspace || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (C != 3 && C != 1) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const unsigned gx = ml1_slots(HW);
    const dim3 grid(gx, B);
    const float inv_n = 1.f / ((float)C * (float)HW);
    float* slots = (float*)workspace;
    count_launch(2);
    if (C == 3) k_masked_l1_fwd<3, true><<<grid, ML1_THREADS, 0, st>>>(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, slots, HW, inv_n);
    else k_masked_l1_fwd<1, true><<<grid, ML1_THREADS, 0, st>>>(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, slots, HW, inv_n);
    k_sum_slot_rows<<<(B + 127) / 128, 128, 0, st>>>(slots, loss, B, (int)gx);
    UMR_RET_LAST();
}

extern "C" size_t umr_loss_head_workspace_bytes_deterministic(int32_t B, int64_t HW) {
    if (B <= 0 || HW <= 0) return 0;
    return (size_t)3 * B * lh_slots(HW) * sizeof(float);
}
extern "C" int umr_loss_head_forward_deterministic(const float* rgba, const float* gt, const float* mask_gt, float* stats,
                                                   float* per_image, float* loss, int32_t B, int64_t HW, float w_iou,
                                                   float w_tex, void* workspace, void* stream_) {
    if (!rgba || !gt || !mask_gt || !stats || !per_image || !loss || !workspace || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const unsigned gx = lh_slots(HW);
    float* slots = (float*)workspace;
    count_launch(3);
    k_losshead_partial<true><<<dim3(gx, B), LH_THREADS, 0, st>>>(rgba, gt, mask_gt, slots, HW);
    k_losshead_sum_det<<<(3 * B + 127) / 128, 128, 0, st>>>(slots, stats, B, (int)gx);
    k_losshead_finalize<<<1, 32, 0, st>>>(stats, per_image, loss, B, 1.f / (3.f * (float)HW), w_iou, w_tex);
    return (int)cudaGetLastError();
}

// Sampler (include/umr_b200.h): grad_flow from k_sample_bwd itself (one writer per element, no image gradient there), the
// image gradient from a per-pixel gather over the cell table.
extern "C" int umr_bilinear_sample_cells(const float* flow, int32_t* cells, int32_t B, int32_t H, int32_t W, int32_t N,
                                         void* stream_) {
    if (!flow || !cells || B <= 0 || H <= 0 || W <= 0 || N <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535 || (int64_t)B * ((int64_t)H + 1) * ((int64_t)W + 1) > INT_MAX) return UMR_ERR_TOO_LARGE;
    count_launch(); k_sample_cells<<<dim3((N + 255) / 256, B), 256, 0, (cudaStream_t)stream_>>>(
        reinterpret_cast<const float2*>(flow), cells, B, H, W, N);
    UMR_RET_LAST();
}
extern "C" int umr_bilinear_sample_backward_deterministic(const float* image, const float* flow, const float* grad_out,
                                                          float* grad_flow, float* grad_image, int32_t B, int32_t C, int32_t H,
                                                          int32_t W, int32_t N, const int32_t* cell_rowptr,
                                                          const int32_t* cell_samples, void* stream_) {
    if (!image || !flow || !grad_out || !grad_flow || B <= 0 || C <= 0 || H <= 0 || W <= 0 || N <= 0)
        return UMR_ERR_BAD_ARG;
    if (grad_image && (!cell_rowptr || !cell_samples)) return UMR_ERR_BAD_ARG;
    if (B > 65535 || (int64_t)B * ((int64_t)H + 1) * ((int64_t)W + 1) > INT_MAX) return UMR_ERR_TOO_LARGE;
    if (C < 1 || C > 4) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const dim3 grid((N + 255) / 256, B), gpix((H * W + 255) / 256, B);
    const float2* fl = reinterpret_cast<const float2*>(flow);
    float2* gf = reinterpret_cast<float2*>(grad_flow);
    count_launch(grad_image ? 2 : 1);
    switch (C) {
        case 1: k_sample_bwd<1><<<grid, 256, 0, st>>>(image, fl, grad_out, gf, nullptr, H, W, N); break;
        case 2: k_sample_bwd<2><<<grid, 256, 0, st>>>(image, fl, grad_out, gf, nullptr, H, W, N); break;
        case 3: k_sample_bwd<3><<<grid, 256, 0, st>>>(image, fl, grad_out, gf, nullptr, H, W, N); break;
        default: k_sample_bwd<4><<<grid, 256, 0, st>>>(image, fl, grad_out, gf, nullptr, H, W, N); break;
    }
    if (grad_image) {
        switch (C) {
            case 1: k_sample_bwd_image_gather<1><<<gpix, 256, 0, st>>>(fl, grad_out, cell_rowptr, cell_samples, grad_image, H, W); break;
            case 2: k_sample_bwd_image_gather<2><<<gpix, 256, 0, st>>>(fl, grad_out, cell_rowptr, cell_samples, grad_image, H, W); break;
            case 3: k_sample_bwd_image_gather<3><<<gpix, 256, 0, st>>>(fl, grad_out, cell_rowptr, cell_samples, grad_image, H, W); break;
            default: k_sample_bwd_image_gather<4><<<gpix, 256, 0, st>>>(fl, grad_out, cell_rowptr, cell_samples, grad_image, H, W); break;
        }
    }
    UMR_RET_LAST();
}
