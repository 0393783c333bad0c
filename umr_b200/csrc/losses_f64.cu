// losses_f64.cu -- float64 loss kernels (sm_90a): double twins of the deterministic loss kernels of losses.cu,
// mesh_ops.cu (Laplacian, flatten) and vertex.cu (CorrLossChamfer), behind the `umr_*_f64` entry points of
// include/umr_b200.h.  ops.py takes them when any floating-point input of an op is float64 (DESIGN.md §10).
//
// Structure: every reduction CTA stores its partial into a workspace slot (grids sized from the shapes only) and a
// finalize kernel sums each row's slots in ascending order; every gradient element has exactly one writer (per-sample
// stores, or gathers over a transposed table built by the caller).  There are no atomics, so every output is bitwise
// reproducible for identical inputs on the same device type and library build, with no separate deterministic variant.
// Compiled with -fmad=false: each product and sum is rounded once, in the order written here.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <climits>

#include "common.cuh"
#include "umr_b200.h"

namespace umr {

// losses.cu: the face-visibility bitmap of a float face-id plane (shared with the float32 TexCycle)
__global__ void k_visible(const float* __restrict__ ids, uint8_t* __restrict__ vis, int F, int64_t P);

namespace f64 {

__device__ __forceinline__ double warp_sum(double v) {
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}
// the partials of one 256-thread CTA in a fixed tree: warp_sum per warp, then warp 0 over the 8 warp sums.  The result is
// valid in thread 0.
__device__ __forceinline__ double cta_sum(double v, double* s8) {
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s8[warp] = v;
    __syncthreads();
    v = 0.0;
    if (warp == 0) {
        v = lane < 8 ? s8[lane] : 0.0;
        v = warp_sum(v);
    }
    return v;
}
__device__ __forceinline__ double sum_ascending(const double* p, int n) {
    double t = 0.0;
    for (int k = 0; k < n; ++k) t += p[k];
    return t;
}
// out[r] = row r's n slots summed in ascending order
__global__ void k_sum_slot_rows(const double* __restrict__ slots, double* __restrict__ out, int rows, int n) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < rows) out[r] = sum_ascending(slots + (size_t)r * n, n);
}

constexpr int THREADS = 256;
constexpr int PER_CTA = THREADS * 8;  // elements (pixels) per reduction CTA of IoU, masked L1 and the loss head
static unsigned slots_of(int64_t n, int per) { return (unsigned)((n + per - 1) / per); }

// ---------------------------------------------------------------------------------------------
// bilinear sampler: grid_sample(bilinear, zeros, align_corners=True) with the coordinate map in double, as torch
// computes it for double: ix = ((x + 1) / 2) * (W - 1)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool inb(int x, int y, int W, int H) { return x >= 0 && x < W && y >= 0 && y < H; }

struct Corners {
    double wx1, wx0, wy1, wy0;
    int x0, y0;
    bool v00, v10, v01, v11;
};
__device__ __forceinline__ Corners corners(double2 xy, int H, int W) {
    Corners c;
    const double ix = ((xy.x + 1.0) / 2.0) * (double)(W - 1);
    const double iy = ((xy.y + 1.0) / 2.0) * (double)(H - 1);
    c.x0 = (int)floor(ix); c.y0 = (int)floor(iy);
    const int x1 = c.x0 + 1, y1 = c.y0 + 1;
    c.wx1 = (double)x1 - ix; c.wx0 = ix - (double)c.x0; c.wy1 = (double)y1 - iy; c.wy0 = iy - (double)c.y0;
    c.v00 = inb(c.x0, c.y0, W, H); c.v10 = inb(x1, c.y0, W, H); c.v01 = inb(c.x0, y1, W, H); c.v11 = inb(x1, y1, W, H);
    return c;
}

template <int C>
__global__ void __launch_bounds__(256) k_sample_fwd(const double* __restrict__ image, const double2* __restrict__ flow,
                                                    double* __restrict__ out, int H, int W, int N) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= N) return;
    const Corners k = corners(__ldg(flow + (size_t)b * N + n), H, W);
    const double nw = k.wx1 * k.wy1, ne = k.wx0 * k.wy1, sw = k.wx1 * k.wy0, se = k.wx0 * k.wy0;
    const double* img = image + (size_t)b * C * H * W;
    double* o = out + ((size_t)b * N + n) * C;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const double* p = img + (size_t)c * H * W;
        double acc = 0.0;
        if (k.v00) acc += __ldg(p + (size_t)k.y0 * W + k.x0) * nw;
        if (k.v10) acc += __ldg(p + (size_t)k.y0 * W + k.x0 + 1) * ne;
        if (k.v01) acc += __ldg(p + (size_t)(k.y0 + 1) * W + k.x0) * sw;
        if (k.v11) acc += __ldg(p + (size_t)(k.y0 + 1) * W + k.x0 + 1) * se;
        o[c] = acc;
    }
}

// grad_flow, one writer per sample
template <int C>
__global__ void __launch_bounds__(256) k_sample_bwd_flow(const double* __restrict__ image, const double2* __restrict__ flow,
                                                         const double* __restrict__ gout, double2* __restrict__ gflow, int H,
                                                         int W, int N) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= N) return;
    const Corners k = corners(__ldg(flow + (size_t)b * N + n), H, W);
    const double* img = image + (size_t)b * C * H * W;
    const double* go = gout + ((size_t)b * N + n) * C;
    double gix = 0.0, giy = 0.0;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const double* p = img + (size_t)c * H * W;
        const double g = __ldg(go + c);
        const double a00 = k.v00 ? __ldg(p + (size_t)k.y0 * W + k.x0) : 0.0;
        const double a10 = k.v10 ? __ldg(p + (size_t)k.y0 * W + k.x0 + 1) : 0.0;
        const double a01 = k.v01 ? __ldg(p + (size_t)(k.y0 + 1) * W + k.x0) : 0.0;
        const double a11 = k.v11 ? __ldg(p + (size_t)(k.y0 + 1) * W + k.x0 + 1) : 0.0;
        gix += g * ((a10 - a00) * k.wy1 + (a11 - a01) * k.wy0);
        giy += g * ((a01 - a00) * k.wx1 + (a11 - a10) * k.wx0);
    }
    gflow[(size_t)b * N + n] = make_double2(gix * ((double)(W - 1) / 2.0), giy * ((double)(H - 1) / 2.0));
}

// cell key of every sample (the layout of losses.cu k_sample_cells) from the double coordinate map
__global__ void __launch_bounds__(256) k_sample_cells(const double2* __restrict__ flow, int32_t* __restrict__ cells, int B,
                                                      int H, int W, int N) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= N) return;
    const Corners k = corners(__ldg(flow + (size_t)b * N + n), H, W);
    const int cell = (H + 1) * (W + 1);
    cells[(size_t)b * N + n] = (k.v00 || k.v10 || k.v01 || k.v11) ? b * cell + (k.y0 + 1) * (W + 1) + (k.x0 + 1) : B * cell;
}

// grad_image, one thread per (image, pixel): roles 00 of cell (y,x), 10 of (y,x-1), 01 of (y-1,x), 11 of (y-1,x-1), the
// samples of each cell in ascending order (losses.cu k_sample_bwd_image_gather in double)
template <int C>
__global__ void __launch_bounds__(256) k_sample_bwd_image(const double2* __restrict__ flow, const double* __restrict__ gout,
                                                          const int32_t* __restrict__ rowptr,
                                                          const int32_t* __restrict__ samples, double* __restrict__ gimage,
                                                          int H, int W) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (p >= H * W) return;
    const int y = p / W, x = p - y * W;
    const size_t c0 = (size_t)b * (H + 1) * (W + 1);
    const size_t cell[4] = {c0 + (size_t)(y + 1) * (W + 1) + (x + 1), c0 + (size_t)(y + 1) * (W + 1) + x,
                            c0 + (size_t)y * (W + 1) + (x + 1), c0 + (size_t)y * (W + 1) + x};
    double acc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] = 0.0;
#pragma unroll
    for (int role = 0; role < 4; ++role) {
        const int k1 = __ldg(rowptr + cell[role] + 1);
        for (int k = __ldg(rowptr + cell[role]); k < k1; ++k) {
            const int s = __ldg(samples + k);
            const Corners q = corners(__ldg(flow + s), H, W);
            const double wa = (role & 1) ? q.wx0 : q.wx1, wb = (role & 2) ? q.wy0 : q.wy1;
            const double* go = gout + (size_t)s * C;
#pragma unroll
            for (int c = 0; c < C; ++c) acc[c] += (__ldg(go + c) * wa) * wb;
        }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) gimage[((size_t)b * C + c) * H * W + p] = acc[c];
}

// ---------------------------------------------------------------------------------------------
// IoU: slots si / su [B][gridDim.x]
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(THREADS) k_iou_partial(const double* __restrict__ p, const double* __restrict__ t,
                                                         double* __restrict__ si, double* __restrict__ su, int64_t N,
                                                         int64_t p_bstride) {
    __shared__ double s[2][8];
    const int b = blockIdx.y;
    const double* pb = p + (size_t)b * p_bstride;
    const double* tb = t + (size_t)b * N;
    const int64_t begin = (int64_t)blockIdx.x * PER_CTA;
    const int64_t end = min(N, begin + PER_CTA);
    double i_ = 0.0, u_ = 0.0;
    for (int64_t i = begin + threadIdx.x; i < end; i += THREADS) {
        const double a = __ldg(pb + i), c = __ldg(tb + i);
        i_ += a * c;
        u_ += a + c - a * c;
    }
    i_ = cta_sum(i_, s[0]);
    u_ = cta_sum(u_, s[1]);
    if (threadIdx.x == 0) {
        const size_t slot = (size_t)b * gridDim.x + blockIdx.x;
        si[slot] = i_;
        su[slot] = u_;
    }
}
__global__ void k_iou_finalize(const double* __restrict__ si, const double* __restrict__ su, double* __restrict__ inter,
                               double* __restrict__ uni, double* __restrict__ loss, int B, int nslot) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const double I = sum_ascending(si + (size_t)b * nslot, nslot);
    const double u = sum_ascending(su + (size_t)b * nslot, nslot) + 1e-6;
    inter[b] = I;
    uni[b] = u;
    loss[b] = 1.0 - I / u;
}
__global__ void __launch_bounds__(256) k_iou_bwd(const double* __restrict__ t, const double* __restrict__ inter,
                                                 const double* __restrict__ uni, const double* __restrict__ gl,
                                                 double* __restrict__ gp, int64_t N) {
    const int b = blockIdx.y;
    const double I = __ldg(inter + b), U = __ldg(uni + b), g = __ldg(gl + b);
    const double k = -g / (U * U);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
        const double tt = __ldg(t + (size_t)b * N + i);
        gp[(size_t)b * N + i] = k * (tt * U - I * (1.0 - tt));
    }
}

// ---------------------------------------------------------------------------------------------
// masked L1: slots [B][gridDim.x], each the CTA's sum times 1 / (C * HW)
// ---------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(THREADS) k_masked_l1_fwd(const double* __restrict__ pred, int64_t pred_bs,
                                                           const double* __restrict__ mpred, int64_t mpred_bs,
                                                           const double* __restrict__ gt, const double* __restrict__ mgt,
                                                           double* __restrict__ slots, int64_t HW, double inv_n) {
    __shared__ double s[8];
    const int b = blockIdx.y;
    const double* p = pred + (size_t)b * pred_bs;
    const double* mp = mpred + (size_t)b * mpred_bs;
    const double* g = gt + (size_t)b * C * HW;
    const double* mg = mgt + (size_t)b * HW;
    const int64_t begin = (int64_t)blockIdx.x * PER_CTA;
    const int64_t end = min(HW, begin + PER_CTA);
    double acc = 0.0;
    for (int64_t i = begin + threadIdx.x; i < end; i += THREADS) {
        const double a = __ldg(mp + i), m = __ldg(mg + i);
#pragma unroll
        for (int c = 0; c < C; ++c) acc += fabs(__ldg(p + (size_t)c * HW + i) * a - __ldg(g + (size_t)c * HW + i) * m);
    }
    acc = cta_sum(acc, s);
    if (threadIdx.x == 0) slots[(size_t)b * gridDim.x + blockIdx.x] = acc * inv_n;
}
template <int C>
__global__ void __launch_bounds__(256) k_masked_l1_bwd(const double* __restrict__ pred, int64_t pred_bs,
                                                       const double* __restrict__ mpred, int64_t mpred_bs,
                                                       const double* __restrict__ gt, const double* __restrict__ mgt,
                                                       const double* __restrict__ gl, double* __restrict__ gpred,
                                                       double* __restrict__ gmask, int64_t HW, double inv_n) {
    const int b = blockIdx.y;
    const double* p = pred + (size_t)b * pred_bs;
    const double* mp = mpred + (size_t)b * mpred_bs;
    const double* g = gt + (size_t)b * C * HW;
    const double* mg = mgt + (size_t)b * HW;
    const double k = __ldg(gl + b) * inv_n;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (int64_t)gridDim.x * blockDim.x) {
        const double a = __ldg(mp + i), m = __ldg(mg + i);
        double gm = 0.0;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const double pv = __ldg(p + (size_t)c * HW + i);
            const double d = pv * a - __ldg(g + (size_t)c * HW + i) * m;
            const double sg = d > 0.0 ? k : (d < 0.0 ? -k : 0.0);  // torch: grad * sign(d), sign(0) = 0
            if (gpred) gpred[((size_t)b * C + c) * HW + i] = sg * a;
            gm += sg * pv;
        }
        if (gmask) gmask[(size_t)b * HW + i] = gm;
    }
}

// ---------------------------------------------------------------------------------------------
// fused loss head: slots [B][gridDim.x][3] of (sum alpha*m, sum alpha + m - alpha*m, sum_c |rgb_c*alpha - gt_c*m|)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(THREADS) k_losshead_partial(const double* __restrict__ rgba, const double* __restrict__ gt,
                                                              const double* __restrict__ mgt, double* __restrict__ slots,
                                                              int64_t HW) {
    __shared__ double s[3][8];
    const int b = blockIdx.y;
    const double* im = rgba + (size_t)b * 4 * HW;
    const double* g = gt + (size_t)b * 3 * HW;
    const double* mg = mgt + (size_t)b * HW;
    const int64_t begin = (int64_t)blockIdx.x * PER_CTA;
    const int64_t end = min(HW, begin + PER_CTA);
    double si = 0.0, su = 0.0, sl = 0.0;
    for (int64_t i = begin + threadIdx.x; i < end; i += THREADS) {
        const double a = __ldg(im + 3 * HW + i), m = __ldg(mg + i);
        si += a * m;
        su += a + m - a * m;
#pragma unroll
        for (int c = 0; c < 3; ++c) sl += fabs(__ldg(im + (size_t)c * HW + i) * a - __ldg(g + (size_t)c * HW + i) * m);
    }
    si = cta_sum(si, s[0]);
    su = cta_sum(su, s[1]);
    sl = cta_sum(sl, s[2]);
    if (threadIdx.x == 0) {
        double* o = slots + ((size_t)b * gridDim.x + blockIdx.x) * 3;
        o[0] = si; o[1] = su; o[2] = sl;
    }
}
__global__ void k_losshead_sum(const double* __restrict__ slots, double* __restrict__ stats, int B, int nslot) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;  // (b, k)
    if (r >= B * 3) return;
    const double* s = slots + (size_t)(r / 3) * nslot * 3 + r % 3;
    double t = 0.0;
    for (int c = 0; c < nslot; ++c) t += s[(size_t)c * 3];
    stats[r] = t;
}
// one warp: stats[b] = (I, U + 1e-6, L1 sum); per_image[b] = (1 - I/U, L1 mean); loss = weighted batch means
__global__ void k_losshead_finalize(double* __restrict__ acc, double* __restrict__ per_image, double* __restrict__ loss, int B,
                                    double inv_n, double w_iou, double w_tex) {
    double t_iou = 0.0, t_tex = 0.0;
    for (int b = threadIdx.x; b < B; b += 32) {
        const double I = acc[b * 3 + 0], U = acc[b * 3 + 1] + 1e-6, L = acc[b * 3 + 2] * inv_n;
        acc[b * 3 + 1] = U;
        const double li = 1.0 - I / U;
        per_image[b * 2 + 0] = li;
        per_image[b * 2 + 1] = L;
        t_iou += li;
        t_tex += L;
    }
    t_iou = warp_sum(t_iou);
    t_tex = warp_sum(t_tex);
    if (threadIdx.x == 0) loss[0] = w_iou * (t_iou / B) + w_tex * (t_tex / B);
}
__global__ void __launch_bounds__(256) k_losshead_bwd(const double* __restrict__ rgba, const double* __restrict__ gt,
                                                      const double* __restrict__ mgt, const double* __restrict__ acc,
                                                      const double* __restrict__ gloss, double* __restrict__ grgba, int64_t HW,
                                                      int B, double inv_n, double w_iou, double w_tex) {
    const int b = blockIdx.y;
    const double* im = rgba + (size_t)b * 4 * HW;
    const double* g = gt + (size_t)b * 3 * HW;
    const double* mg = mgt + (size_t)b * HW;
    double* go = grgba + (size_t)b * 4 * HW;
    const double gl = __ldg(gloss);
    const double I = __ldg(acc + b * 3 + 0), U = __ldg(acc + b * 3 + 1);
    const double ki = -(gl * w_iou / B) / (U * U);
    const double kt = gl * w_tex / B * inv_n;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (int64_t)gridDim.x * blockDim.x) {
        const double a = __ldg(im + 3 * HW + i), m = __ldg(mg + i);
        double ga = ki * (m * U - I * (1.0 - m));
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double pv = __ldg(im + (size_t)c * HW + i);
            const double d = pv * a - __ldg(g + (size_t)c * HW + i) * m;
            const double sg = d > 0.0 ? kt : (d < 0.0 ? -kt : 0.0);
            go[(size_t)c * HW + i] = sg * a;
            ga += sg * pv;
        }
        go[3 * HW + i] = ga;
    }
}

// ---------------------------------------------------------------------------------------------
// chamfer: one warp per query point, lanes stride over the keys; P = (|q|^2 + |k|^2) - 2 (q.k) with
// |p|^2 = ((p0 p0 + p1 p1) + p2 p2), a.b = ((a0 b0 + a1 b1) + a2 b2), every operation rounded once (-fmad=false);
// lexicographic (value, index) minimum, so the lowest index wins ties as in torch.min
// ---------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(256) k_chamfer_nn(const double* __restrict__ q, const double* __restrict__ k,
                                                    double* __restrict__ dist, int32_t* __restrict__ idx, int NQ, int NK) {
    const int lane = threadIdx.x & 31;
    const int qi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int b = blockIdx.y;
    if (qi >= NQ) return;
    const double* qp = q + ((size_t)b * NQ + qi) * D;
    double qv[D];
#pragma unroll
    for (int d = 0; d < D; ++d) qv[d] = __ldg(qp + d);
    double qq = qv[0] * qv[0];
#pragma unroll
    for (int d = 1; d < D; ++d) qq = qq + qv[d] * qv[d];
    double best = __longlong_as_double(0x7ff0000000000000ll);  // +inf
    int bi = 0x7fffffff;
    const double* kb = k + (size_t)b * NK * D;
    for (int j = lane; j < NK; j += 32) {
        double kv[D];
#pragma unroll
        for (int d = 0; d < D; ++d) kv[d] = __ldg(kb + (size_t)j * D + d);
        double kk = kv[0] * kv[0], zz = qv[0] * kv[0];
#pragma unroll
        for (int d = 1; d < D; ++d) {
            kk = kk + kv[d] * kv[d];
            zz = zz + qv[d] * kv[d];
        }
        const double P = (qq + kk) - 2.0 * zz;
        if (P < best) { best = P; bi = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) {
        dist[(size_t)b * NQ + qi] = best;
        idx[(size_t)b * NQ + qi] = bi;
    }
}

// gq[i] = own term 2 gd_q[i] (q_i - k_idx[i]) + sum over j with idx_k[j] == i of -2 gd_k[j] (k_j - q_i): lane l owns
// the j = l (mod 32) in ascending order, the lanes meet in warp_sum's fixed tree (losses.cu k_chamfer_bwd_gather)
template <int D>
__global__ void __launch_bounds__(256) k_chamfer_bwd_gather(const double* __restrict__ q, const double* __restrict__ k,
                                                            const int32_t* __restrict__ idx_q, const int32_t* __restrict__ idx_k,
                                                            const double* __restrict__ gd_q, const double* __restrict__ gd_k,
                                                            double* __restrict__ gq, int NQ, int NK) {
    const int lane = threadIdx.x & 31;
    const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int b = blockIdx.y;
    if (i >= NQ) return;
    double qv[D], acc[D];
#pragma unroll
    for (int d = 0; d < D; ++d) { qv[d] = __ldg(q + ((size_t)b * NQ + i) * D + d); acc[d] = 0.0; }
    if (gd_k != nullptr) {
        const int32_t* ik = idx_k + (size_t)b * NK;
        for (int j0 = 0; j0 < NK; j0 += 32) {
            const int j = j0 + lane;
            const bool hit = j < NK && __ldg(ik + j) == i;
            if (__ballot_sync(0xffffffffu, hit) == 0u) continue;
            if (hit) {
                const double g = __ldg(gd_k + (size_t)b * NK + j);
#pragma unroll
                for (int d = 0; d < D; ++d) acc[d] += -2.0 * g * (__ldg(k + ((size_t)b * NK + j) * D + d) - qv[d]);
            }
        }
#pragma unroll
        for (int d = 0; d < D; ++d) acc[d] = warp_sum(acc[d]);
    }
    if (lane != 0) return;
    double own[D];
#pragma unroll
    for (int d = 0; d < D; ++d) own[d] = 0.0;
    if (gd_q != nullptr) {
        const double g = __ldg(gd_q + (size_t)b * NQ + i);
        const int j = __ldg(idx_q + (size_t)b * NQ + i);
#pragma unroll
        for (int d = 0; d < D; ++d) own[d] = 2.0 * g * (qv[d] - __ldg(k + ((size_t)b * NK + j) * D + d));
    }
#pragma unroll
    for (int d = 0; d < D; ++d) gq[((size_t)b * NQ + i) * D + d] = own[d] + acc[d];
}

// ---------------------------------------------------------------------------------------------
// texture cycle: one thread per (b, f), slots [gridDim.x] of the CTA sums times 1 / (2 B F)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_texcycle_fwd(const double2* __restrict__ flow, const double2* __restrict__ prob,
                                                      const uint8_t* __restrict__ vis, double* __restrict__ slots, int n, int T2,
                                                      double scale) {
    __shared__ double s[8];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    double acc = 0.0;
    if (i < n && vis[i]) {
        double sx = 0.0, sy = 0.0;
        for (int t = 0; t < T2; ++t) {
            const double2 v = __ldg(flow + (size_t)i * T2 + t);
            sx += v.x; sy += v.y;
        }
        const double2 p = __ldg(prob + i);
        const double dx = sx / (double)T2 - p.x, dy = sy / (double)T2 - p.y;
        acc = dx * dx + dy * dy;
    }
    acc = cta_sum(acc, s);
    if (threadIdx.x == 0) slots[blockIdx.x] = acc * scale;
}
__global__ void __launch_bounds__(256) k_texcycle_bwd(const double2* __restrict__ flow, const double2* __restrict__ prob,
                                                      const uint8_t* __restrict__ vis, const double* __restrict__ gl,
                                                      double2* __restrict__ gflow, int n, int T2, double scale) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double gx = 0.0, gy = 0.0;
    if (vis[i]) {
        double sx = 0.0, sy = 0.0;
        for (int t = 0; t < T2; ++t) {
            const double2 v = __ldg(flow + (size_t)i * T2 + t);
            sx += v.x; sy += v.y;
        }
        const double2 p = __ldg(prob + i);
        const double k = 2.0 * __ldg(gl) * scale / (double)T2;
        gx = k * (sx / (double)T2 - p.x);
        gy = k * (sy / (double)T2 - p.y);
    }
    for (int t = 0; t < T2; ++t) gflow[(size_t)i * T2 + t] = make_double2(gx, gy);
}

// ---------------------------------------------------------------------------------------------
// Laplacian (mesh_ops.cu k_laplacian_*): y_i = x_i + sum_j coef[i,j] x_j, loss_b = sum_i |y_i|^2; slots [B][gridDim.x]
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_laplacian_fwd(const double* __restrict__ x, const int32_t* __restrict__ rowptr,
                                                       const int32_t* __restrict__ col, const double* __restrict__ coef,
                                                       double* __restrict__ y, double* __restrict__ slots, int V) {
    __shared__ double s[8];
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    double acc = 0.0;
    if (i < V) {
        const double* xb = x + (size_t)b * V * 3;
        double y0 = xb[i * 3], y1 = xb[i * 3 + 1], y2 = xb[i * 3 + 2];
        for (int e = __ldg(rowptr + i); e < __ldg(rowptr + i + 1); ++e) {
            const int j = __ldg(col + e);
            const double c = __ldg(coef + e);
            y0 += c * xb[j * 3]; y1 += c * xb[j * 3 + 1]; y2 += c * xb[j * 3 + 2];
        }
        double* yb = y + ((size_t)b * V + i) * 3;
        yb[0] = y0; yb[1] = y1; yb[2] = y2;
        acc = y0 * y0 + y1 * y1 + y2 * y2;
    }
    acc = cta_sum(acc, s);
    if (threadIdx.x == 0) slots[(size_t)b * gridDim.x + blockIdx.x] = acc;
}
__global__ void __launch_bounds__(256) k_laplacian_bwd(const double* __restrict__ y, const int32_t* __restrict__ rowptr,
                                                       const int32_t* __restrict__ col, const double* __restrict__ tcoef,
                                                       const double* __restrict__ gl, double* __restrict__ gx, int V) {
    const int b = blockIdx.y;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= V) return;
    const double* yb = y + (size_t)b * V * 3;
    double g0 = yb[j * 3], g1 = yb[j * 3 + 1], g2 = yb[j * 3 + 2];
    for (int e = __ldg(rowptr + j); e < __ldg(rowptr + j + 1); ++e) {
        const int i = __ldg(col + e);
        const double c = __ldg(tcoef + e);
        g0 += c * yb[i * 3]; g1 += c * yb[i * 3 + 1]; g2 += c * yb[i * 3 + 2];
    }
    const double k = 2.0 * __ldg(gl + b);
    double* o = gx + ((size_t)b * V + j) * 3;
    o[0] = k * g0; o[1] = k * g1; o[2] = k * g2;
}

// ---------------------------------------------------------------------------------------------
// flatten (mesh_ops.cu k_flatten / perp_fwd / perp_bwd in double)
// ---------------------------------------------------------------------------------------------
struct Perp {
    double a[3], b[3], cb[3];
    double al2, bl2, al1, bl1, ab, cosv, sinv, k, q, l;
};
__device__ __forceinline__ void perp_fwd(const double* a, const double* b, double eps, Perp& P) {
#pragma unroll
    for (int d = 0; d < 3; ++d) { P.a[d] = a[d]; P.b[d] = b[d]; }
    P.al2 = a[0] * a[0] + a[1] * a[1] + a[2] * a[2];
    P.bl2 = b[0] * b[0] + b[1] * b[1] + b[2] * b[2];
    P.al1 = sqrt(P.al2 + eps);
    P.bl1 = sqrt(P.bl2 + eps);
    P.ab = a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
    P.q = P.al1 * P.bl1 + eps;
    P.cosv = P.ab / P.q;
    P.sinv = sqrt(1 - P.cosv * P.cosv + eps);
    P.k = P.ab / (P.al2 + eps);
#pragma unroll
    for (int d = 0; d < 3; ++d) P.cb[d] = b[d] - a[d] * P.k;
    P.l = P.bl1 * P.sinv;
}
__device__ __forceinline__ void perp_bwd(const Perp& P, const double* dcb, double dl, double eps, double* da, double* db) {
    double dbl1 = dl * P.sinv;
    const double dsinv = dl * P.bl1;
    double dk = 0.0;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        db[d] += dcb[d];
        da[d] += -dcb[d] * P.k;
        dk += -dcb[d] * P.a[d];
    }
    double dab = dk / (P.al2 + eps);
    double dal2 = -dk * P.ab / ((P.al2 + eps) * (P.al2 + eps));
    const double ds = dsinv / (2.0 * P.sinv);
    const double dcosv = -2.0 * P.cosv * ds;
    dab += dcosv / P.q;
    const double dq = -dcosv * P.ab / (P.q * P.q);
    const double dal1 = dq * P.bl1;
    dbl1 += dq * P.al1;
    dal2 += dal1 / (2.0 * P.al1);
    const double dbl2 = dbl1 / (2.0 * P.bl1);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        da[d] += dab * P.b[d] + 2.0 * dal2 * P.a[d];
        db[d] += dab * P.a[d] + 2.0 * dbl2 * P.b[d];
    }
}
// forward (BWD = false): slots [B][gridDim.x]; backward: per-edge terms [B][E][4][3] (roles v0..v3) for k_flatten_gather
template <bool BWD>
__global__ void __launch_bounds__(128) k_flatten(const double* __restrict__ verts, const int32_t* __restrict__ edges,
                                                 double* __restrict__ slots, const double* __restrict__ gl,
                                                 double* __restrict__ terms, int V, int E, double eps) {
    const int b = blockIdx.y;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    double acc = 0.0;
    if (e < E) {
        const double* vb = verts + (size_t)b * V * 3;
        const int i0 = __ldg(edges + e * 4), i1 = __ldg(edges + e * 4 + 1), i2 = __ldg(edges + e * 4 + 2), i3 = __ldg(edges + e * 4 + 3);
        double a[3], b1[3], b2[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const double p0 = vb[i0 * 3 + d];
            a[d] = vb[i1 * 3 + d] - p0;
            b1[d] = vb[i2 * 3 + d] - p0;
            b2[d] = vb[i3 * 3 + d] - p0;
        }
        Perp P1, P2;
        perp_fwd(a, b1, eps, P1);
        perp_fwd(a, b2, eps, P2);
        const double num = P1.cb[0] * P2.cb[0] + P1.cb[1] * P2.cb[1] + P1.cb[2] * P2.cb[2];
        const double den = P1.l * P2.l + eps;
        const double cosd = num / den;
        acc = (cosd + 1) * (cosd + 1);
        if (BWD) {
            const double dcos = 2.0 * (cosd + 1) * __ldg(gl + b);
            const double dnum = dcos / den, dden = -dcos * num / (den * den);
            double dcb1[3], dcb2[3], da[3] = {0, 0, 0}, db1[3] = {0, 0, 0}, db2[3] = {0, 0, 0};
#pragma unroll
            for (int d = 0; d < 3; ++d) { dcb1[d] = dnum * P2.cb[d]; dcb2[d] = dnum * P1.cb[d]; }
            perp_bwd(P1, dcb1, dden * P2.l, eps, da, db1);
            perp_bwd(P2, dcb2, dden * P1.l, eps, da, db2);
            double* t = terms + ((size_t)b * E + e) * 12;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                t[d] = -(da[d] + db1[d] + db2[d]);
                t[3 + d] = da[d];
                t[6 + d] = db1[d];
                t[9 + d] = db2[d];
            }
        }
    }
    if (!BWD) {
        __shared__ double s[4];
        acc = warp_sum(acc);
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        if (lane == 0) s[warp] = acc;
        __syncthreads();
        if (threadIdx.x == 0) slots[(size_t)b * gridDim.x + blockIdx.x] = ((s[0] + s[1]) + s[2]) + s[3];
    }
}
// grad[b][v] = v's terms summed over the transposed table (vrowptr [V+1], vinc: edge * 4 + role / j ascending), `width`
// terms of 3 per batch item; a vertex with no entry gets 0.  Used by flatten (width 4E) and CorrLossChamfer (width NS).
__global__ void __launch_bounds__(256) k_gather3(const double* __restrict__ terms, const int32_t* __restrict__ vrowptr,
                                                 const int32_t* __restrict__ vinc, double* __restrict__ gverts, int V,
                                                 int64_t width) {
    const int b = blockIdx.y;
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const double* tb = terms + (size_t)b * width * 3;
    double g0 = 0.0, g1 = 0.0, g2 = 0.0;
    for (int k = __ldg(vrowptr + v); k < __ldg(vrowptr + v + 1); ++k) {
        const double* t = tb + (size_t)__ldg(vinc + k) * 3;
        g0 += t[0]; g1 += t[1]; g2 += t[2];
    }
    double* o = gverts + ((size_t)b * V + v) * 3;
    o[0] = g0; o[1] = g1; o[2] = g2;
}

// ---------------------------------------------------------------------------------------------
// CorrLossChamfer (vertex.cu k_corr_fwd / k_corr_bwd in double): one CTA per render
// ---------------------------------------------------------------------------------------------
struct Cam {
    double s, tx, ty, q0, q1, q2, q3;
};
__device__ __forceinline__ Cam load_cam(const double* __restrict__ cams, int b) {
    const double* c = cams + (size_t)b * 7;
    Cam k;
    k.s = __ldg(c); k.tx = __ldg(c + 1); k.ty = __ldg(c + 2);
    k.q0 = __ldg(c + 3); k.q1 = __ldg(c + 4); k.q2 = __ldg(c + 5); k.q3 = __ldg(c + 6);
    return k;
}
// quat_rotate (geom_utils.py:147-165), products in the reference's order (hamilton_product, :119-144)
__device__ __forceinline__ void quat_rotate(const Cam& k, double x, double y, double z, double& r1, double& r2, double& r3) {
    const double b0 = k.q0, b1 = -k.q1, b2 = -k.q2, b3 = -k.q3;
    const double a0 = x * 0.0;
    const double t0 = a0 * b0 - x * b1 - y * b2 - z * b3;
    const double t1 = a0 * b1 + x * b0 + y * b3 - z * b2;
    const double t2 = a0 * b2 - x * b3 + y * b0 + z * b1;
    const double t3 = a0 * b3 + x * b2 - y * b1 + z * b0;
    r1 = k.q0 * t1 + k.q1 * t0 + k.q2 * t3 - k.q3 * t2;
    r2 = k.q0 * t2 - k.q1 * t3 + k.q2 * t0 + k.q3 * t1;
    r3 = k.q0 * t3 + k.q1 * t2 - k.q2 * t1 + k.q3 * t0;
}
__device__ __forceinline__ void project_point_backward(const Cam& k, double X, double Y, double Z, double gx, double gy,
                                                       double* gc, double& o0, double& o1, double& o2) {
    double r1, r2, r3;
    quat_rotate(k, X, Y, Z, r1, r2, r3);
    gc[0] += gx * r1 + gy * r2;
    gc[1] += gx;
    gc[2] += gy;
    const double Gx = k.s * gx, Gy = k.s * gy, Gz = 0.0;
    const double vx = k.q1, vy = k.q2, vz = k.q3, q0 = k.q0;
    const double vv = vx * vx + vy * vy + vz * vz;
    const double vG = vx * Gx + vy * Gy + vz * Gz;
    const double vX = vx * X + vy * Y + vz * Z;
    const double XG = X * Gx + Y * Gy + Z * Gz;
    const double c0 = q0 * q0 - vv;
    const double cx = vy * Gz - vz * Gy, cy = vz * Gx - vx * Gz, cz = vx * Gy - vy * Gx;  // v x G
    o0 = c0 * Gx + 2.0 * vG * vx - 2.0 * q0 * cx;
    o1 = c0 * Gy + 2.0 * vG * vy - 2.0 * q0 * cy;
    o2 = c0 * Gz + 2.0 * vG * vz - 2.0 * q0 * cz;
    const double wx = vy * Z - vz * Y, wy = vz * X - vx * Z, wz = vx * Y - vy * X;  // v x X
    gc[3] += 2.0 * (q0 * XG + (Gx * wx + Gy * wy + Gz * wz));
    const double ex = Y * Gz - Z * Gy, ey = Z * Gx - X * Gz, ez = X * Gy - Y * Gx;  // X x G
    gc[4] += 2.0 * (-XG * vx + vG * X + vX * Gx + q0 * ex);
    gc[5] += 2.0 * (-XG * vy + vG * Y + vX * Gy + q0 * ey);
    gc[6] += 2.0 * (-XG * vz + vG * Z + vX * Gz + q0 * ez);
}

struct CorrCfg {
    const double* tgt[4];  // [B, m[g], 2] target points of part g
    int m[4];
    int end[4];            // exclusive end of part g in the concatenated selection
    double w[4];
};
__device__ __forceinline__ int corr_part(const CorrCfg& c, int j) { return j < c.end[0] ? 0 : (j < c.end[1] ? 1 : (j < c.end[2] ? 2 : 3)); }

__global__ void __launch_bounds__(256) k_corr_fwd(const double* __restrict__ verts, int64_t verts_bstride,
                                                  const double* __restrict__ cams, const int32_t* __restrict__ sel, CorrCfg c,
                                                  double* __restrict__ vert2d, int32_t* __restrict__ nn, double* __restrict__ loss,
                                                  int NS) {
    __shared__ double s_part[8];
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const Cam k = load_cam(cams, b);
    double acc = 0.0;  // meaningful in lane 0
    for (int j = warp; j < NS; j += 8) {
        const double* p = verts + (size_t)b * verts_bstride + (size_t)__ldg(sel + j) * 3;
        double r1, r2, r3;
        quat_rotate(k, __ldg(p), __ldg(p + 1), __ldg(p + 2), r1, r2, r3);
        const double qx = k.s * r1 + k.tx, qy = k.s * r2 + k.ty;
        const int g = corr_part(c, j);
        const double* tb = c.tgt[g] + (size_t)b * c.m[g] * 2;
        const double qq = qx * qx + qy * qy;
        double best = __longlong_as_double(0x7ff0000000000000ll);
        int bi = 0x7fffffff;
        for (int t = lane; t < c.m[g]; t += 32) {
            const double kx = __ldg(tb + 2 * t), ky = __ldg(tb + 2 * t + 1);
            const double kk = kx * kx + ky * ky;
            const double zz = qx * kx + qy * ky;
            const double P = (qq + kk) - 2.0 * zz;
            if (P < best) { best = P; bi = t; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
        if (lane == 0) {
            vert2d[((size_t)b * NS + j) * 2 + 0] = qx;
            vert2d[((size_t)b * NS + j) * 2 + 1] = qy;
            nn[(size_t)b * NS + j] = bi;
            acc += best * c.w[g];
        }
    }
    if (lane == 0) s_part[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += s_part[w];
        loss[b] = t / (double)NS;
    }
}
// terms [B,NS,3] (per-(render, j) vertex gradients, summed per vertex by k_gather3) or NULL; gcams [B,7] or NULL
__global__ void __launch_bounds__(256) k_corr_bwd(const double* __restrict__ verts, int64_t verts_bstride,
                                                  const double* __restrict__ cams, const int32_t* __restrict__ sel, CorrCfg c,
                                                  const double* __restrict__ vert2d, const int32_t* __restrict__ nn,
                                                  const double* __restrict__ grad_loss, const double* __restrict__ grad_vert2d,
                                                  double* __restrict__ terms, double* __restrict__ gcams, int NS) {
    __shared__ double s[8][7];
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const Cam k = load_cam(cams, b);
    const double gl = __ldg(grad_loss + b) / (double)NS;
    double gc[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int j = threadIdx.x; j < NS; j += 256) {
        const int g = corr_part(c, j);
        const double* p = verts + (size_t)b * verts_bstride + (size_t)__ldg(sel + j) * 3;
        const double qx = __ldg(vert2d + ((size_t)b * NS + j) * 2), qy = __ldg(vert2d + ((size_t)b * NS + j) * 2 + 1);
        const double* t = c.tgt[g] + ((size_t)b * c.m[g] + __ldg(nn + (size_t)b * NS + j)) * 2;
        const double gd = gl * c.w[g];
        double gx = gd * (2.0 * qx - 2.0 * __ldg(t)), gy = gd * (2.0 * qy - 2.0 * __ldg(t + 1));
        if (grad_vert2d != nullptr) {
            gx += __ldg(grad_vert2d + ((size_t)b * NS + j) * 2);
            gy += __ldg(grad_vert2d + ((size_t)b * NS + j) * 2 + 1);
        }
        double o0, o1, o2;
        project_point_backward(k, __ldg(p), __ldg(p + 1), __ldg(p + 2), gx, gy, gc, o0, o1, o2);
        if (terms != nullptr) {
            double* o = terms + ((size_t)b * NS + j) * 3;
            o[0] = o0; o[1] = o1; o[2] = o2;
        }
    }
    if (gcams == nullptr) return;
#pragma unroll
    for (int i = 0; i < 7; ++i) {
        const double r = warp_sum(gc[i]);
        if (lane == 0) s[warp][i] = r;
    }
    __syncthreads();
    if (threadIdx.x < 7) {
        double r = 0.0;
        for (int w = 0; w < 8; ++w) r += s[w][threadIdx.x];
        gcams[(size_t)b * 7 + threadIdx.x] = r;
    }
}

}  // namespace f64
}  // namespace umr

using namespace umr;
using namespace umr::f64;

#define UMR_RET_LAST() return (int)cudaGetLastError()

// ---------------------------------------------------------------------------------------------
// C entry points (include/umr_b200.h, "float64 loss kernels")
// ---------------------------------------------------------------------------------------------
static bool cells_too_large(int32_t B, int32_t H, int32_t W) {
    return B > 65535 || (int64_t)B * ((int64_t)H + 1) * ((int64_t)W + 1) > INT_MAX;
}

extern "C" int umr_bilinear_sample_forward_f64(const double* image, const double* flow, double* out, int32_t B, int32_t C,
                                               int32_t H, int32_t W, int32_t N, void* stream_) {
    if (!image || !flow || !out || B <= 0 || C <= 0 || H <= 0 || W <= 0 || N <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (C > 4) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const dim3 grid((N + 255) / 256, B);
    const double2* fl = reinterpret_cast<const double2*>(flow);
    count_launch();
    switch (C) {
        case 1: k_sample_fwd<1><<<grid, 256, 0, st>>>(image, fl, out, H, W, N); break;
        case 2: k_sample_fwd<2><<<grid, 256, 0, st>>>(image, fl, out, H, W, N); break;
        case 3: k_sample_fwd<3><<<grid, 256, 0, st>>>(image, fl, out, H, W, N); break;
        default: k_sample_fwd<4><<<grid, 256, 0, st>>>(image, fl, out, H, W, N); break;
    }
    UMR_RET_LAST();
}

extern "C" int umr_bilinear_sample_cells_f64(const double* flow, int32_t* cells, int32_t B, int32_t H, int32_t W, int32_t N,
                                             void* stream_) {
    if (!flow || !cells || B <= 0 || H <= 0 || W <= 0 || N <= 0) return UMR_ERR_BAD_ARG;
    if (cells_too_large(B, H, W)) return UMR_ERR_TOO_LARGE;
    count_launch();
    k_sample_cells<<<dim3((N + 255) / 256, B), 256, 0, (cudaStream_t)stream_>>>(reinterpret_cast<const double2*>(flow), cells,
                                                                                 B, H, W, N);
    UMR_RET_LAST();
}

extern "C" int umr_bilinear_sample_backward_f64(const double* image, const double* flow, const double* grad_out,
                                                double* grad_flow, double* grad_image, int32_t B, int32_t C, int32_t H,
                                                int32_t W, int32_t N, const int32_t* cell_rowptr,
                                                const int32_t* cell_samples, void* stream_) {
    if (!image || !flow || !grad_out || !grad_flow || B <= 0 || C <= 0 || H <= 0 || W <= 0 || N <= 0)
        return UMR_ERR_BAD_ARG;
    if (grad_image && (!cell_rowptr || !cell_samples)) return UMR_ERR_BAD_ARG;
    if (cells_too_large(B, H, W)) return UMR_ERR_TOO_LARGE;
    if (C > 4) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const dim3 grid((N + 255) / 256, B), gpix((H * W + 255) / 256, B);
    const double2* fl = reinterpret_cast<const double2*>(flow);
    double2* gf = reinterpret_cast<double2*>(grad_flow);
    count_launch(grad_image ? 2 : 1);
    switch (C) {
        case 1: k_sample_bwd_flow<1><<<grid, 256, 0, st>>>(image, fl, grad_out, gf, H, W, N); break;
        case 2: k_sample_bwd_flow<2><<<grid, 256, 0, st>>>(image, fl, grad_out, gf, H, W, N); break;
        case 3: k_sample_bwd_flow<3><<<grid, 256, 0, st>>>(image, fl, grad_out, gf, H, W, N); break;
        default: k_sample_bwd_flow<4><<<grid, 256, 0, st>>>(image, fl, grad_out, gf, H, W, N); break;
    }
    if (grad_image) {
        switch (C) {
            case 1: k_sample_bwd_image<1><<<gpix, 256, 0, st>>>(fl, grad_out, cell_rowptr, cell_samples, grad_image, H, W); break;
            case 2: k_sample_bwd_image<2><<<gpix, 256, 0, st>>>(fl, grad_out, cell_rowptr, cell_samples, grad_image, H, W); break;
            case 3: k_sample_bwd_image<3><<<gpix, 256, 0, st>>>(fl, grad_out, cell_rowptr, cell_samples, grad_image, H, W); break;
            default: k_sample_bwd_image<4><<<gpix, 256, 0, st>>>(fl, grad_out, cell_rowptr, cell_samples, grad_image, H, W); break;
        }
    }
    UMR_RET_LAST();
}

extern "C" size_t umr_iou_workspace_bytes_f64(int32_t B, int64_t N) {
    if (B <= 0 || N <= 0) return 0;
    return (size_t)2 * B * slots_of(N, PER_CTA) * sizeof(double);
}
extern "C" int umr_iou_forward_f64(const double* predict, int64_t predict_bstride, const double* target, double* inter,
                                   double* uni, double* loss, int32_t B, int64_t N, void* workspace, void* stream_) {
    if (!predict || !target || !inter || !uni || !loss || !workspace || B <= 0 || N <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const unsigned gx = slots_of(N, PER_CTA);
    double* si = (double*)workspace;
    double* su = si + (size_t)B * gx;
    count_launch(2);
    k_iou_partial<<<dim3(gx, B), THREADS, 0, st>>>(predict, target, si, su, N, predict_bstride);
    k_iou_finalize<<<(B + 127) / 128, 128, 0, st>>>(si, su, inter, uni, loss, B, (int)gx);
    UMR_RET_LAST();
}
extern "C" int umr_iou_backward_f64(const double* target, const double* inter, const double* uni, const double* grad_loss,
                                    double* grad_predict, int32_t B, int64_t N, void* stream_) {
    if (!target || !inter || !uni || !grad_loss || !grad_predict || B <= 0 || N <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    const unsigned gx = (unsigned)std::min<int64_t>((N + 1023) / 1024, 1024);
    count_launch();
    k_iou_bwd<<<dim3(gx, B), 256, 0, (cudaStream_t)stream_>>>(target, inter, uni, grad_loss, grad_predict, N);
    UMR_RET_LAST();
}

extern "C" size_t umr_masked_l1_workspace_bytes_f64(int32_t B, int64_t HW) {
    if (B <= 0 || HW <= 0) return 0;
    return (size_t)B * slots_of(HW, PER_CTA) * sizeof(double);
}
extern "C" int umr_masked_l1_forward_f64(const double* pred, int64_t pred_bstride, const double* mask_pred,
                                         int64_t mask_pred_bstride, const double* gt, const double* mask_gt, double* loss,
                                         int32_t B, int32_t C, int64_t HW, void* workspace, void* stream_) {
    if (!pred || !mask_pred || !gt || !mask_gt || !loss || !workspace || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (C != 3 && C != 1) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const unsigned gx = slots_of(HW, PER_CTA);
    const double inv_n = 1.0 / ((double)C * (double)HW);
    double* slots = (double*)workspace;
    count_launch(2);
    if (C == 3) k_masked_l1_fwd<3><<<dim3(gx, B), THREADS, 0, st>>>(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, slots, HW, inv_n);
    else k_masked_l1_fwd<1><<<dim3(gx, B), THREADS, 0, st>>>(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, slots, HW, inv_n);
    k_sum_slot_rows<<<(B + 127) / 128, 128, 0, st>>>(slots, loss, B, (int)gx);
    UMR_RET_LAST();
}
extern "C" int umr_masked_l1_backward_f64(const double* pred, int64_t pred_bstride, const double* mask_pred,
                                          int64_t mask_pred_bstride, const double* gt, const double* mask_gt,
                                          const double* grad_loss, double* grad_pred, double* grad_mask_pred, int32_t B,
                                          int32_t C, int64_t HW, void* stream_) {
    if (!pred || !mask_pred || !gt || !mask_gt || !grad_loss || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (C != 3 && C != 1) return UMR_ERR_UNSUPPORTED;
    const unsigned gx = (unsigned)std::min<int64_t>((HW + 1023) / 1024, 1024);
    const double inv_n = 1.0 / ((double)C * (double)HW);
    cudaStream_t st = (cudaStream_t)stream_;
    count_launch();
    if (C == 3) k_masked_l1_bwd<3><<<dim3(gx, B), 256, 0, st>>>(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, grad_loss, grad_pred, grad_mask_pred, HW, inv_n);
    else k_masked_l1_bwd<1><<<dim3(gx, B), 256, 0, st>>>(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, grad_loss, grad_pred, grad_mask_pred, HW, inv_n);
    UMR_RET_LAST();
}

extern "C" size_t umr_loss_head_workspace_bytes_f64(int32_t B, int64_t HW) {
    if (B <= 0 || HW <= 0) return 0;
    return (size_t)3 * B * slots_of(HW, PER_CTA) * sizeof(double);
}
extern "C" int umr_loss_head_forward_f64(const double* rgba, const double* gt, const double* mask_gt, double* stats,
                                         double* per_image, double* loss, int32_t B, int64_t HW, double w_iou, double w_tex,
                                         void* workspace, void* stream_) {
    if (!rgba || !gt || !mask_gt || !stats || !per_image || !loss || !workspace || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const unsigned gx = slots_of(HW, PER_CTA);
    double* slots = (double*)workspace;
    count_launch(3);
    k_losshead_partial<<<dim3(gx, B), THREADS, 0, st>>>(rgba, gt, mask_gt, slots, HW);
    k_losshead_sum<<<(3 * B + 127) / 128, 128, 0, st>>>(slots, stats, B, (int)gx);
    k_losshead_finalize<<<1, 32, 0, st>>>(stats, per_image, loss, B, 1.0 / (3.0 * (double)HW), w_iou, w_tex);
    UMR_RET_LAST();
}
extern "C" int umr_loss_head_backward_f64(const double* rgba, const double* gt, const double* mask_gt, const double* stats,
                                          const double* grad_loss, double* grad_rgba, int32_t B, int64_t HW, double w_iou,
                                          double w_tex, void* stream_) {
    if (!rgba || !gt || !mask_gt || !stats || !grad_loss || !grad_rgba || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    const unsigned gx = (unsigned)std::min<int64_t>((HW + 255) / 256, 1024);
    count_launch();
    k_losshead_bwd<<<dim3(gx, B), 256, 0, (cudaStream_t)stream_>>>(rgba, gt, mask_gt, stats, grad_loss, grad_rgba, HW, B,
                                                                   1.0 / (3.0 * (double)HW), w_iou, w_tex);
    UMR_RET_LAST();
}

extern "C" int umr_chamfer_forward_f64(const double* a, const double* b, double* dist_ab, double* dist_ba, int32_t* idx_ab,
                                       int32_t* idx_ba, int32_t B, int32_t N, int32_t M, int32_t D, void* stream_) {
    if (!a || !b || !dist_ab || !dist_ba || !idx_ab || !idx_ba || B <= 0 || N <= 0 || M <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (D != 2 && D != 3) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const dim3 g1((N + 7) / 8, B), g2((M + 7) / 8, B);
    count_launch(2);
    if (D == 2) {
        k_chamfer_nn<2><<<g1, 256, 0, st>>>(a, b, dist_ab, idx_ab, N, M);
        k_chamfer_nn<2><<<g2, 256, 0, st>>>(b, a, dist_ba, idx_ba, M, N);
    } else {
        k_chamfer_nn<3><<<g1, 256, 0, st>>>(a, b, dist_ab, idx_ab, N, M);
        k_chamfer_nn<3><<<g2, 256, 0, st>>>(b, a, dist_ba, idx_ba, M, N);
    }
    UMR_RET_LAST();
}
extern "C" int umr_chamfer_backward_f64(const double* a, const double* b, const int32_t* idx_ab, const int32_t* idx_ba,
                                        const double* grad_dist_ab, const double* grad_dist_ba, double* grad_a, double* grad_b,
                                        int32_t B, int32_t N, int32_t M, int32_t D, void* stream_) {
    if (!a || !b || !grad_a || !grad_b || B <= 0 || N <= 0 || M <= 0) return UMR_ERR_BAD_ARG;
    if ((grad_dist_ab && !idx_ab) || (grad_dist_ba && !idx_ba)) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (D != 2 && D != 3) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    const dim3 g1((N + 7) / 8, B), g2((M + 7) / 8, B);  // one warp per output point
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

extern "C" size_t umr_texcycle_workspace_bytes_f64(int32_t B, int32_t F) {
    if (B <= 0 || F <= 0) return 0;
    return (size_t)(((int64_t)B * F + 255) / 256) * sizeof(double);
}
extern "C" int umr_texcycle_forward_f64(const double* flow, const double* prob, const float* face_ids, uint8_t* visible,
                                        double* loss, int32_t B, int32_t F, int32_t T2, int64_t P, void* workspace,
                                        void* stream_) {
    if (!flow || !prob || !visible || !loss || !workspace || B <= 0 || F <= 0 || T2 <= 0 || (face_ids && P <= 0))
        return UMR_ERR_BAD_ARG;
    if (B > 65535 || (int64_t)B * F > INT_MAX) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    if (face_ids) {   // the float32 plane's bitmap (losses.cu); the bitmap only ever receives 1s, so its bytes are fixed
        cudaError_t e = cudaMemsetAsync(visible, 0, (size_t)B * F, st);
        if (e != cudaSuccess) return (int)e;
        const int64_t blocks = (P / 4 + 255) / 256 + 1;
        count_launch(); umr::k_visible<<<dim3((unsigned)(blocks > 1024 ? 1024 : blocks), B), 256, 0, st>>>(face_ids, visible, F, P);
    }
    const int n = B * F;
    const int gx = (n + 255) / 256;
    double* slots = (double*)workspace;
    count_launch(2);
    k_texcycle_fwd<<<gx, 256, 0, st>>>(reinterpret_cast<const double2*>(flow), reinterpret_cast<const double2*>(prob), visible,
                                       slots, n, T2, 1.0 / ((double)n * 2.0));
    k_sum_slot_rows<<<1, 32, 0, st>>>(slots, loss, 1, gx);
    UMR_RET_LAST();
}
extern "C" int umr_texcycle_backward_f64(const double* flow, const double* prob, const uint8_t* visible, const double* grad_loss,
                                         double* grad_flow, int32_t B, int32_t F, int32_t T2, void* stream_) {
    if (!flow || !prob || !visible || !grad_loss || !grad_flow || B <= 0 || F <= 0 || T2 <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535 || (int64_t)B * F > INT_MAX) return UMR_ERR_TOO_LARGE;
    const int n = B * F;
    count_launch();
    k_texcycle_bwd<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream_>>>(reinterpret_cast<const double2*>(flow),
                                                                       reinterpret_cast<const double2*>(prob), visible, grad_loss,
                                                                       reinterpret_cast<double2*>(grad_flow), n, T2,
                                                                       1.0 / ((double)n * 2.0));
    UMR_RET_LAST();
}

extern "C" size_t umr_laplacian_workspace_bytes_f64(int32_t B, int32_t V) {
    if (B <= 0 || V <= 0) return 0;
    return (size_t)B * ((V + 255) / 256) * sizeof(double);
}
extern "C" int umr_laplacian_forward_f64(const double* x, const int32_t* rowptr, const int32_t* col, const double* coef,
                                         double* y, double* loss, int32_t B, int32_t V, void* workspace, void* stream_) {
    if (!x || !rowptr || !col || !coef || !y || !loss || !workspace || B <= 0 || V <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const int gx = (V + 255) / 256;
    double* slots = (double*)workspace;
    count_launch(2);
    k_laplacian_fwd<<<dim3(gx, B), 256, 0, st>>>(x, rowptr, col, coef, y, slots, V);
    k_sum_slot_rows<<<(B + 127) / 128, 128, 0, st>>>(slots, loss, B, gx);
    UMR_RET_LAST();
}
extern "C" int umr_laplacian_backward_f64(const double* y, const int32_t* rowptr, const int32_t* col, const double* tcoef,
                                          const double* grad_loss, double* grad_x, int32_t B, int32_t V, void* stream_) {
    if (!y || !rowptr || !col || !tcoef || !grad_loss || !grad_x || B <= 0 || V <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    count_launch();
    k_laplacian_bwd<<<dim3((V + 255) / 256, B), 256, 0, (cudaStream_t)stream_>>>(y, rowptr, col, tcoef, grad_loss, grad_x, V);
    UMR_RET_LAST();
}

extern "C" size_t umr_flatten_forward_workspace_bytes_f64(int32_t B, int32_t E) {
    if (B <= 0 || E <= 0) return 0;
    return (size_t)B * ((E + 127) / 128) * sizeof(double);
}
extern "C" int umr_flatten_forward_f64(const double* vertices, const int32_t* edges, double* loss, int32_t B, int32_t V,
                                       int32_t E, double eps, void* workspace, void* stream_) {
    if (!vertices || !edges || !loss || !workspace || B <= 0 || V <= 0 || E <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const int gx = (E + 127) / 128;
    double* slots = (double*)workspace;
    count_launch(2);
    k_flatten<false><<<dim3(gx, B), 128, 0, st>>>(vertices, edges, slots, nullptr, nullptr, V, E, eps);
    k_sum_slot_rows<<<(B + 127) / 128, 128, 0, st>>>(slots, loss, B, gx);
    UMR_RET_LAST();
}
extern "C" size_t umr_flatten_backward_workspace_bytes_f64(int32_t B, int32_t E) {
    if (B <= 0 || E <= 0) return 0;
    return (size_t)B * E * 12 * sizeof(double);
}
extern "C" int umr_flatten_backward_f64(const double* vertices, const int32_t* edges, const int32_t* vert_rowptr,
                                        const int32_t* vert_incidence, const double* grad_loss, double* grad_vertices,
                                        int32_t B, int32_t V, int32_t E, double eps, void* workspace, void* stream_) {
    if (!vertices || !edges || !vert_rowptr || !vert_incidence || !grad_loss || !grad_vertices || !workspace || B <= 0 ||
        V <= 0 || E <= 0)
        return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    double* terms = (double*)workspace;
    count_launch(2);
    k_flatten<true><<<dim3((E + 127) / 128, B), 128, 0, st>>>(vertices, edges, nullptr, grad_loss, terms, V, E, eps);
    k_gather3<<<dim3((V + 255) / 256, B), 256, 0, st>>>(terms, vert_rowptr, vert_incidence, grad_vertices, V, (int64_t)E * 4);
    UMR_RET_LAST();
}

static int make_corr_cfg(CorrCfg& c, const double* const* targets, const int32_t* target_counts, const int32_t* part_ends,
                         const double* weights, int NS) {
    int prev = 0;
    for (int g = 0; g < 4; ++g) {
        if (!targets[g] || target_counts[g] <= 0 || part_ends[g] < prev) return UMR_ERR_BAD_ARG;
        c.tgt[g] = targets[g]; c.m[g] = target_counts[g]; c.end[g] = part_ends[g]; c.w[g] = weights[g];
        prev = part_ends[g];
    }
    return prev == NS ? UMR_OK : UMR_ERR_BAD_ARG;
}

extern "C" int umr_corr_chamfer_forward_f64(const double* vertices, int64_t vertices_batch_stride, const double* cams,
                                            const int32_t* selection, const double* const* targets,
                                            const int32_t* target_counts, const int32_t* part_ends, const double* weights,
                                            double* vert2d, int32_t* nearest, double* loss, int32_t B, int32_t NS,
                                            void* stream_) {
    if (!vertices || !cams || !selection || !targets || !target_counts || !part_ends || !weights || !vert2d || !nearest ||
        !loss || B <= 0 || NS <= 0)
        return UMR_ERR_BAD_ARG;
    CorrCfg c;
    const int rc = make_corr_cfg(c, targets, target_counts, part_ends, weights, NS);
    if (rc) return rc;
    count_launch();
    k_corr_fwd<<<B, 256, 0, (cudaStream_t)stream_>>>(vertices, vertices_batch_stride, cams, selection, c, vert2d, nearest, loss, NS);
    UMR_RET_LAST();
}
extern "C" size_t umr_corr_chamfer_workspace_bytes_f64(int32_t B, int32_t NS) {
    if (B <= 0 || NS <= 0) return 0;
    return (size_t)B * NS * 3 * sizeof(double);
}
extern "C" int umr_corr_chamfer_backward_f64(const double* vertices, int64_t vertices_batch_stride, const double* cams,
                                             const int32_t* selection, const double* const* targets,
                                             const int32_t* target_counts, const int32_t* part_ends, const double* weights,
                                             const double* vert2d, const int32_t* nearest, const double* grad_loss,
                                             const double* grad_vert2d, double* grad_vertices, double* grad_cams, int32_t B,
                                             int32_t NS, int32_t V, const int32_t* vert_rowptr, const int32_t* vert_selection,
                                             void* workspace, void* stream_) {
    if (!vertices || !cams || !selection || !targets || !target_counts || !part_ends || !weights || !vert2d || !nearest ||
        !grad_loss || B <= 0 || NS <= 0 || V <= 0)
        return UMR_ERR_BAD_ARG;
    if (grad_vertices && (!vert_rowptr || !vert_selection || !workspace)) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    CorrCfg c;
    const int rc = make_corr_cfg(c, targets, target_counts, part_ends, weights, NS);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream_;
    double* terms = grad_vertices ? (double*)workspace : nullptr;
    count_launch(grad_vertices ? 2 : 1);
    k_corr_bwd<<<B, 256, 0, st>>>(vertices, vertices_batch_stride, cams, selection, c, vert2d, nearest, grad_loss, grad_vert2d,
                                  terms, grad_cams, NS);
    if (grad_vertices)
        k_gather3<<<dim3((V + 255) / 256, B), 256, 0, st>>>(terms, vert_rowptr, vert_selection, grad_vertices, V, (int64_t)NS);
    UMR_RET_LAST();
}
