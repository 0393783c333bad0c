// mesh_ops.cu -- the remaining SoftRas natives and the per-step mesh regularisers / distance transform around the
// render path (SURVEY.md §8f-3, §8f-4).  Compiled with -fmad=false: the two texture-atlas kernels are arithmetic twins
// of the reference kernels (same float/double promotions), checked bit-for-bit against a numpy restatement.
//
//   k_create_texture_image  external/SoftRas/soft_renderer/cuda/create_texture_image_cuda_kernel.cu:10-70
//                           (face textures -> texture atlas image; reached through Mesh.save_obj, train_s2.py:454)
//   k_load_textures         external/SoftRas/soft_renderer/cuda/load_textures_cuda_kernel.cu:8-66
//                           (texture image + uv faces -> [F,R*R,3] face textures; Mesh.from_obj(load_texture=True))
//   k_laplacian_*           SoftRas/losses.py:6-37  LaplacianLoss: the reference multiplies by a dense V x V matrix
//                           (642^2 = 1.6 MB read per batch item); here a CSR neighbour gather.
//   k_flatten_*             SoftRas/losses.py:39-114 FlattenLoss (dihedral-angle regulariser), one thread per (b, edge),
//                           forward and hand-derived backward instead of ~40 elementwise torch kernels.
//   k_edt_*                 utils/image.py:130-141 compute_dt_barrier: exact Euclidean distance transform of the GT mask,
//                           scipy on the host CPU per image per step in the reference (train_s2.py:196).
// The Laplacian / flatten sums and the flatten backward have deterministic variants (DET template parameter,
// k_flatten_gather; `*_deterministic` entry points at the end of this file; DESIGN.md §2).
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "common.cuh"
#include "umr_b200.h"

namespace umr {

// ---------------------------------------------------------------------------------------------
// texture atlas
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_create_texture_image(const float* __restrict__ faces, const float* __restrict__ textures,
                                                              float* __restrict__ image, int64_t npix, int num_faces, int R,
                                                              int R_out, int tile_width, float eps) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const int x = (int)(i % ((int64_t)tile_width * R_out));
    const int y = (int)(i / ((int64_t)tile_width * R_out));
    const int row = x / R_out, column = y / R_out;
    const int fn = row + column * tile_width;
    if (fn >= num_faces) return;
    const float* texture = textures + (size_t)fn * R * R * 3;
    const float* p0 = faces + (size_t)fn * 6;
    const float* p1 = p0 + 2;
    const float* p2 = p0 + 4;
    float face_inv[9] = {p1[1] - p2[1], p2[0] - p1[0], p1[0] * p2[1] - p2[0] * p1[1],
                         p2[1] - p0[1], p0[0] - p2[0], p2[0] * p0[1] - p0[0] * p2[1],
                         p0[1] - p1[1], p1[0] - p0[0], p0[0] * p1[1] - p1[0] * p0[1]};
    const float den = p2[0] * (p0[1] - p1[1]) + p0[0] * (p1[1] - p2[1]) + p1[0] * (p2[1] - p0[1]);
#pragma unroll
    for (int k = 0; k < 9; ++k) face_inv[k] /= (den + eps);
    float w[3], w_sum = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        w[k] = face_inv[3 * k + 0] * x + face_inv[3 * k + 1] * y + face_inv[3 * k + 2];
        w[k] = fmaxf(fminf(w[k], 1.f), 0.f);  // max(min(w, 1.), 0.): a selection, identical in float
        w_sum += w[k];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) w[k] /= (w_sum + eps);
    const int w_x = (int)(w[0] * R), w_y = (int)(w[1] * R);
    const float* src = ((w[0] + w[1]) * R - w_x - w_y <= 1) ? texture + (size_t)(w_y * R + w_x) * 3
                                                           : texture + (size_t)((R - 1 - w_y) * R + (R - 1 - w_x)) * 3;
    image[i * 3 + 0] = src[0];
    image[i * 3 + 1] = src[1];
    image[i * 3 + 2] = src[2];
}

__global__ void __launch_bounds__(256) k_load_textures(const float* __restrict__ image, const float* __restrict__ faces,
                                                       const int32_t* __restrict__ is_update, float* __restrict__ textures,
                                                       int64_t ntexel, int R, int image_height, int image_width) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ntexel) return;
    const int fn = (int)(i / (R * R));
    const int w_y = (int)((i % (R * R)) / R), w_x = (int)(i % R);
    float w0, w1, w2;  // (w + 1./3.) / R etc. are evaluated in double by the reference and stored as float
    if (w_x + w_y < R) {
        w0 = (float)(((double)w_x + 1. / 3.) / (double)R);
        w1 = (float)(((double)w_y + 1. / 3.) / (double)R);
    } else {
        w0 = (float)((((double)R - 1. - (double)w_x) + 2. / 3.) / (double)R);
        w1 = (float)((((double)R - 1. - (double)w_y) + 2. / 3.) / (double)R);
    }
    w2 = (float)(1. - (double)w0 - (double)w1);
    if (__ldg(is_update + fn) == 0) return;
    const float* face = faces + (size_t)fn * 6;
    const float pos_x = (face[0] * w0 + face[2] * w1 + face[4] * w2) * (float)(image_width - 1);
    const float pos_y = (face[1] * w0 + face[3] * w1 + face[5] * w2) * (float)(image_height - 1);
    const float wx1 = pos_x - (int)pos_x, wx0 = 1 - wx1;
    const float wy1 = pos_y - (int)pos_y, wy0 = 1 - wy1;
    const int ix = (int)pos_x, iy = (int)pos_y, iy1 = (int)(pos_y + 1);
    // The reference reads these four corners unclamped: uv = 1 on a whole face puts ix + 1 = W or iy1 = H (with weight
    // 0), negative uv puts them below 0, and (int)(pos_y + 1) can skip to H when pos_y lies just below H - 1.  Clamped
    // into the image here (DESIGN.md §2); a texel whose corners are all inside computes the reference's bits.
    const int x0 = min(max(ix, 0), image_width - 1), x1 = max(min(ix, image_width - 2) + 1, 0);
    const int y0 = min(max(iy, 0), image_height - 1), y1 = min(max(iy1, 0), image_height - 1);
    float* texture = textures + i * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float c = 0.f;
        c += image[((size_t)y0 * image_width + x0) * 3 + k] * (wx0 * wy0);
        c += image[((size_t)y1 * image_width + x0) * 3 + k] * (wx0 * wy1);
        c += image[((size_t)y0 * image_width + x1) * 3 + k] * (wx1 * wy0);
        c += image[((size_t)y1 * image_width + x1) * 3 + k] * (wx1 * wy1);
        texture[k] = c;
    }
}

// ---------------------------------------------------------------------------------------------
// Laplacian regulariser on a CSR neighbour table: y_i = x_i + sum_j coef[i,j] x_j  (coef = -1/deg_i as float32,
// exactly the off-diagonal entries of the reference's row-normalised matrix), loss_b = sum_i |y_i|^2
// ---------------------------------------------------------------------------------------------
// DET: `loss` is the workspace slot array [B][gridDim.x]; every CTA stores its partial
template <bool DET>
__global__ void __launch_bounds__(256) k_laplacian_fwd(const float* __restrict__ x, const int32_t* __restrict__ rowptr,
                                                       const int32_t* __restrict__ col, const float* __restrict__ coef,
                                                       float* __restrict__ y, float* __restrict__ loss, int V) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float acc = 0.f;
    if (i < V) {
        const float* xb = x + (size_t)b * V * 3;
        float y0 = xb[i * 3], y1 = xb[i * 3 + 1], y2 = xb[i * 3 + 2];
        for (int e = __ldg(rowptr + i); e < __ldg(rowptr + i + 1); ++e) {
            const int j = __ldg(col + e);
            const float c = __ldg(coef + e);
            y0 += c * xb[j * 3]; y1 += c * xb[j * 3 + 1]; y2 += c * xb[j * 3 + 2];
        }
        float* yb = y + ((size_t)b * V + i) * 3;
        yb[0] = y0; yb[1] = y1; yb[2] = y2;
        acc = y0 * y0 + y1 * y1 + y2 * y2;
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
            if (lane == 0) loss[(size_t)b * gridDim.x + blockIdx.x] = acc;
        } else {
            if (lane == 0) atomicAdd(loss + b, acc);
        }
    }
}
// deterministic finalize of the Laplacian / flatten sums: loss[b] = image b's n slots summed in ascending CTA order
__global__ void k_mesh_loss_sum_det(const float* __restrict__ slots, float* __restrict__ loss, int B, int n) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B) loss[b] = sum_ascending(slots + (size_t)b * n, n);
}
// grad_x_j = 2 g_b (y_j + sum_{i : j in N(i)} coef[i,j] y_i); the neighbour relation is symmetric, so the transposed
// entry of (j, i) is looked up through tcoef[e] = coef of row col[e] towards j (precomputed on the host)
__global__ void __launch_bounds__(256) k_laplacian_bwd(const float* __restrict__ y, const int32_t* __restrict__ rowptr,
                                                       const int32_t* __restrict__ col, const float* __restrict__ tcoef,
                                                       const float* __restrict__ gl, float* __restrict__ gx, int V) {
    const int b = blockIdx.y;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= V) return;
    const float* yb = y + (size_t)b * V * 3;
    float g0 = yb[j * 3], g1 = yb[j * 3 + 1], g2 = yb[j * 3 + 2];
    for (int e = __ldg(rowptr + j); e < __ldg(rowptr + j + 1); ++e) {
        const int i = __ldg(col + e);
        const float c = __ldg(tcoef + e);
        g0 += c * yb[i * 3]; g1 += c * yb[i * 3 + 1]; g2 += c * yb[i * 3 + 2];
    }
    const float k = 2.f * __ldg(gl + b);
    float* o = gx + ((size_t)b * V + j) * 3;
    o[0] = k * g0; o[1] = k * g1; o[2] = k * g2;
}

// ---------------------------------------------------------------------------------------------
// Flatten regulariser: per edge (v0, v1) with opposite corners v2, v3 (losses.py:71-108)
// ---------------------------------------------------------------------------------------------
struct Perp {  // forward values of one `perp(a, b)` block kept for the backward
    float a[3], b[3], cb[3];
    float al2, bl2, al1, bl1, ab, cosv, sinv, k, q, l;
};
__device__ __forceinline__ void perp_fwd(const float* a, const float* b, float eps, Perp& P) {
#pragma unroll
    for (int d = 0; d < 3; ++d) { P.a[d] = a[d]; P.b[d] = b[d]; }
    P.al2 = a[0] * a[0] + a[1] * a[1] + a[2] * a[2];
    P.bl2 = b[0] * b[0] + b[1] * b[1] + b[2] * b[2];
    P.al1 = sqrtf(P.al2 + eps);
    P.bl1 = sqrtf(P.bl2 + eps);
    P.ab = a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
    P.q = P.al1 * P.bl1 + eps;
    P.cosv = P.ab / P.q;
    P.sinv = sqrtf(1 - P.cosv * P.cosv + eps);
    P.k = P.ab / (P.al2 + eps);
#pragma unroll
    for (int d = 0; d < 3; ++d) P.cb[d] = b[d] - a[d] * P.k;
    P.l = P.bl1 * P.sinv;
}
// reverse mode through perp(): inputs dcb[3], dl -> accumulates da[3], db[3]
__device__ __forceinline__ void perp_bwd(const Perp& P, const float* dcb, float dl, float eps, float* da, float* db) {
    float dbl1 = dl * P.sinv;
    const float dsinv = dl * P.bl1;
    float dk = 0.f;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        db[d] += dcb[d];
        da[d] += -dcb[d] * P.k;
        dk += -dcb[d] * P.a[d];
    }
    float dab = dk / (P.al2 + eps);
    float dal2 = -dk * P.ab / ((P.al2 + eps) * (P.al2 + eps));
    const float ds = dsinv / (2.f * P.sinv);
    const float dcosv = -2.f * P.cosv * ds;
    dab += dcosv / P.q;
    const float dq = -dcosv * P.ab / (P.q * P.q);
    const float dal1 = dq * P.bl1;
    dbl1 += dq * P.al1;
    dal2 += dal1 / (2.f * P.al1);
    const float dbl2 = dbl1 / (2.f * P.bl1);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        da[d] += dab * P.b[d] + 2.f * dal2 * P.a[d];
        db[d] += dab * P.a[d] + 2.f * dbl2 * P.b[d];
    }
}
// DET forward: `loss` is the workspace slot array [B][gridDim.x].  DET backward: `gverts` is the per-edge term array
// [B][E][4][3] (roles v0..v3), summed per vertex by k_flatten_gather.
template <bool BWD, bool DET>
__global__ void __launch_bounds__(128) k_flatten(const float* __restrict__ verts, const int32_t* __restrict__ edges,
                                                 float* __restrict__ loss, const float* __restrict__ gl,
                                                 float* __restrict__ gverts, int V, int E, float eps) {
    const int b = blockIdx.y;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    float acc = 0.f;
    if (e < E) {
        const float* vb = verts + (size_t)b * V * 3;
        const int i0 = __ldg(edges + e * 4), i1 = __ldg(edges + e * 4 + 1), i2 = __ldg(edges + e * 4 + 2), i3 = __ldg(edges + e * 4 + 3);
        float a[3], b1[3], b2[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const float p0 = vb[i0 * 3 + d];
            a[d] = vb[i1 * 3 + d] - p0;
            b1[d] = vb[i2 * 3 + d] - p0;
            b2[d] = vb[i3 * 3 + d] - p0;
        }
        Perp P1, P2;
        perp_fwd(a, b1, eps, P1);
        perp_fwd(a, b2, eps, P2);
        const float num = P1.cb[0] * P2.cb[0] + P1.cb[1] * P2.cb[1] + P1.cb[2] * P2.cb[2];
        const float den = P1.l * P2.l + eps;
        const float cosd = num / den;
        acc = (cosd + 1) * (cosd + 1);
        if (BWD) {
            const float dcos = 2.f * (cosd + 1) * __ldg(gl + b);
            const float dnum = dcos / den, dden = -dcos * num / (den * den);
            float dcb1[3], dcb2[3], da[3] = {0, 0, 0}, db1[3] = {0, 0, 0}, db2[3] = {0, 0, 0};
#pragma unroll
            for (int d = 0; d < 3; ++d) { dcb1[d] = dnum * P2.cb[d]; dcb2[d] = dnum * P1.cb[d]; }
            perp_bwd(P1, dcb1, dden * P2.l, eps, da, db1);
            perp_bwd(P2, dcb2, dden * P1.l, eps, da, db2);
            if (DET) {
                float* t = gverts + ((size_t)b * E + e) * 12;
#pragma unroll
                for (int d = 0; d < 3; ++d) {
                    t[d] = -(da[d] + db1[d] + db2[d]);
                    t[3 + d] = da[d];
                    t[6 + d] = db1[d];
                    t[9 + d] = db2[d];
                }
            } else {
                float* gb = gverts + (size_t)b * V * 3;
#pragma unroll
                for (int d = 0; d < 3; ++d) {
                    atomicAdd(gb + i1 * 3 + d, da[d]);
                    atomicAdd(gb + i2 * 3 + d, db1[d]);
                    atomicAdd(gb + i3 * 3 + d, db2[d]);
                    atomicAdd(gb + i0 * 3 + d, -(da[d] + db1[d] + db2[d]));
                }
            }
        }
    }
    if (!BWD) {
        acc = warp_sum(acc);
        __shared__ float s[4];
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        if (lane == 0) s[warp] = acc;
        __syncthreads();
        if (warp == 0) {
            acc = lane < 4 ? s[lane] : 0.f;
            acc = warp_sum(acc);
            if (DET) {
                if (lane == 0) loss[(size_t)b * gridDim.x + blockIdx.x] = acc;
            } else {
                if (lane == 0) atomicAdd(loss + b, acc);
            }
        }
    }
}
// grad_vertices[b][v] = sum of v's per-edge terms over the transposed incidence table: vrowptr [V+1], vinc [4E] lists
// edge * 4 + role in ascending order, so the sum order is fixed; a vertex on no edge gets 0
__global__ void __launch_bounds__(256) k_flatten_gather(const float* __restrict__ terms, const int32_t* __restrict__ vrowptr,
                                                        const int32_t* __restrict__ vinc, float* __restrict__ gverts, int V,
                                                        int E) {
    const int b = blockIdx.y;
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const float* tb = terms + (size_t)b * E * 12;
    float g0 = 0.f, g1 = 0.f, g2 = 0.f;
    for (int k = __ldg(vrowptr + v); k < __ldg(vrowptr + v + 1); ++k) {
        const float* t = tb + (size_t)__ldg(vinc + k) * 3;
        g0 += t[0]; g1 += t[1]; g2 += t[2];
    }
    float* o = gverts + ((size_t)b * V + v) * 3;
    o[0] = g0; o[1] = g1; o[2] = g2;
}

// ---------------------------------------------------------------------------------------------
// exact Euclidean distance transform + barrier sigmoid (utils/image.py:130-141)
//   pass 1 (per column): g(y, x) = distance along the column to the nearest FEATURE pixel (inf if none)
//   pass 2 (per row):    d^2(y, x) = min_x' (x - x')^2 + g(y, x')^2      -- exact integers
// run for feature = (mask == 1) [dist_out = edt(1 - mask): distance to the object] and feature = (mask == 0) [dist_in =
// edt(mask)].  On a binary mask the two are complements; a value strictly between (the bilinear edge of a resized mask)
// is a feature of neither, as in scipy.
// ---------------------------------------------------------------------------------------------
constexpr int EDT_INF = 1 << 28;
__global__ void __launch_bounds__(256) k_edt_columns(const float* __restrict__ mask, int32_t* __restrict__ g_out,
                                                     int32_t* __restrict__ g_in, int H, int W) {
    const int b = blockIdx.y;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= W) return;
    const float* m = mask + (size_t)b * H * W;
    int32_t* go = g_out + (size_t)b * H * W;
    int32_t* gi = g_in + (size_t)b * H * W;
    int d_obj = EDT_INF, d_bg = EDT_INF;  // distance to the last object / background pixel above
    for (int y = 0; y < H; ++y) {
        const float v = m[(size_t)y * W + x];
        const bool obj = v == 1.f, bg = v == 0.f;
        d_obj = obj ? 0 : (d_obj >= EDT_INF ? EDT_INF : d_obj + 1);
        d_bg = bg ? 0 : (d_bg >= EDT_INF ? EDT_INF : d_bg + 1);
        go[(size_t)y * W + x] = d_obj;
        gi[(size_t)y * W + x] = d_bg;
    }
    d_obj = EDT_INF; d_bg = EDT_INF;
    for (int y = H - 1; y >= 0; --y) {
        const float v = m[(size_t)y * W + x];
        const bool obj = v == 1.f, bg = v == 0.f;
        d_obj = obj ? 0 : (d_obj >= EDT_INF ? EDT_INF : d_obj + 1);
        d_bg = bg ? 0 : (d_bg >= EDT_INF ? EDT_INF : d_bg + 1);
        go[(size_t)y * W + x] = min(go[(size_t)y * W + x], d_obj);
        gi[(size_t)y * W + x] = min(gi[(size_t)y * W + x], d_bg);
    }
}
// one CTA per image row; the row's two column-distance vectors are staged in shared memory
__global__ void __launch_bounds__(256) k_edt_rows(const int32_t* __restrict__ g_out, const int32_t* __restrict__ g_in,
                                                  float* __restrict__ dt, int H, int W, float k, float inv_norm) {
    extern __shared__ int32_t s_g[];  // [2][W]
    const int b = blockIdx.y, y = blockIdx.x;
    const int32_t* go = g_out + ((size_t)b * H + y) * W;
    const int32_t* gi = g_in + ((size_t)b * H + y) * W;
    for (int x = threadIdx.x; x < W; x += blockDim.x) { s_g[x] = go[x]; s_g[W + x] = gi[x]; }
    __syncthreads();
    for (int x = threadIdx.x; x < W; x += blockDim.x) {
        // exact in 32 bits: dx^2 <= 4095^2 and g^2 <= 65535^2 would overflow, so columns are capped at W <= 4096 and
        // column distances above 32767 cannot beat any finite candidate -- they are clamped to "infinite"
        constexpr int NONE = 0x7fffffff;
        int best_o = NONE, best_i = NONE;
#pragma unroll 4
        for (int xp = 0; xp < W; ++xp) {
            const int dx = x - xp, dx2 = dx * dx;
            const int a = s_g[xp], c = s_g[W + xp];
            if (a < 32768) best_o = min(best_o, dx2 + a * a);
            if (c < 32768) best_i = min(best_i, dx2 + c * c);
        }
        // no feature pixel in the whole image (full / empty mask): scipy's distance_transform_edt then measures from a
        // virtual pixel at (row -1, column 0) -- reproduced so that degenerate masks match the reference too
        const int virt = (y + 1) * (y + 1) + x * x;
        if (best_o == NONE) best_o = virt;
        if (best_i == NONE) best_i = virt;
        const double d_out = sqrt((double)best_o), d_in = sqrt((double)best_i);
        const double diff = (d_out - d_in) * (double)inv_norm;
        dt[((size_t)b * H + y) * W + x] = (float)(1. / (1. + exp((double)k * -diff)));
    }
}

}  // namespace umr

using namespace umr;

#define UMR_RET() return (int)cudaGetLastError()

extern "C" int umr_create_texture_image(const float* faces_uv, const float* textures, float* image, int32_t num_faces,
                                        int32_t texture_res_in, int32_t image_height, int32_t image_width, float eps,
                                        void* stream_) {
    if (!faces_uv || !textures || !image || num_faces <= 0 || texture_res_in <= 0 || image_height <= 0 || image_width <= 0)
        return UMR_ERR_BAD_ARG;
    const int tile_width = (int)sqrt((double)(num_faces - 1)) + 1;  // create_texture_image_cuda_kernel.cu:81
    const int R_out = image_width / tile_width;                       // :82 (image.size(1) / tile_width)
    if (R_out <= 0) return UMR_ERR_BAD_ARG;
    const int64_t npix = (int64_t)image_height * image_width;
    count_launch();
    k_create_texture_image<<<(unsigned)((npix + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(
        faces_uv, textures, image, npix, num_faces, texture_res_in, R_out, tile_width, eps);
    UMR_RET();
}

extern "C" int umr_load_textures(const float* image, const float* faces_uv, const int32_t* is_update, float* textures,
                                 int32_t num_faces, int32_t texture_res, int32_t image_height, int32_t image_width,
                                 void* stream_) {
    if (!image || !faces_uv || !is_update || !textures || num_faces <= 0 || texture_res <= 0 || image_height <= 1 || image_width <= 1)
        return UMR_ERR_BAD_ARG;
    const int64_t ntexel = (int64_t)num_faces * texture_res * texture_res;
    count_launch();
    k_load_textures<<<(unsigned)((ntexel + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(image, faces_uv, is_update, textures,
                                                                                         ntexel, texture_res, image_height,
                                                                                         image_width);
    UMR_RET();
}

extern "C" int umr_laplacian_forward(const float* x, const int32_t* rowptr, const int32_t* col, const float* coef, float* y,
                                     float* loss, int32_t B, int32_t V, void* stream_) {
    if (!x || !rowptr || !col || !coef || !y || !loss || B <= 0 || V <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(loss, 0, (size_t)B * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    count_launch();
    k_laplacian_fwd<false><<<dim3((V + 255) / 256, B), 256, 0, st>>>(x, rowptr, col, coef, y, loss, V);
    UMR_RET();
}
extern "C" int umr_laplacian_backward(const float* y, const int32_t* rowptr, const int32_t* col, const float* tcoef,
                                      const float* grad_loss, float* grad_x, int32_t B, int32_t V, void* stream_) {
    if (!y || !rowptr || !col || !tcoef || !grad_loss || !grad_x || B <= 0 || V <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    count_launch();
    k_laplacian_bwd<<<dim3((V + 255) / 256, B), 256, 0, (cudaStream_t)stream_>>>(y, rowptr, col, tcoef, grad_loss, grad_x, V);
    UMR_RET();
}

extern "C" int umr_flatten_forward(const float* vertices, const int32_t* edges, float* loss, int32_t B, int32_t V, int32_t E,
                                   float eps, void* stream_) {
    if (!vertices || !edges || !loss || B <= 0 || V <= 0 || E <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(loss, 0, (size_t)B * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    count_launch();
    k_flatten<false, false><<<dim3((E + 127) / 128, B), 128, 0, st>>>(vertices, edges, loss, nullptr, nullptr, V, E, eps);
    UMR_RET();
}
extern "C" int umr_flatten_backward(const float* vertices, const int32_t* edges, const float* grad_loss, float* grad_vertices,
                                    int32_t B, int32_t V, int32_t E, float eps, void* stream_) {
    if (!vertices || !edges || !grad_loss || !grad_vertices || B <= 0 || V <= 0 || E <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(grad_vertices, 0, (size_t)B * V * 3 * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    count_launch();
    k_flatten<true, false><<<dim3((E + 127) / 128, B), 128, 0, st>>>(vertices, edges, nullptr, grad_loss, grad_vertices, V, E, eps);
    UMR_RET();
}

extern "C" size_t umr_dt_barrier_workspace_bytes(int32_t B, int32_t H, int32_t W) {
    if (B <= 0 || H <= 0 || W <= 0) return 0;
    return (size_t)2 * B * H * W * sizeof(int32_t);
}
extern "C" int umr_dt_barrier(const float* mask, float* dt, void* workspace, int32_t B, int32_t H, int32_t W, float k,
                              void* stream_) {
    if (!mask || !dt || !workspace || B <= 0 || H <= 0 || W <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535 || H > 32767 || W > 4096) return UMR_ERR_TOO_LARGE;  // 32-bit exact squared distances (k_edt_rows)
    cudaStream_t st = (cudaStream_t)stream_;
    int32_t* g_out = (int32_t*)workspace;
    int32_t* g_in = g_out + (size_t)B * H * W;
    count_launch(2);
    k_edt_columns<<<dim3((W + 255) / 256, B), 256, 0, st>>>(mask, g_out, g_in, H, W);
    k_edt_rows<<<dim3(H, B), 256, (size_t)2 * W * sizeof(int32_t), st>>>(g_out, g_in, dt, H, W, k, 1.f / (float)std::max(H, W));
    UMR_RET();
}

// ---------------------------------------------------------------------------------------------
// deterministic mode (include/umr_b200.h, DESIGN.md §2): per-CTA partials stored in workspace slots and summed in
// ascending CTA order; the flatten backward writes per-edge terms and gathers them per vertex
// ---------------------------------------------------------------------------------------------
extern "C" size_t umr_laplacian_workspace_bytes_deterministic(int32_t B, int32_t V) {
    if (B <= 0 || V <= 0) return 0;
    return (size_t)B * ((V + 255) / 256) * sizeof(float);
}
extern "C" int umr_laplacian_forward_deterministic(const float* x, const int32_t* rowptr, const int32_t* col, const float* coef,
                                                   float* y, float* loss, int32_t B, int32_t V, void* workspace, void* stream_) {
    if (!x || !rowptr || !col || !coef || !y || !loss || !workspace || B <= 0 || V <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const int gx = (V + 255) / 256;
    float* slots = (float*)workspace;
    count_launch(2);
    k_laplacian_fwd<true><<<dim3(gx, B), 256, 0, st>>>(x, rowptr, col, coef, y, slots, V);
    k_mesh_loss_sum_det<<<(B + 127) / 128, 128, 0, st>>>(slots, loss, B, gx);
    UMR_RET();
}

extern "C" size_t umr_flatten_forward_workspace_bytes_deterministic(int32_t B, int32_t E) {
    if (B <= 0 || E <= 0) return 0;
    return (size_t)B * ((E + 127) / 128) * sizeof(float);
}
extern "C" int umr_flatten_forward_deterministic(const float* vertices, const int32_t* edges, float* loss, int32_t B, int32_t V,
                                                 int32_t E, float eps, void* workspace, void* stream_) {
    if (!vertices || !edges || !loss || !workspace || B <= 0 || V <= 0 || E <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const int gx = (E + 127) / 128;
    float* slots = (float*)workspace;
    count_launch(2);
    k_flatten<false, true><<<dim3(gx, B), 128, 0, st>>>(vertices, edges, slots, nullptr, nullptr, V, E, eps);
    k_mesh_loss_sum_det<<<(B + 127) / 128, 128, 0, st>>>(slots, loss, B, gx);
    UMR_RET();
}

extern "C" size_t umr_flatten_backward_workspace_bytes_deterministic(int32_t B, int32_t E) {
    if (B <= 0 || E <= 0) return 0;
    return (size_t)B * E * 12 * sizeof(float);
}
extern "C" int umr_flatten_backward_deterministic(const float* vertices, const int32_t* edges, const int32_t* vert_rowptr,
                                                  const int32_t* vert_incidence, const float* grad_loss, float* grad_vertices,
                                                  int32_t B, int32_t V, int32_t E, float eps, void* workspace, void* stream_) {
    if (!vertices || !edges || !vert_rowptr || !vert_incidence || !grad_loss || !grad_vertices || !workspace || B <= 0 ||
        V <= 0 || E <= 0)
        return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    float* terms = (float*)workspace;
    count_launch(2);
    k_flatten<true, true><<<dim3((E + 127) / 128, B), 128, 0, st>>>(vertices, edges, nullptr, grad_loss, terms, V, E, eps);
    k_flatten_gather<<<dim3((V + 255) / 256, B), 256, 0, st>>>(terms, vert_rowptr, vert_incidence, grad_vertices, V, E);
    UMR_RET();
}
