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
// The Laplacian / flatten sums and the flatten backward have deterministic variants (DET template parameter, k_gather3;
// `*_deterministic` entry points at the end of this file; DESIGN.md §2).  The Laplacian and flatten kernels are templated
// on the scalar type: the float64 entry points at the end of this file (DESIGN.md §10) run their double instantiations,
// which share the deterministic structure and launchers.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <type_traits>

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
template <typename T, bool DET>
__global__ void __launch_bounds__(256) k_laplacian_fwd(const T* __restrict__ x, const int32_t* __restrict__ rowptr,
                                                       const int32_t* __restrict__ col, const T* __restrict__ coef,
                                                       T* __restrict__ y, T* __restrict__ loss, int V) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    T acc = 0;
    if (i < V) {
        const T* xb = x + (size_t)b * V * 3;
        T y0 = xb[i * 3], y1 = xb[i * 3 + 1], y2 = xb[i * 3 + 2];
        for (int e = __ldg(rowptr + i); e < __ldg(rowptr + i + 1); ++e) {
            const int j = __ldg(col + e);
            const T c = __ldg(coef + e);
            y0 += c * xb[j * 3]; y1 += c * xb[j * 3 + 1]; y2 += c * xb[j * 3 + 2];
        }
        T* yb = y + ((size_t)b * V + i) * 3;
        yb[0] = y0; yb[1] = y1; yb[2] = y2;
        acc = y0 * y0 + y1 * y1 + y2 * y2;
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
            if (lane == 0) loss[(size_t)b * gridDim.x + blockIdx.x] = acc;
        } else {
            if (lane == 0) atomicAdd(loss + b, acc);
        }
    }
}
// grad_x_j = 2 g_b (y_j + sum_{i : j in N(i)} coef[i,j] y_i); the neighbour relation is symmetric, so the transposed
// entry of (j, i) is looked up through tcoef[e] = coef of row col[e] towards j (precomputed on the host)
template <typename T>
__global__ void __launch_bounds__(256) k_laplacian_bwd(const T* __restrict__ y, const int32_t* __restrict__ rowptr,
                                                       const int32_t* __restrict__ col, const T* __restrict__ tcoef,
                                                       const T* __restrict__ gl, T* __restrict__ gx, int V) {
    const int b = blockIdx.y;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= V) return;
    const T* yb = y + (size_t)b * V * 3;
    T g0 = yb[j * 3], g1 = yb[j * 3 + 1], g2 = yb[j * 3 + 2];
    for (int e = __ldg(rowptr + j); e < __ldg(rowptr + j + 1); ++e) {
        const int i = __ldg(col + e);
        const T c = __ldg(tcoef + e);
        g0 += c * yb[i * 3]; g1 += c * yb[i * 3 + 1]; g2 += c * yb[i * 3 + 2];
    }
    const T k = T(2) * __ldg(gl + b);
    T* o = gx + ((size_t)b * V + j) * 3;
    o[0] = k * g0; o[1] = k * g1; o[2] = k * g2;
}

// ---------------------------------------------------------------------------------------------
// Flatten regulariser: per edge (v0, v1) with opposite corners v2, v3 (losses.py:71-108)
// ---------------------------------------------------------------------------------------------
template <typename T>
struct Perp {  // forward values of one `perp(a, b)` block kept for the backward
    T a[3], b[3], cb[3];
    T al2, bl2, al1, bl1, ab, cosv, sinv, k, q, l;
};
template <typename T>
__device__ __forceinline__ void perp_fwd(const T* a, const T* b, T eps, Perp<T>& P) {
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
// reverse mode through perp(): inputs dcb[3], dl -> accumulates da[3], db[3]
template <typename T>
__device__ __forceinline__ void perp_bwd(const Perp<T>& P, const T* dcb, T dl, T eps, T* da, T* db) {
    T dbl1 = dl * P.sinv;
    const T dsinv = dl * P.bl1;
    T dk = 0;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        db[d] += dcb[d];
        da[d] += -dcb[d] * P.k;
        dk += -dcb[d] * P.a[d];
    }
    T dab = dk / (P.al2 + eps);
    T dal2 = -dk * P.ab / ((P.al2 + eps) * (P.al2 + eps));
    const T ds = dsinv / (T(2) * P.sinv);
    const T dcosv = T(-2) * P.cosv * ds;
    dab += dcosv / P.q;
    const T dq = -dcosv * P.ab / (P.q * P.q);
    const T dal1 = dq * P.bl1;
    dbl1 += dq * P.al1;
    dal2 += dal1 / (T(2) * P.al1);
    const T dbl2 = dbl1 / (T(2) * P.bl1);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        da[d] += dab * P.b[d] + T(2) * dal2 * P.a[d];
        db[d] += dab * P.a[d] + T(2) * dbl2 * P.b[d];
    }
}
// DET forward: `loss` is the workspace slot array [B][gridDim.x].  DET backward: `gverts` is the per-edge term array
// [B][E][4][3] (roles v0..v3), summed per vertex by k_gather3.  Float64 runs only the DET forms.
template <typename T, bool BWD, bool DET>
__global__ void __launch_bounds__(128) k_flatten(const T* __restrict__ verts, const int32_t* __restrict__ edges,
                                                 T* __restrict__ loss, const T* __restrict__ gl,
                                                 T* __restrict__ gverts, int V, int E, T eps) {
    const int b = blockIdx.y;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    T acc = 0;
    if (e < E) {
        const T* vb = verts + (size_t)b * V * 3;
        const int i0 = __ldg(edges + e * 4), i1 = __ldg(edges + e * 4 + 1), i2 = __ldg(edges + e * 4 + 2), i3 = __ldg(edges + e * 4 + 3);
        T a[3], b1[3], b2[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const T p0 = vb[i0 * 3 + d];
            a[d] = vb[i1 * 3 + d] - p0;
            b1[d] = vb[i2 * 3 + d] - p0;
            b2[d] = vb[i3 * 3 + d] - p0;
        }
        Perp<T> P1, P2;
        perp_fwd(a, b1, eps, P1);
        perp_fwd(a, b2, eps, P2);
        const T num = P1.cb[0] * P2.cb[0] + P1.cb[1] * P2.cb[1] + P1.cb[2] * P2.cb[2];
        const T den = P1.l * P2.l + eps;
        const T cosd = num / den;
        acc = (cosd + 1) * (cosd + 1);
        if (BWD) {
            const T dcos = T(2) * (cosd + 1) * __ldg(gl + b);
            const T dnum = dcos / den, dden = -dcos * num / (den * den);
            T dcb1[3], dcb2[3], da[3] = {0, 0, 0}, db1[3] = {0, 0, 0}, db2[3] = {0, 0, 0};
#pragma unroll
            for (int d = 0; d < 3; ++d) { dcb1[d] = dnum * P2.cb[d]; dcb2[d] = dnum * P1.cb[d]; }
            perp_bwd(P1, dcb1, dden * P2.l, eps, da, db1);
            perp_bwd(P2, dcb2, dden * P1.l, eps, da, db2);
            if (DET) {
                T* t = gverts + ((size_t)b * E + e) * 12;
#pragma unroll
                for (int d = 0; d < 3; ++d) {
                    t[d] = -(da[d] + db1[d] + db2[d]);
                    t[3 + d] = da[d];
                    t[6 + d] = db1[d];
                    t[9 + d] = db2[d];
                }
            } else {
                T* gb = gverts + (size_t)b * V * 3;
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
        __shared__ T s[4];
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        if (lane == 0) s[warp] = acc;
        __syncthreads();
        // the four warp sums meet as (s0 + s2) + (s1 + s3) in float32 (warp_sum) and as ((s0 + s1) + s2) + s3 in float64:
        // each precision keeps the bits it always had
        if constexpr (std::is_same<T, double>::value) {
            if (threadIdx.x == 0) loss[(size_t)b * gridDim.x + blockIdx.x] = ((s[0] + s[1]) + s[2]) + s[3];
        } else if (warp == 0) {
            acc = lane < 4 ? s[lane] : T(0);
            acc = warp_sum(acc);
            if (DET) {
                if (lane == 0) loss[(size_t)b * gridDim.x + blockIdx.x] = acc;
            } else {
                if (lane == 0) atomicAdd(loss + b, acc);
            }
        }
    }
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

extern "C" int umr_create_texture_image(const float* faces_uv, const float* textures, float* image, int32_t num_faces,
                                        int32_t texture_res_in, int32_t image_height, int32_t image_width, float eps,
                                        void* stream_) {
    if (!faces_uv || !textures || !image || num_faces <= 0 || texture_res_in <= 0 || image_height <= 0 || image_width <= 0)
        return UMR_ERR_BAD_ARG;
    const int tile_width = (int)sqrt((double)(num_faces - 1)) + 1;  // create_texture_image_cuda_kernel.cu:81
    const int R_out = image_width / tile_width;                       // :82 (image.size(1) / tile_width)
    if (R_out <= 0) return UMR_ERR_BAD_ARG;
    const int64_t npix = (int64_t)image_height * image_width;
    launch(k_create_texture_image, (unsigned)((npix + 255) / 256), 256, 0, (cudaStream_t)stream_, faces_uv, textures, image,
           npix, num_faces, texture_res_in, R_out, tile_width, eps);
    return (int)cudaGetLastError();
}

extern "C" int umr_load_textures(const float* image, const float* faces_uv, const int32_t* is_update, float* textures,
                                 int32_t num_faces, int32_t texture_res, int32_t image_height, int32_t image_width,
                                 void* stream_) {
    if (!image || !faces_uv || !is_update || !textures || num_faces <= 0 || texture_res <= 0 || image_height <= 1 || image_width <= 1)
        return UMR_ERR_BAD_ARG;
    const int64_t ntexel = (int64_t)num_faces * texture_res * texture_res;
    launch(k_load_textures, (unsigned)((ntexel + 255) / 256), 256, 0, (cudaStream_t)stream_, image, faces_uv, is_update,
           textures, ntexel, texture_res, image_height, image_width);
    return (int)cudaGetLastError();
}

extern "C" int umr_laplacian_forward(const float* x, const int32_t* rowptr, const int32_t* col, const float* coef, float* y,
                                     float* loss, int32_t B, int32_t V, void* stream_) {
    if (!x || !rowptr || !col || !coef || !y || !loss || B <= 0 || V <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(loss, 0, (size_t)B * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    launch(k_laplacian_fwd<float, false>, dim3((V + 255) / 256, B), 256, 0, st, x, rowptr, col, coef, y, loss, V);
    return (int)cudaGetLastError();
}
// float32 (default and deterministic mode: one writer per element) and float64
template <typename T>
static int laplacian_backward(const T* y, const int32_t* rowptr, const int32_t* col, const T* tcoef, const T* grad_loss,
                              T* grad_x, int32_t B, int32_t V, void* stream_) {
    if (!y || !rowptr || !col || !tcoef || !grad_loss || !grad_x || B <= 0 || V <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    launch(k_laplacian_bwd<T>, dim3((V + 255) / 256, B), 256, 0, (cudaStream_t)stream_, y, rowptr, col, tcoef, grad_loss,
           grad_x, V);
    return (int)cudaGetLastError();
}
extern "C" int umr_laplacian_backward(const float* y, const int32_t* rowptr, const int32_t* col, const float* tcoef,
                                      const float* grad_loss, float* grad_x, int32_t B, int32_t V, void* stream_) {
    return laplacian_backward(y, rowptr, col, tcoef, grad_loss, grad_x, B, V, stream_);
}

extern "C" int umr_flatten_forward(const float* vertices, const int32_t* edges, float* loss, int32_t B, int32_t V, int32_t E,
                                   float eps, void* stream_) {
    if (!vertices || !edges || !loss || B <= 0 || V <= 0 || E <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(loss, 0, (size_t)B * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    launch(k_flatten<float, false, false>, dim3((E + 127) / 128, B), 128, 0, st, vertices, edges, loss, nullptr, nullptr, V, E,
           eps);
    return (int)cudaGetLastError();
}
extern "C" int umr_flatten_backward(const float* vertices, const int32_t* edges, const float* grad_loss, float* grad_vertices,
                                    int32_t B, int32_t V, int32_t E, float eps, void* stream_) {
    if (!vertices || !edges || !grad_loss || !grad_vertices || B <= 0 || V <= 0 || E <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(grad_vertices, 0, (size_t)B * V * 3 * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    launch(k_flatten<float, true, false>, dim3((E + 127) / 128, B), 128, 0, st, vertices, edges, nullptr, grad_loss,
           grad_vertices, V, E, eps);
    return (int)cudaGetLastError();
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
    launch(k_edt_columns, dim3((W + 255) / 256, B), 256, 0, st, mask, g_out, g_in, H, W);
    launch(k_edt_rows, dim3(H, B), 256, (size_t)2 * W * sizeof(int32_t), st, g_out, g_in, dt, H, W, k,
           1.f / (float)std::max(H, W));
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// deterministic float32 and float64 (include/umr_b200.h, DESIGN.md §2, §10): per-CTA partials stored in workspace slots
// and summed in ascending CTA order; the flatten backward writes per-edge terms and gathers them per vertex.  One launcher
// per op serves both precisions.
// ---------------------------------------------------------------------------------------------
template <typename T>
static size_t laplacian_workspace_bytes(int32_t B, int32_t V) {
    if (B <= 0 || V <= 0) return 0;
    return (size_t)B * ((V + 255) / 256) * sizeof(T);
}
template <typename T>
static int laplacian_forward_slots(const T* x, const int32_t* rowptr, const int32_t* col, const T* coef, T* y, T* loss,
                                   int32_t B, int32_t V, void* workspace, void* stream_) {
    if (!x || !rowptr || !col || !coef || !y || !loss || !workspace || B <= 0 || V <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const int gx = (V + 255) / 256;
    T* slots = (T*)workspace;
    launch(k_laplacian_fwd<T, true>, dim3(gx, B), 256, 0, st, x, rowptr, col, coef, y, slots, V);
    launch(k_sum_slot_rows<T>, (B + 127) / 128, 128, 0, st, slots, loss, B, gx);
    return (int)cudaGetLastError();
}
template <typename T>
static size_t flatten_forward_workspace_bytes(int32_t B, int32_t E) {
    if (B <= 0 || E <= 0) return 0;
    return (size_t)B * ((E + 127) / 128) * sizeof(T);
}
template <typename T>
static int flatten_forward_slots(const T* vertices, const int32_t* edges, T* loss, int32_t B, int32_t V, int32_t E, T eps,
                                 void* workspace, void* stream_) {
    if (!vertices || !edges || !loss || !workspace || B <= 0 || V <= 0 || E <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const int gx = (E + 127) / 128;
    T* slots = (T*)workspace;
    launch(k_flatten<T, false, true>, dim3(gx, B), 128, 0, st, vertices, edges, slots, nullptr, nullptr, V, E, eps);
    launch(k_sum_slot_rows<T>, (B + 127) / 128, 128, 0, st, slots, loss, B, gx);
    return (int)cudaGetLastError();
}
template <typename T>
static size_t flatten_backward_workspace_bytes(int32_t B, int32_t E) {
    if (B <= 0 || E <= 0) return 0;
    return (size_t)B * E * 12 * sizeof(T);
}
template <typename T>
static int flatten_backward_gather(const T* vertices, const int32_t* edges, const int32_t* vert_rowptr,
                                   const int32_t* vert_incidence, const T* grad_loss, T* grad_vertices, int32_t B, int32_t V,
                                   int32_t E, T eps, void* workspace, void* stream_) {
    if (!vertices || !edges || !vert_rowptr || !vert_incidence || !grad_loss || !grad_vertices || !workspace || B <= 0 ||
        V <= 0 || E <= 0)
        return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    T* terms = (T*)workspace;
    launch(k_flatten<T, true, true>, dim3((E + 127) / 128, B), 128, 0, st, vertices, edges, nullptr, grad_loss, terms, V, E,
           eps);
    launch(k_gather3<T>, dim3((V + 255) / 256, B), 256, 0, st, terms, vert_rowptr, vert_incidence, grad_vertices, V,
           (int64_t)E * 4);
    return (int)cudaGetLastError();
}

extern "C" size_t umr_laplacian_workspace_bytes_deterministic(int32_t B, int32_t V) { return laplacian_workspace_bytes<float>(B, V); }
extern "C" int umr_laplacian_forward_deterministic(const float* x, const int32_t* rowptr, const int32_t* col, const float* coef,
                                                   float* y, float* loss, int32_t B, int32_t V, void* workspace, void* stream_) {
    return laplacian_forward_slots(x, rowptr, col, coef, y, loss, B, V, workspace, stream_);
}
extern "C" size_t umr_flatten_forward_workspace_bytes_deterministic(int32_t B, int32_t E) {
    return flatten_forward_workspace_bytes<float>(B, E);
}
extern "C" int umr_flatten_forward_deterministic(const float* vertices, const int32_t* edges, float* loss, int32_t B, int32_t V,
                                                 int32_t E, float eps, void* workspace, void* stream_) {
    return flatten_forward_slots(vertices, edges, loss, B, V, E, eps, workspace, stream_);
}
extern "C" size_t umr_flatten_backward_workspace_bytes_deterministic(int32_t B, int32_t E) {
    return flatten_backward_workspace_bytes<float>(B, E);
}
extern "C" int umr_flatten_backward_deterministic(const float* vertices, const int32_t* edges, const int32_t* vert_rowptr,
                                                  const int32_t* vert_incidence, const float* grad_loss, float* grad_vertices,
                                                  int32_t B, int32_t V, int32_t E, float eps, void* workspace, void* stream_) {
    return flatten_backward_gather(vertices, edges, vert_rowptr, vert_incidence, grad_loss, grad_vertices, B, V, E, eps,
                                   workspace, stream_);
}

// float64 (include/umr_b200.h, "float64 loss kernels"): the deterministic structure is the only one
extern "C" size_t umr_laplacian_workspace_bytes_f64(int32_t B, int32_t V) { return laplacian_workspace_bytes<double>(B, V); }
extern "C" int umr_laplacian_forward_f64(const double* x, const int32_t* rowptr, const int32_t* col, const double* coef,
                                         double* y, double* loss, int32_t B, int32_t V, void* workspace, void* stream_) {
    return laplacian_forward_slots(x, rowptr, col, coef, y, loss, B, V, workspace, stream_);
}
extern "C" int umr_laplacian_backward_f64(const double* y, const int32_t* rowptr, const int32_t* col, const double* tcoef,
                                          const double* grad_loss, double* grad_x, int32_t B, int32_t V, void* stream_) {
    return laplacian_backward(y, rowptr, col, tcoef, grad_loss, grad_x, B, V, stream_);
}
extern "C" size_t umr_flatten_forward_workspace_bytes_f64(int32_t B, int32_t E) { return flatten_forward_workspace_bytes<double>(B, E); }
extern "C" int umr_flatten_forward_f64(const double* vertices, const int32_t* edges, double* loss, int32_t B, int32_t V,
                                       int32_t E, double eps, void* workspace, void* stream_) {
    return flatten_forward_slots(vertices, edges, loss, B, V, E, eps, workspace, stream_);
}
extern "C" size_t umr_flatten_backward_workspace_bytes_f64(int32_t B, int32_t E) { return flatten_backward_workspace_bytes<double>(B, E); }
extern "C" int umr_flatten_backward_f64(const double* vertices, const int32_t* edges, const int32_t* vert_rowptr,
                                        const int32_t* vert_incidence, const double* grad_loss, double* grad_vertices,
                                        int32_t B, int32_t V, int32_t E, double eps, void* workspace, void* stream_) {
    return flatten_backward_gather(vertices, edges, vert_rowptr, vert_incidence, grad_loss, grad_vertices, B, V, E, eps,
                                   workspace, stream_);
}
