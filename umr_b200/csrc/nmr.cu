// nmr.cu -- hard z-buffer renderer with NMR's conventions (the `neural_renderer.Renderer` that UMR builds for its
// textured visuals, experiments/train_s2.py:111-113, demo.py:64-67, and for MultiTextureLoss(renderer="nmr"),
// loss_utils.py:282-285,309-311).  The render contract is DESIGN.md §7; oracle/nmr.py restates it in numpy.
//
//   k_nmr_prep     one thread per (image, face copy): gather, two-sided light, look_at translation, a 128-byte
//                  record (NDC vertices, depths, pixel-unit barycentric inverse, light) and the pixel box.
//   k_nmr_zbuf     one CTA per 64x64 raster bin: a z-buffer of packed (depth bits << 32 | face copy) keys in shared
//                  memory (the k_visible_faces scheme); warps take 32-face chunks, ballot the faces whose box meets
//                  the bin and test only the pixels of box x bin; atomicMin keeps the lexicographic minimum of
//                  (depth, face), which is NMR's ascending strict-'<' walk.  Writes the face-index and depth planes.
//   k_nmr_shade    thread = 4 output pixels: texture cube, light, background, vertical flip and the 2x2 pool fused,
//                  128-bit stores.  The winner's barycentrics are recomputed with the z-buffer's exact op sequence.
//   k_nmr_bwd_tex  thread = output pixel: the texture adjoint of k_nmr_shade, red.global into [B/G, F, T^3, 3].
//   k_nmr_shade_raster / k_nmr_grad_faces  the functional rasteriser's geometry gradient (DESIGN.md §14): the raster-
//                  resolution colour plane, then one warp per face for NMR's edge term and the depth term.
//   k_nmr_light_fwd / k_nmr_light_bwd / k_nmr_light_reduce  neural_renderer.lighting (DESIGN.md §15), float and double:
//                  textures * light per face, and its gradients with one warp per face and no atomics.
//
// Compiled with -fmad=false (umr_b200/build.py): every product and sum rounds once, in the contract's order.
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "umr_b200.h"

namespace umr {
namespace nmr {

constexpr int REC = 32;  // floats per face-copy record (128 B)
constexpr int R_X = 0;   // 6: x0 y0 x1 y1 x2 y2 (NDC)
constexpr int R_Z = 6;   // 3: z0 z1 z2 (after look_at)
constexpr int R_INV = 9; // 9: barycentric inverse in pixel units, row-major
constexpr int R_L = 18;  // 3: light rgb
constexpr int BIN = 64;  // z-buffer bin side (raster pixels)
constexpr int CTA = 256;
constexpr int NWARP = CTA / 32;

struct Consts {
    int B, V, F, Fc, T, S, IS, aa, tex_div;
    float eye_z, near_, far_, Ia, Id;
    float ca[3], cd[3], dir[3], bg[3];
};

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
inline size_t rec_bytes(int B, int Fc) { return align256((size_t)B * Fc * REC * sizeof(float)); }
inline size_t box_bytes(int B, int Fc) { return align256((size_t)B * Fc * sizeof(int4)); }

// (2 i + 1 - S) / S, evaluated by NMR in double and stored as float: one float division is bit-identical
// (double rounding is innocuous for a quotient of two floats, see raster.cu pixel_coord)
__device__ __forceinline__ float pixel_coord(int i, int S) { return __fdiv_rn((float)(2 * i + 1 - S), (float)S); }

// ---------------------------------------------------------------------------------------------
// per-face light (DESIGN.md §7 step 2), shared by k_nmr_prep and the lighting kernels (§15)
// ---------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ T light_eps();
template <> __device__ __forceinline__ float light_eps<float>() { return 1e-5f; }
template <> __device__ __forceinline__ double light_eps<double>() { return 1e-5; }

// the intermediates the lighting backward chains through
template <typename T>
struct LightParts {
    T a[3], b[3];  // v0 - v1, v2 - v1
    T nrm, den;    // |cross|, max(|cross|, eps)
    T n[3];        // normal
    T cs;          // relu(n . d)
};

// n = normalize(cross(v0 - v1, v2 - v1), eps=1e-5), light = Ia*ca + Id*(cd*relu(n.d)); a term whose intensity is 0 is
// not added
template <typename T>
__device__ __forceinline__ void face_light(const T v[3][3], T Ia, T Id, const T* ca, const T* cd, const T* dir, T l[3],
                                           LightParts<T>* q) {
    const T ax = v[0][0] - v[1][0], ay = v[0][1] - v[1][1], az = v[0][2] - v[1][2];
    const T bx = v[2][0] - v[1][0], by = v[2][1] - v[1][1], bz = v[2][2] - v[1][2];
    const T c0 = ay * bz - az * by, c1 = az * bx - ax * bz, c2 = ax * by - ay * bx;
    const T nrm = sqrt((c0 * c0 + c1 * c1) + c2 * c2);
    const T den = fmax(nrm, light_eps<T>());
    const T n0 = c0 / den, n1 = c1 / den, n2 = c2 / den;
    T cs = (n0 * dir[0] + n1 * dir[1]) + n2 * dir[2];
    cs = cs < T(0) ? T(0) : cs;  // relu (NaN stays NaN)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        T lc = T(0);
        if (Ia != T(0)) lc = lc + Ia * ca[c];
        if (Id != T(0)) lc = lc + Id * (cd[c] * cs);
        l[c] = lc;
    }
    if (q) {  // NULL where only the light is wanted (k_nmr_prep)
        q->a[0] = ax; q->a[1] = ay; q->a[2] = az;
        q->b[0] = bx; q->b[1] = by; q->b[2] = bz;
        q->nrm = nrm;
        q->den = den;
        q->n[0] = n0; q->n[1] = n1; q->n[2] = n2;
        q->cs = cs;
    }
}

// ---------------------------------------------------------------------------------------------
// prep
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_nmr_prep(const float* __restrict__ verts, const int32_t* __restrict__ faces,
                                                  float* __restrict__ rec, int4* __restrict__ box, Consts K) {
    const int fc = blockIdx.x * blockDim.x + threadIdx.x;
    if (fc >= K.Fc) return;
    const int b = blockIdx.y;
    const int f = fc < K.F ? fc : fc - K.F;
    const int32_t* fi = faces + ((size_t)b * K.F + f) * 3;
    int id[3] = {__ldg(fi), __ldg(fi + 1), __ldg(fi + 2)};
    if (fc >= K.F) { const int t = id[0]; id[0] = id[2]; id[2] = t; }  // fill_back copy: vertex order reversed
    float v[3][3];
    const float qnan = __int_as_float(0x7fffffff);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const bool ok = id[k] >= 0 && id[k] < K.V;  // an out-of-range index is never dereferenced: NaN face, never drawn
        const float* p = verts + ((size_t)b * K.V + (ok ? id[k] : 0)) * 3;
#pragma unroll
        for (int d = 0; d < 3; ++d) v[k][d] = ok ? __ldg(p + d) : qnan;
    }
    float out[REC];
#pragma unroll
    for (int k = 0; k < REC; ++k) out[k] = 0.f;
    // light from the vertices before look_at
    {
        float l[3];
        face_light<float>(v, K.Ia, K.Id, K.ca, K.cd, K.dir, l, nullptr);
#pragma unroll
        for (int c = 0; c < 3; ++c) out[R_L + c] = l[c];
    }
    const float Sf = (float)K.S;
    float px[3], py[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        out[R_X + 2 * k] = v[k][0];
        out[R_X + 2 * k + 1] = v[k][1];
        out[R_Z + k] = v[k][2] - K.eye_z;  // look_at with eye (0, 0, e): a translation along z
        px[k] = 0.5f * ((v[k][0] * Sf + Sf) - 1.f);
        py[k] = 0.5f * ((v[k][1] * Sf + Sf) - 1.f);
    }
    {
        float inv[9] = {py[1] - py[2], px[2] - px[1], px[1] * py[2] - px[2] * py[1],
                        py[2] - py[0], px[0] - px[2], px[2] * py[0] - px[0] * py[2],
                        py[0] - py[1], px[1] - px[0], px[0] * py[1] - px[1] * py[0]};
        const float den = (px[2] * (py[0] - py[1]) + px[0] * (py[1] - py[2])) + px[1] * (py[2] - py[0]);
#pragma unroll
        for (int k = 0; k < 9; ++k) out[R_INV + k] = inv[k] / den;
    }
    float4* dst = reinterpret_cast<float4*>(rec + ((size_t)b * K.Fc + fc) * REC);
#pragma unroll
    for (int k = 0; k < REC / 4; ++k) dst[k] = make_float4(out[4 * k], out[4 * k + 1], out[4 * k + 2], out[4 * k + 3]);

    // pixel box.  A back-facing copy is never drawn: empty box.
    const float x0 = v[0][0], y0 = v[0][1], x1 = v[1][0], y1 = v[1][1], x2 = v[2][0], y2 = v[2][1];
    int4 bb;
    if ((y2 - y0) * (x1 - x0) < (y1 - y0) * (x2 - x0)) {
        bb = make_int4(1, 0, 1, 0);
    } else {
        // The float edge tests admit a pixel at most ~6 ulp * |p - v| beyond an edge line, which is within
        // 2e-4 * (1 + max|coord|) NDC of the triangle while its smallest angle has a sine >= 1e-2.  Thinner
        // (or NaN) faces are tested on every pixel of the image.
        const float l01 = (x1 - x0) * (x1 - x0) + (y1 - y0) * (y1 - y0);
        const float l02 = (x2 - x0) * (x2 - x0) + (y2 - y0) * (y2 - y0);
        const float l12 = (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1);
        const float lmin = fminf(fminf(l01, l02), l12);
        const float prod2 = (l01 * l02 * l12) / fmaxf(lmin, 1e-30f);  // product of the two longest squared edges
        const float a2 = x2 * (y0 - y1) + x0 * (y1 - y2) + x1 * (y2 - y0);
        const float m = fmaxf(fmaxf(fmaxf(fabsf(x0), fabsf(x1)), fmaxf(fabsf(x2), fabsf(y0))), fmaxf(fabsf(y1), fabsf(y2)));
        if (!(a2 * a2 >= 1e-4f * prod2) || !(m < 1e6f)) {
            bb = make_int4(0, K.S - 1, 0, K.S - 1);
        } else {
            const float marg = 2.f + 2e-4f * (1.f + m) * Sf;
            const float lo_x = fminf(fminf(px[0], px[1]), px[2]) - marg, hi_x = fmaxf(fmaxf(px[0], px[1]), px[2]) + marg;
            const float lo_y = fminf(fminf(py[0], py[1]), py[2]) - marg, hi_y = fmaxf(fmaxf(py[0], py[1]), py[2]) + marg;
            // clamped to [-1, S] in float before the conversion to int
            bb.x = max((int)floorf(fmaxf(lo_x, -1.f)), 0);
            bb.y = min((int)ceilf(fminf(hi_x, Sf)), K.S - 1);
            bb.z = max((int)floorf(fmaxf(lo_y, -1.f)), 0);
            bb.w = min((int)ceilf(fminf(hi_y, Sf)), K.S - 1);
        }
    }
    box[(size_t)b * K.Fc + fc] = bb;
}

// ---------------------------------------------------------------------------------------------
// shared per-(pixel, face) arithmetic: the contract's op order, identical in every kernel
// ---------------------------------------------------------------------------------------------
// w = clamp01(face_inv . (xi, yi, 1)) / sum;  zp = 1 / (w0/z0 + w1/z1 + w2/z2)
__device__ __forceinline__ void bary(const float* __restrict__ rc, int xi, int yi, float w[3], float& zp) {
    const float fx = (float)xi, fy = (float)yi;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float t = (__ldg(rc + R_INV + 3 * k) * fx + __ldg(rc + R_INV + 3 * k + 1) * fy) + __ldg(rc + R_INV + 3 * k + 2);
        t = fminf(fmaxf(t, 0.f), 1.f);  // NMR clamps with double literals: a selection, NaN -> 0 like fmax
        w[k] = t;
        s = s + t;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) w[k] = w[k] / s;
    const float z0 = __ldg(rc + R_Z), z1 = __ldg(rc + R_Z + 1), z2 = __ldg(rc + R_Z + 2);
    zp = __fdiv_rn(1.f, (w[0] / z0 + w[1] / z1) + w[2] / z2);  // 1. / x in double, stored as float: same bits
}

// trilinear sample of the T^3 cube at the winner's barycentrics; calls fn(texel, weight) for the 8 corners in
// NMR's order.  `texel` indexes the ORIGINAL cube: a fill_back copy reads (t2, t1, t0).
template <typename Fn>
__device__ __forceinline__ void corners(const float w[3], float zp, const float* __restrict__ rc, int T, bool back,
                                        Fn fn) {
    const float tm1 = (float)(T - 1), lim = (float)(T - 1) - 1e-3f;
    float tif[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float t = (w[k] * tm1) * (zp / __ldg(rc + R_Z + k));
        tif[k] = fminf(fmaxf(t, 0.f), lim);
    }
#pragma unroll
    for (int pn = 0; pn < 8; ++pn) {
        float wt = 1.f;
        int i[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            int ti = (int)tif[k];
            if (((pn >> k) & 1) == 0) {
                wt = wt * (1.f - (tif[k] - (float)ti));
            } else {
                wt = wt * (tif[k] - (float)ti);
                ti += 1;
            }
            i[k] = ti;
        }
        const int idx = back ? (i[2] * T + i[1]) * T + i[0] : (i[0] * T + i[1]) * T + i[2];
        fn(idx, wt);
    }
}

// ---------------------------------------------------------------------------------------------
// z-buffer
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(CTA) k_nmr_zbuf(const float* __restrict__ rec, const int4* __restrict__ box,
                                                  int32_t* __restrict__ face_index, float* __restrict__ rdepth, Consts K) {
    __shared__ unsigned long long s_z[BIN * BIN];  // 32 KB
    __shared__ int s_next;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z, S = K.S, Fc = K.Fc;
    const int bx0 = blockIdx.x * BIN, by0 = blockIdx.y * BIN;
    const int bx1 = min(bx0 + BIN, S) - 1, by1 = min(by0 + BIN, S) - 1;
    for (int i = tid; i < BIN * BIN; i += CTA) s_z[i] = ~0ull;
    if (tid == 0) s_next = NWARP;
    __syncthreads();
    const float* rec_img = rec + (size_t)b * Fc * REC;
    const int4* box_img = box + (size_t)b * Fc;
    const int nchunk = (Fc + 31) / 32;
    // 32-face chunks handed out from a shared counter: face boxes differ by orders of magnitude
    for (int c = warp; c < nchunk;) {
        const int f = c * 32 + lane;
        int4 bb = make_int4(1, 0, 1, 0);
        if (f < Fc) bb = __ldg(box_img + f);
        const bool hit = bb.x <= bb.y && bb.z <= bb.w && bb.x <= bx1 && bb.y >= bx0 && bb.z <= by1 && bb.w >= by0;
        unsigned m = __ballot_sync(0xffffffffu, hit);
        while (m) {
            const int l = __ffs(m) - 1;
            m &= m - 1;
            const int ff = c * 32 + l;
            const int c0 = max(__shfl_sync(0xffffffffu, bb.x, l), bx0), c1 = min(__shfl_sync(0xffffffffu, bb.y, l), bx1);
            const int r0 = max(__shfl_sync(0xffffffffu, bb.z, l), by0), r1 = min(__shfl_sync(0xffffffffu, bb.w, l), by1);
            const int w = c1 - c0 + 1, n = w * (r1 - r0 + 1);
            const float* rc = rec_img + (size_t)ff * REC;
            const float x0 = __ldg(rc + 0), y0 = __ldg(rc + 1), x1 = __ldg(rc + 2), y1 = __ldg(rc + 3);
            const float x2 = __ldg(rc + 4), y2 = __ldg(rc + 5);
            for (int p = lane; p < n; p += 32) {
                const int lr = p / w, xi = c0 + (p - lr * w), yi = r0 + lr;
                const float xp = pixel_coord(xi, S), yp = pixel_coord(yi, S);
                if ((yp - y0) * (x1 - x0) < (xp - x0) * (y1 - y0) || (yp - y1) * (x2 - x1) < (xp - x1) * (y2 - y1) ||
                    (yp - y2) * (x0 - x2) < (xp - x2) * (y0 - y2))
                    continue;
                float wb[3], zp;
                bary(rc, xi, yi, wb, zp);
                if (!(zp > K.near_ && zp < K.far_)) continue;  // zp <= near, zp >= far or NaN
                // -0 packs as +0: NMR's '<' does not order them (near < 0 admits both); the epilogue restores the sign
                uint32_t zb = __float_as_uint(zp == 0.f ? 0.f : zp);
                zb = (zb & 0x80000000u) ? ~zb : (zb | 0x80000000u);  // total order of floats as unsigned integers
                atomicMin(&s_z[(yi - by0) * BIN + (xi - bx0)], ((unsigned long long)zb << 32) | (uint32_t)ff);
            }
        }
        int nx = 0;
        if (lane == 0) nx = atomicAdd(&s_next, 1);
        c = __shfl_sync(0xffffffffu, nx, 0);
    }
    __syncthreads();
    for (int i = tid; i < BIN * BIN; i += CTA) {
        const int row = i / BIN, col = i - row * BIN;
        if (by0 + row > by1 || bx0 + col > bx1) continue;
        const unsigned long long key = s_z[i];
        int32_t fi = -1;
        float z = K.far_;
        if (key != ~0ull) {
            fi = (int32_t)(uint32_t)(key & 0xffffffffull);
            uint32_t zb = (uint32_t)(key >> 32);
            zb = (zb & 0x80000000u) ? (zb & 0x7fffffffu) : ~zb;
            z = __uint_as_float(zb);
            if (z == 0.f) {  // the winner's own zero, sign included
                float wb[3];
                bary(rec_img + (size_t)fi * REC, bx0 + col, by0 + row, wb, z);
            }
        }
        const size_t o = ((size_t)b * S + by0 + row) * S + bx0 + col;
        face_index[o] = fi;
        rdepth[o] = z;
    }
}

// ---------------------------------------------------------------------------------------------
// shading: texture, light, background, flip, pool
// ---------------------------------------------------------------------------------------------
// colour of raster pixel (xi, yi) won by face copy fi >= 0
__device__ __forceinline__ void shade_color(const float* __restrict__ rec, const float* __restrict__ textures,
                                            const Consts& K, int b, int fi, int xi, int yi, float rgb[3]) {
    const float* rc = rec + ((size_t)b * K.Fc + fi) * REC;
    float w[3], zp;
    bary(rc, xi, yi, w, zp);
    const bool back = fi >= K.F;
    const int f = back ? fi - K.F : fi;
    const int T3 = K.T * K.T * K.T;
    const float* tex = textures + ((size_t)(b / K.tex_div) * K.F + f) * T3 * 3;
    const float l0 = __ldg(rc + R_L), l1 = __ldg(rc + R_L + 1), l2 = __ldg(rc + R_L + 2);
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    corners(w, zp, rc, K.T, back, [&](int idx, float wt) {
        const float* t = tex + (size_t)idx * 3;
        s0 = s0 + wt * (__ldg(t) * l0);  // the texel is lit before blending (textures *= light)
        s1 = s1 + wt * (__ldg(t + 1) * l1);
        s2 = s2 + wt * (__ldg(t + 2) * l2);
    });
    rgb[0] = s0; rgb[1] = s1; rgb[2] = s2;
}

// one raster pixel
__device__ __forceinline__ void shade_px(const float* __restrict__ rec, const int32_t* __restrict__ face_index,
                                         const float* __restrict__ rdepth, const float* __restrict__ textures,
                                         const Consts& K, int b, int xi, int yi, float rgb[3], float& a, float& d) {
    const size_t o = ((size_t)b * K.S + yi) * K.S + xi;
    const int fi = __ldg(face_index + o);
    d = __ldg(rdepth + o);
    if (fi < 0) {
        a = 0.f;
        rgb[0] = K.bg[0]; rgb[1] = K.bg[1]; rgb[2] = K.bg[2];
        return;
    }
    a = 1.f;
    if (textures == nullptr) return;
    shade_color(rec, textures, K, b, fi, xi, yi, rgb);
}

// V output pixels per thread (4: 128-bit stores).  rgb [B,3,is,is], alpha / depth [B,is,is]; any may be NULL.
template <int V>
__global__ void __launch_bounds__(256) k_nmr_shade(const float* __restrict__ rec, const int32_t* __restrict__ face_index,
                                                   const float* __restrict__ rdepth, const float* __restrict__ textures,
                                                   float* __restrict__ rgb, float* __restrict__ alpha,
                                                   float* __restrict__ depth, Consts K) {
    const int IS = K.IS, ng = IS / V;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)K.B * IS * ng) return;
    const int g = (int)(t % ng), r = (int)((t / ng) % IS), b = (int)(t / ((size_t)ng * IS));
    float oc[3][V], oa[V], od[V];
#pragma unroll
    for (int v = 0; v < V; ++v) {
        const int c = g * V + v;
        float pc[3], pa, pd;
        if (K.aa) {
            // flipped image row-major over the 2x2 window: raster rows S-1-2r, then S-2-2r; columns 2c, 2c+1
            float sc[3] = {0.f, 0.f, 0.f}, sa = 0.f, sd = 0.f;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int yi = K.S - 1 - 2 * r - (q >> 1), xi = 2 * c + (q & 1);
                float qc[3], qa, qd;
                shade_px(rec, face_index, rdepth, textures, K, b, xi, yi, qc, qa, qd);
                sc[0] = sc[0] + qc[0]; sc[1] = sc[1] + qc[1]; sc[2] = sc[2] + qc[2];
                sa = sa + qa;
                sd = sd + qd;
            }
            pc[0] = sc[0] / 4.f; pc[1] = sc[1] / 4.f; pc[2] = sc[2] / 4.f;
            pa = sa / 4.f;
            pd = sd / 4.f;
        } else {
            shade_px(rec, face_index, rdepth, textures, K, b, c, K.S - 1 - r, pc, pa, pd);
        }
        oc[0][v] = pc[0]; oc[1][v] = pc[1]; oc[2][v] = pc[2];
        oa[v] = pa;
        od[v] = pd;
    }
    const size_t plane = (size_t)IS * IS, o = (size_t)r * IS + (size_t)g * V;
    auto store = [&](float* dst, const float* s) {
        if constexpr (V == 4) *reinterpret_cast<float4*>(dst) = make_float4(s[0], s[1], s[2], s[3]);
        else dst[0] = s[0];
    };
    if (rgb) {
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) store(rgb + ((size_t)b * 3 + ch) * plane + o, oc[ch]);
    }
    if (alpha) store(alpha + (size_t)b * plane + o, oa);
    if (depth) store(depth + (size_t)b * plane + o, od);
}

// ---------------------------------------------------------------------------------------------
// texture gradient: grad_rgb [B,3,is,is] -> grad_textures [B/G, F, T^3, 3] (zero-filled by the caller)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_nmr_bwd_tex(const float* __restrict__ rec, const int32_t* __restrict__ face_index,
                                                     const float* __restrict__ grad_rgb, float* __restrict__ grad_tex,
                                                     Consts K) {
    const int IS = K.IS;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)K.B * IS * IS) return;
    const int c = (int)(t % IS), r = (int)((t / IS) % IS), b = (int)(t / ((size_t)IS * IS));
    const size_t plane = (size_t)IS * IS, o = (size_t)r * IS + c;
    float g[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) g[ch] = __ldg(grad_rgb + ((size_t)b * 3 + ch) * plane + o);
    if (K.aa) { g[0] = g[0] / 4.f; g[1] = g[1] / 4.f; g[2] = g[2] / 4.f; }
    if (g[0] == 0.f && g[1] == 0.f && g[2] == 0.f) return;
    const int T3 = K.T * K.T * K.T;
    const int nq = K.aa ? 4 : 1;
    for (int q = 0; q < nq; ++q) {
        const int yi = K.aa ? K.S - 1 - 2 * r - (q >> 1) : K.S - 1 - r;
        const int xi = K.aa ? 2 * c + (q & 1) : c;
        const int fi = __ldg(face_index + ((size_t)b * K.S + yi) * K.S + xi);
        if (fi < 0) continue;
        const float* rc = rec + ((size_t)b * K.Fc + fi) * REC;
        float w[3], zp;
        bary(rc, xi, yi, w, zp);
        const bool back = fi >= K.F;
        const int f = back ? fi - K.F : fi;
        float* gt = grad_tex + ((size_t)(b / K.tex_div) * K.F + f) * T3 * 3;
        const float l0 = __ldg(rc + R_L), l1 = __ldg(rc + R_L + 1), l2 = __ldg(rc + R_L + 2);
        corners(w, zp, rc, K.T, back, [&](int idx, float wt) {
            red_add3_global(gt + (size_t)idx * 3, (l0 * wt) * g[0], (l1 * wt) * g[1], (l2 * wt) * g[2]);
        });
    }
}

// ---------------------------------------------------------------------------------------------
// deterministic texture gradient: a face-parallel gather.  One warp per (texture group, face f) is the only writer of
// face f's texels.  It walks the group's G images in ascending order; in each, copy f and then (fill_back) copy F + f;
// for each copy the pixel box of k_nmr_prep (the one k_nmr_zbuf tests, so it holds every pixel the copy can win) in
// ascending rows, lanes over 32-pixel row segments.  A raster pixel the copy won contributes k_nmr_bwd_tex's terms.
// Per corner, the lanes that hit one texel are summed in ascending lane order and the lowest of them adds the sum in.
// ---------------------------------------------------------------------------------------------
constexpr int DET_WARPS = 8;

__global__ void __launch_bounds__(DET_WARPS * 32) k_nmr_bwd_tex_det(const float* __restrict__ rec, const int4* __restrict__ box,
                                                                    const int32_t* __restrict__ face_index,
                                                                    const float* __restrict__ grad_rgb,
                                                                    float* __restrict__ grad_tex, Consts K) {
    __shared__ float s_v[DET_WARPS][3][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long gw = (long long)blockIdx.x * DET_WARPS + warp;
    if (gw >= (long long)(K.B / K.tex_div) * K.F) return;  // whole warps
    const int grp = (int)(gw / K.F), f = (int)(gw - (long long)grp * K.F);
    const int T3 = K.T * K.T * K.T, IS = K.IS, S = K.S;
    const size_t plane = (size_t)IS * IS;
    float* gt = grad_tex + ((size_t)grp * K.F + f) * T3 * 3;
    for (int i = 0; i < K.tex_div; ++i) {
        const int b = grp * K.tex_div + i;
        for (int fc = f; fc < K.Fc; fc += K.F) {
            const int4 bb = __ldg(box + (size_t)b * K.Fc + fc);
            const bool back = fc >= K.F;
            const float* rc = rec + ((size_t)b * K.Fc + fc) * REC;
            const float l0 = __ldg(rc + R_L), l1 = __ldg(rc + R_L + 1), l2 = __ldg(rc + R_L + 2);
            for (int yi = bb.z; yi <= bb.w; ++yi) {
                const int r = K.aa ? (S - 1 - yi) >> 1 : S - 1 - yi;
                for (int xs = bb.x; xs <= bb.y; xs += 32) {
                    const int xi = xs + lane;
                    float g[3] = {0.f, 0.f, 0.f};
                    bool hit = false;
                    if (xi <= bb.y && __ldg(face_index + ((size_t)b * S + yi) * S + xi) == fc) {
                        const size_t o = (size_t)r * IS + (K.aa ? xi >> 1 : xi);
#pragma unroll
                        for (int ch = 0; ch < 3; ++ch) g[ch] = __ldg(grad_rgb + ((size_t)b * 3 + ch) * plane + o);
                        if (K.aa) { g[0] = g[0] / 4.f; g[1] = g[1] / 4.f; g[2] = g[2] / 4.f; }
                        hit = !(g[0] == 0.f && g[1] == 0.f && g[2] == 0.f);
                    }
                    if (!__any_sync(0xffffffffu, hit)) continue;
                    int idx[8];
                    float wt[8];
#pragma unroll
                    for (int pn = 0; pn < 8; ++pn) { idx[pn] = -1; wt[pn] = 0.f; }
                    if (hit) {
                        float w[3], zp;
                        bary(rc, xi, yi, w, zp);
                        int pn = 0;
                        corners(w, zp, rc, K.T, back, [&](int id, float wgt) { idx[pn] = id; wt[pn] = wgt; ++pn; });
                    }
#pragma unroll
                    for (int pn = 0; pn < 8; ++pn) {
                        const unsigned same = __match_any_sync(0xffffffffu, idx[pn]);
                        s_v[warp][0][lane] = (l0 * wt[pn]) * g[0];
                        s_v[warp][1][lane] = (l1 * wt[pn]) * g[1];
                        s_v[warp][2][lane] = (l2 * wt[pn]) * g[2];
                        __syncwarp();
                        if (hit && lane == __ffs(same) - 1) {
                            float a0 = 0.f, a1 = 0.f, a2 = 0.f;
                            for (unsigned m = same; m; m &= m - 1) {
                                const int l = __ffs(m) - 1;
                                a0 = a0 + s_v[warp][0][l];
                                a1 = a1 + s_v[warp][1][l];
                                a2 = a2 + s_v[warp][2][l];
                            }
                            float* t = gt + (size_t)idx[pn] * 3;
                            t[0] = t[0] + a0; t[1] = t[1] + a1; t[2] = t[2] + a2;
                        }
                        __syncwarp();
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// geometry gradient (DESIGN.md §14): NMR's approximate edge gradient plus the analytic depth gradient
// ---------------------------------------------------------------------------------------------
// raster-resolution colour plane [B,S,S,3] (background where no face wins), k_nmr_shade's op sequence per pixel
__global__ void __launch_bounds__(256) k_nmr_shade_raster(const float* __restrict__ rec, const int32_t* __restrict__ face_index,
                                                          const float* __restrict__ textures, float* __restrict__ color,
                                                          Consts K) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t plane = (size_t)K.S * K.S;
    if (t >= (size_t)K.B * plane) return;
    const int b = (int)(t / plane), yi = (int)((t % plane) / K.S), xi = (int)(t % K.S);
    const int fi = __ldg(face_index + t);
    float c[3] = {K.bg[0], K.bg[1], K.bg[2]};
    if (fi >= 0) shade_color(rec, textures, K, b, fi, xi, yi, c);
    float* o = color + t * 3;
    o[0] = c[0]; o[1] = c[1]; o[2] = c[2];
}

// The output-resolution adjoint planes read at raster pixel (xi, yi): flip, then the 2x2 pool's 1/4.
struct GradPlanes {
    const float* rgb;    // [B,3,is,is] or NULL
    const float* alpha;  // [B,is,is] or NULL
    const float* depth;  // [B,is,is] or NULL
    const float* color;  // raster colour plane [B,S,S,3] (with rgb)
    const int32_t* fidx; // [B,S,S]
};

__device__ __forceinline__ size_t out_index(const Consts& K, int b, int xi, int yi) {
    const int r = K.aa ? (K.S - 1 - yi) >> 1 : K.S - 1 - yi;
    const int c = K.aa ? xi >> 1 : xi;
    return ((size_t)b * K.IS + r) * K.IS + c;
}

__device__ __forceinline__ float out_grad(const Consts& K, const float* g, size_t o) {
    const float v = __ldg(g + o);
    return K.aa ? v / 4.f : v;
}

// the channels the edge term compares: alpha, then rgb
struct Px {
    float a, c[3];
};

__device__ __forceinline__ Px px_value(const GradPlanes& G, const Consts& K, int b, int xi, int yi) {
    const size_t o = ((size_t)b * K.S + yi) * K.S + xi;
    Px v;
    v.a = __ldg(G.fidx + o) >= 0 ? 1.f : 0.f;
    if (G.rgb) {
        v.c[0] = __ldg(G.color + o * 3); v.c[1] = __ldg(G.color + o * 3 + 1); v.c[2] = __ldg(G.color + o * 3 + 2);
    } else {
        v.c[0] = v.c[1] = v.c[2] = 0.f;
    }
    return v;
}

// diff = sum over the requested channels of (I_p - I_ref) * g_p, alpha first, then r, g, b
__device__ __forceinline__ float edge_diff(const GradPlanes& G, const Consts& K, int b, int xi, int yi, const Px& ref) {
    const Px p = px_value(G, K, b, xi, yi);
    const size_t o = out_index(K, b, xi, yi);
    const size_t plane = (size_t)K.IS * K.IS;
    float diff = 0.f;
    if (G.alpha) diff = diff + (p.a - ref.a) * out_grad(K, G.alpha, o);
    if (G.rgb) {
        const size_t oc = o + (size_t)b * 2 * plane;  // [B,3,is,is]: b * 3 * plane + ch * plane + pixel
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) diff = diff + (p.c[ch] - ref.c[ch]) * out_grad(K, G.rgb, oc + ch * plane);
    }
    return diff;
}

// One edge term at walk pixel d1 of line d0, skipped unless diff > 0: -diff / dist to the line's vertex a (ga) and b (gb),
// dist moved away from zero by eps.
__device__ __forceinline__ void edge_term(float& ga, float& gb, float diff, int d1, float vc, float ua, float ub, float d0f,
                                          float Sf, float eps) {
    if (!(diff > 0.f)) return;
    const float dd = (float)d1 - vc;
    if (ub != d0f) {
        float dist = ((((ub - ua) / (ub - d0f)) * dd) * 2.f) / Sf;
        dist = dist > 0.f ? dist + eps : dist - eps;
        ga = ga - diff / dist;
    }
    if (ua != d0f) {
        float dist = ((((ub - ua) / (d0f - ua)) * dd) * 2.f) / Sf;
        dist = dist > 0.f ? dist + eps : dist - eps;
        gb = gb - diff / dist;
    }
}

__device__ __forceinline__ float sel3(const float a[3], int k) { return k == 0 ? a[0] : (k == 1 ? a[1] : a[2]); }

// Line (e, axis, d0) of face f: the growing walk (only when the 'in' pixel is this face's) and the shrinking walk.
// Returns the line's sums for the moving coordinate of vertex a = e (ga) and b = e + 1 (gb).
__device__ __forceinline__ void edge_line(float& ga, float& gb, const GradPlanes& G, const Consts& K, int b, int f, const float px[3],
                          const float py[3], int e, int axis, int d0, float eps) {
    const int S = K.S;
    const float Sf = (float)S, d0f = (float)d0;
    const int ka = e, kb = e == 2 ? 0 : e + 1, ko = e == 0 ? 2 : e - 1;
    const float ua = sel3(axis == 0 ? px : py, ka), ub = sel3(axis == 0 ? px : py, kb), uo = sel3(axis == 0 ? px : py, ko);
    const float va = sel3(axis == 0 ? py : px, ka), vb = sel3(axis == 0 ? py : px, kb), vo = sel3(axis == 0 ? py : px, ko);
    const int dir = axis == 0 ? (ua < ub ? -1 : 1) : (ua < ub ? 1 : -1);
    const float vc = ((vb - va) / (ub - ua)) * (d0f - ua) + va;
    const float fin = dir > 0 ? floorf(vc) : ceilf(vc);
    if (!(fin >= 0.f && fin <= Sf - 1.f)) return;  // NaN included
    const int in = (int)fin, out = in + dir;
    if (out < 0 || out >= S) return;
    // raster pixel of walk position d1: axis 0 walks a column (x = d0), axis 1 a row (y = d0)
    const int step = axis == 0 ? S : 1;
    const int base = axis == 0 ? d0 : d0 * S;
    const size_t img = (size_t)b * S * S;
    auto xy = [&](int d1, int& xi, int& yi) {
        if (axis == 0) { xi = d0; yi = d1; } else { xi = d1; yi = d0; }
    };
    int xi, yi;
    xy(in, xi, yi);
    const Px I_in = px_value(G, K, b, xi, yi);
    const bool in_is_f = __ldg(G.fidx + img + base + in * step) == f;
    xy(out, xi, yi);
    const Px I_out = px_value(G, K, b, xi, yi);
    // growing: from 'out' to the border in direction dir, every pixel compared with I_in
    if (in_is_f) {
        const int p0 = dir > 0 ? out : 0, p1 = dir > 0 ? S - 1 : out;
        for (int p = p0; p <= p1; ++p) {
            xy(p, xi, yi);
            edge_term(ga, gb, edge_diff(G, K, b, xi, yi, I_in), p, vc, ua, ub, d0f, Sf, eps);
        }
    }
    // shrinking: from 'in' to where the line u = d0 meets the other edge (rounded outward), this face's pixels only
    float x;
    if ((d0f - ua) * (d0f - uo) < 0.f) x = ((vo - va) / (uo - ua)) * (d0f - ua) + va;
    else x = ((vb - vo) / (ub - uo)) * (d0f - uo) + vo;
    float lf = dir > 0 ? ceilf(x) : floorf(x);
    lf = lf != lf ? fin : fminf(fmaxf(lf, -1.f), Sf);  // NaN: the 'in' pixel alone; clamped before the conversion
    const int lim = (int)lf;
    const int p0 = max(min(in, lim), 0), p1 = min(max(in, lim), S - 1);
    for (int p = p0; p <= p1; ++p) {
        if (__ldg(G.fidx + img + base + p * step) != f) continue;
        xy(p, xi, yi);
        edge_term(ga, gb, edge_diff(G, K, b, xi, yi, I_out), p, vc, ua, ub, d0f, Sf, eps);
    }
}

// d0 range of (e, axis): [max(ceil(min u), 0), min(floor(max u), S-1)], empty when u_a == u_b
__device__ __forceinline__ void line_range(const float px[3], const float py[3], int e, int axis, int S, int& lo, int& n) {
    const float* U = axis == 0 ? px : py;
    const float ua = U[e], ub = U[(e + 1) % 3];
    lo = 0;
    n = 0;
    if (ua == ub) return;
    const float l = fmaxf(ceilf(fminf(ua, ub)), 0.f), h = fminf(floorf(fmaxf(ua, ub)), (float)(S - 1));
    if (l <= h) { lo = (int)l; n = (int)h - lo + 1; }
}

// One warp per (image, face), the only writer of that face's 9 gradient values.  Lane l takes lines l, l + 32, ... of
// the face's (edge, axis, d0) lines in that order, then the depth pixels of its pixel box (rows ascending, 32-pixel
// row segments); the 9 lane sums are reduced by a fixed xor-shuffle tree.  No atomics: bitwise reproducible.
__global__ void __launch_bounds__(256) k_nmr_grad_faces(const float* __restrict__ rec, const int4* __restrict__ box,
                                                        GradPlanes G, float* __restrict__ grad, float eps, Consts K) {
    const int lane = threadIdx.x & 31;
    const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (gw >= (long long)K.B * K.F) return;  // whole warps
    const int b = (int)(gw / K.F), f = (int)(gw - (long long)b * K.F);
    const float* rc = rec + ((size_t)b * K.Fc + f) * REC;
    const int S = K.S;
    const float Sf = (float)S;
    float acc[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) acc[k] = 0.f;

    if (G.rgb || G.alpha) {
        float x[3], y[3];
        bool finite = true;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            x[k] = __ldg(rc + R_X + 2 * k);
            y[k] = __ldg(rc + R_X + 2 * k + 1);
            finite = finite && isfinite(x[k]) && isfinite(y[k]) && isfinite(__ldg(rc + R_Z + k));
        }
        const bool back = (y[2] - y[0]) * (x[1] - x[0]) < (y[1] - y[0]) * (x[2] - x[0]);
        if (finite && !back) {
            float px[3], py[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                px[k] = 0.5f * ((x[k] * Sf + Sf) - 1.f);
                py[k] = 0.5f * ((y[k] * Sf + Sf) - 1.f);
            }
            int lo[6], n[6], total = 0;
#pragma unroll
            for (int s = 0; s < 6; ++s) {
                line_range(px, py, s >> 1, s & 1, S, lo[s], n[s]);
                total += n[s];
            }
            for (int li = lane; li < total; li += 32) {
                int s = 0, d0 = 0, r = li;
                bool found = false;
#pragma unroll
                for (int q = 0; q < 6; ++q) {
                    if (found) continue;
                    if (r < n[q]) { found = true; s = q; d0 = lo[q] + r; } else { r -= n[q]; }
                }
                const int e = s >> 1, axis = s & 1;
                float ga = 0.f, gb = 0.f;
                edge_line(ga, gb, G, K, b, f, px, py, e, axis, d0, eps);
                // the line moves y (axis 0) or x (axis 1) of vertices e and e + 1
                const int ia = e * 3 + (axis == 0 ? 1 : 0), ib = (e == 2 ? 0 : e + 1) * 3 + (axis == 0 ? 1 : 0);
#pragma unroll
                for (int k = 0; k < 9; ++k) {
                    if (k == ia) acc[k] = acc[k] + ga;
                    if (k == ib) acc[k] = acc[k] + gb;
                }
            }
        }
    }

    if (G.depth) {
        const int4 bb = __ldg(box + (size_t)b * K.Fc + f);
        const float z0 = __ldg(rc + R_Z), z1 = __ldg(rc + R_Z + 1), z2 = __ldg(rc + R_Z + 2);
        const float half = 0.5f * Sf;
        for (int yi = bb.z; yi <= bb.w; ++yi) {
            for (int xs = bb.x; xs <= bb.y; xs += 32) {
                const int xi = xs + lane;
                if (xi > bb.y || __ldg(G.fidx + ((size_t)b * S + yi) * S + xi) != f) continue;
                const float g = out_grad(K, G.depth, out_index(K, b, xi, yi));
                if (g == 0.f) continue;
                float w[3], zp;
                bary(rc, xi, yi, w, zp);
                const float a = (zp * zp) * g;
                const float sx = (__ldg(rc + R_INV + 0) / z0 + __ldg(rc + R_INV + 3) / z1) + __ldg(rc + R_INV + 6) / z2;
                const float sy = (__ldg(rc + R_INV + 1) / z0 + __ldg(rc + R_INV + 4) / z1) + __ldg(rc + R_INV + 7) / z2;
                const float zk[3] = {z0, z1, z2};
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const float t = a * w[k];
                    acc[3 * k] = acc[3 * k] + (t * sx) * half;
                    acc[3 * k + 1] = acc[3 * k + 1] + (t * sy) * half;
                    acc[3 * k + 2] = acc[3 * k + 2] + t / (zk[k] * zk[k]);
                }
            }
        }
    }

#pragma unroll
    for (int k = 0; k < 9; ++k) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) acc[k] = acc[k] + __shfl_xor_sync(0xffffffffu, acc[k], off);
    }
    if (lane == 0) {
        float* o = grad + ((size_t)b * K.F + f) * 9;
#pragma unroll
        for (int k = 0; k < 9; ++k) o[k] = acc[k];
    }
}

// ---------------------------------------------------------------------------------------------
// neural_renderer.lighting (DESIGN.md §15): lit = textures * light[b, f], float and double
// ---------------------------------------------------------------------------------------------
template <typename T>
struct LightArgs {
    const T* faces;  // [B,F,3,3]
    const T* tex;    // [B,F,n3]
    const T *ca, *cd, *dir;
    int sca, scd, sdir;  // batch strides of ca, cd, dir: 0 or 3
    int F, n3;           // n3 = T^3 * 3
    long long N;         // B * F * n3
    T Ia, Id;
};

// light of face bf = b * F + f
template <typename T>
__device__ __forceinline__ void load_light(const LightArgs<T>& A, int bf, T l[3], LightParts<T>* q) {
    const int b = bf / A.F;
    T v[3][3], ca[3], cd[3], dir[3];
    const T* fv = A.faces + (size_t)bf * 9;
#pragma unroll
    for (int k = 0; k < 9; ++k) v[k / 3][k % 3] = __ldg(fv + k);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        ca[c] = __ldg(A.ca + (size_t)b * A.sca + c);
        cd[c] = __ldg(A.cd + (size_t)b * A.scd + c);
        dir[c] = __ldg(A.dir + (size_t)b * A.sdir + c);
    }
    face_light(v, A.Ia, A.Id, ca, cd, dir, l, q);
}

constexpr int LT_CTA = 256;
constexpr int LT_VPT = 4;  // 16-byte vectors per thread

// Forward: each CTA takes LT_CTA * LT_VPT vectors of the flat [B*F*n3] texel array.  Its threads first compute the light
// of every face that range touches into shared memory, then multiply the texels, 16-byte loads and stores when VEC
// (textures and output 16-byte aligned), element by element otherwise and in the ragged tail.
template <typename T>
__host__ __device__ constexpr int lt_elems() { return LT_CTA * LT_VPT * (16 / (int)sizeof(T)); }

template <typename T, bool VEC>
__global__ void __launch_bounds__(LT_CTA) k_nmr_light_fwd(LightArgs<T> A, T* __restrict__ out) {
    constexpr int W = 16 / (int)sizeof(T);
    constexpr int E = lt_elems<T>();
    __shared__ T s_l[E / 3 + 2][3];  // n3 >= 3: at most E / 3 + 2 faces meet the range
    const long long e0 = (long long)blockIdx.x * E;
    const long long e1 = min(e0 + E, A.N);
    const int fa = (int)(e0 / A.n3), nf = (int)((e1 - 1) / A.n3) - fa + 1;
    for (int i = threadIdx.x; i < nf; i += LT_CTA) {
        T l[3];
        load_light<T>(A, fa + i, l, nullptr);
        s_l[i][0] = l[0]; s_l[i][1] = l[1]; s_l[i][2] = l[2];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < LT_VPT; ++k) {
        const long long e = e0 + ((long long)k * LT_CTA + threadIdx.x) * W;
        if (e >= e1) break;
        int fi = (int)(e / A.n3);
        int r = (int)(e - (long long)fi * A.n3);
        fi -= fa;
        int ch = r % 3;
        T x[W];
        const bool full = VEC && e + W <= e1;
        if (full) {
            if constexpr (sizeof(T) == 4) {
                const float4 t = __ldg(reinterpret_cast<const float4*>(A.tex + e));
                x[0] = t.x; x[1] = t.y; x[2] = t.z; x[3] = t.w;
            } else {
                const double2 t = __ldg(reinterpret_cast<const double2*>(A.tex + e));
                x[0] = t.x; x[1] = t.y;
            }
        } else {
#pragma unroll
            for (int j = 0; j < W; ++j) x[j] = e + j < e1 ? __ldg(A.tex + e + j) : T(0);
        }
#pragma unroll
        for (int j = 0; j < W; ++j) {
            if (e + j < e1) x[j] = x[j] * s_l[fi][ch];
            if (++r == A.n3) { r = 0; ++fi; }
            ch = ch == 2 ? 0 : ch + 1;  // n3 is a multiple of 3: a face starts on channel 0
        }
        if (full) {
            if constexpr (sizeof(T) == 4) *reinterpret_cast<float4*>(out + e) = make_float4(x[0], x[1], x[2], x[3]);
            else *reinterpret_cast<double2*>(out + e) = make_double2(x[0], x[1]);
        } else {
#pragma unroll
            for (int j = 0; j < W; ++j)
                if (e + j < e1) out[e + j] = x[j];
        }
    }
}

// Backward: one warp per (image, face), the only writer of that face's outputs.  grad_tex = light * g; per channel
// s_c = sum of tex * g, each lane over its elements in ascending order, then a fixed xor-shuffle tree.  Lane 0 chains
// s through the light (relu, normalize, cross) into grad_faces [B,F,3,3] and the per-face partials of the light
// parameters, part [B][9][F] (ca, cd, dir), reduced by k_nmr_light_reduce.  No atomics.
template <typename T>
__global__ void __launch_bounds__(256) k_nmr_light_bwd(LightArgs<T> A, long long nface, const T* __restrict__ g,
                                                       T* __restrict__ grad_tex, T* __restrict__ grad_faces,
                                                       T* __restrict__ part) {
    const int lane = threadIdx.x & 31;
    const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (gw >= nface) return;  // whole warps
    const int bf = (int)gw;
    T l[3];
    LightParts<T> q;
    load_light<T>(A, bf, l, &q);
    const size_t base = (size_t)bf * A.n3;
    const bool need_s = grad_faces || part;
    // lane l's elements l + 32 k: channel (l + 2 k) mod 3, so phase k mod 3 keeps one channel per lane
    T acc[3] = {T(0), T(0), T(0)};
    for (int k0 = 0; lane + 32 * k0 < A.n3; k0 += 3) {
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const int e = lane + 32 * (k0 + j);
            if (e < A.n3) {
                const int ch = (lane + 2 * j) % 3;
                const T gv = __ldg(g + base + e);
                if (grad_tex) grad_tex[base + e] = l[ch] * gv;
                if (need_s) acc[j] = acc[j] + __ldg(A.tex + base + e) * gv;
            }
        }
    }
    if (!need_s) return;
    T s[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        // the phase j that holds channel c on this lane: (lane + 2 j) mod 3 == c
        const int j = ((c - lane % 3 + 3) * 2) % 3;
        s[c] = j == 0 ? acc[0] : (j == 1 ? acc[1] : acc[2]);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s[c] = s[c] + __shfl_xor_sync(0xffffffffu, s[c], off);
    }
    if (lane != 0) return;
    const int b = bf / A.F, f = bf - b * A.F;
    T gcs = T(0), gca[3], gcd[3], gdir[3], gv[3][3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        gca[c] = A.Ia != T(0) ? A.Ia * s[c] : T(0);
        gcd[c] = A.Id != T(0) ? (A.Id * s[c]) * q.cs : T(0);
        if (A.Id != T(0)) gcs = gcs + (A.Id * s[c]) * __ldg(A.cd + (size_t)b * A.scd + c);
    }
    if (A.Id != T(0)) {
        const T gnd = q.cs <= T(0) ? T(0) : gcs;  // relu: no gradient where the output is 0 (NaN passes)
        T gn[3], gc[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            gdir[k] = gnd * q.n[k];
            gn[k] = gnd * __ldg(A.dir + (size_t)b * A.sdir + k);
        }
        // normalize: n = c / max(|c|, eps); the norm's gradient passes only where |c| >= eps
        const T t = (gn[0] * q.n[0] + gn[1] * q.n[1]) + gn[2] * q.n[2];
        const bool pass = q.nrm >= light_eps<T>();
#pragma unroll
        for (int k = 0; k < 3; ++k) gc[k] = (pass ? gn[k] - t * q.n[k] : gn[k]) / q.den;
        // c = a x b: grad a = b x gc, grad b = gc x a; v0 = a + v1, v2 = b + v1
        const T* a = q.a;
        const T* bb = q.b;
        const T ga[3] = {bb[1] * gc[2] - bb[2] * gc[1], bb[2] * gc[0] - bb[0] * gc[2], bb[0] * gc[1] - bb[1] * gc[0]};
        const T gb[3] = {gc[1] * a[2] - gc[2] * a[1], gc[2] * a[0] - gc[0] * a[2], gc[0] * a[1] - gc[1] * a[0]};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            gv[0][k] = ga[k];
            gv[1][k] = -ga[k] - gb[k];
            gv[2][k] = gb[k];
        }
    } else {
#pragma unroll
        for (int k = 0; k < 3; ++k) { gdir[k] = T(0); gv[0][k] = gv[1][k] = gv[2][k] = T(0); }
    }
    if (grad_faces) {
        T* o = grad_faces + (size_t)bf * 9;
#pragma unroll
        for (int k = 0; k < 9; ++k) o[k] = gv[k / 3][k % 3];
    }
    if (part) {
        T* p = part + (size_t)b * 9 * A.F + f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            p[(size_t)c * A.F] = gca[c];
            p[(size_t)(3 + c) * A.F] = gcd[c];
            p[(size_t)(6 + c) * A.F] = gdir[c];
        }
    }
}

// grad_light [B,9] = sum over f ascending of part[b][k][f], one warp per (image, k).  The lanes load tiles of
// 32 * LR_TILE consecutive partials, the next tile in flight while every lane folds the current one in ascending order
// from shuffles; only the F adds are serial.  It runs only when a light parameter needs a gradient.
constexpr int LR_TILE = 8;

template <typename T>
__global__ void __launch_bounds__(128) k_nmr_light_reduce(const T* __restrict__ part, T* __restrict__ grad_light, int B,
                                                          int F) {
    const int lane = threadIdx.x & 31;
    const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= (long long)B * 9) return;  // whole warps
    const T* p = part + (size_t)w * F;
    auto load = [&](T x[LR_TILE], int f0) {
#pragma unroll
        for (int j = 0; j < LR_TILE; ++j) {
            const int f = f0 + 32 * j + lane;
            x[j] = f < F ? __ldg(p + f) : T(0);
        }
    };
    T s = T(0), x[LR_TILE], nx[LR_TILE];
    load(x, 0);
    for (int f0 = 0; f0 < F; f0 += 32 * LR_TILE) {
        load(nx, f0 + 32 * LR_TILE);
        if (F - f0 >= 32 * LR_TILE) {
#pragma unroll
            for (int j = 0; j < LR_TILE; ++j)
#pragma unroll
                for (int l = 0; l < 32; ++l) s = s + __shfl_sync(0xffffffffu, x[j], l);
        } else {
#pragma unroll
            for (int j = 0; j < LR_TILE; ++j)
                for (int l = 0; l < 32 && f0 + 32 * j + l < F; ++l) s = s + __shfl_sync(0xffffffffu, x[j], l);
        }
#pragma unroll
        for (int j = 0; j < LR_TILE; ++j) x[j] = nx[j];
    }
    if (lane == 0) grad_light[w] = s;
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static int check(const UmrNmrParams* p, bool need_tex) {
    if (!p) return UMR_ERR_BAD_ARG;
    if (p->batch_size <= 0 || p->num_vertices <= 0 || p->num_faces <= 0 || p->image_size <= 0) return UMR_ERR_BAD_ARG;
    if (need_tex && p->texture_res < 2) return UMR_ERR_BAD_ARG;  // T = 1 indexes past the cube in NMR
    if (p->shared_textures > 1 && p->batch_size % p->shared_textures != 0) return UMR_ERR_BAD_ARG;
    const long long S = (long long)p->image_size * (p->anti_aliasing ? 2 : 1);
    const long long Fc = (long long)p->num_faces * (p->fill_back ? 2 : 1);
    if (S > 16384 || Fc > (1ll << 30) || p->batch_size > 65535) return UMR_ERR_TOO_LARGE;
    // T^3 <= 2^20 (T <= 101); T is ignored without textures
    if (need_tex && (p->texture_res > 1024 || (long long)p->texture_res * p->texture_res * p->texture_res > (1 << 20)))
        return UMR_ERR_TOO_LARGE;
    return UMR_OK;
}

static Consts make_consts(const UmrNmrParams* p) {
    Consts K;
    K.B = p->batch_size;
    K.V = p->num_vertices;
    K.F = p->num_faces;
    K.Fc = p->num_faces * (p->fill_back ? 2 : 1);
    K.T = p->texture_res;
    K.IS = p->image_size;
    K.aa = p->anti_aliasing ? 1 : 0;
    K.S = p->image_size * (K.aa ? 2 : 1);
    K.tex_div = p->shared_textures > 1 ? p->shared_textures : 1;
    K.eye_z = p->eye_z;
    K.near_ = p->near_plane;
    K.far_ = p->far_plane;
    K.Ia = p->light_intensity_ambient;
    K.Id = p->light_intensity_directional;
    for (int c = 0; c < 3; ++c) {
        K.ca[c] = p->light_color_ambient[c];
        K.cd[c] = p->light_color_directional[c];
        K.dir[c] = p->light_direction[c];
        K.bg[c] = p->background_color[c];
    }
    return K;
}

// the record and box arrays at the start of every NMR workspace (umr_nmr_workspace_bytes), filled by k_nmr_prep
struct Prepared {
    float* rec;
    int4* box;
};
static Prepared prep(const float* vertices, const int32_t* faces, void* workspace, const Consts& K, cudaStream_t stream) {
    const Prepared w{(float*)workspace, (int4*)((char*)workspace + rec_bytes(K.B, K.Fc))};
    launch(k_nmr_prep, dim3((K.Fc + 127) / 128, K.B), 128, 0, stream, vertices, faces, w.rec, w.box, K);
    return w;
}

// the default and deterministic texture gradients: the same arguments and workspace, k_nmr_bwd_tex_det in place of
// k_nmr_bwd_tex
static int backward_textures(const float* vertices, const int32_t* faces, const int32_t* face_index, const float* grad_rgb,
                             float* grad_textures, const UmrNmrParams* p, void* workspace, void* stream_, bool det) {
    int rc = check(p, true);
    if (rc) return rc;
    if (!vertices || !faces || !face_index || !grad_rgb || !grad_textures || !workspace) return UMR_ERR_BAD_ARG;
    if (((uintptr_t)workspace & 255) != 0 || ((uintptr_t)grad_textures & 3) != 0) return UMR_ERR_BAD_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    const Consts K = make_consts(p);
    const size_t gbytes = (size_t)(K.B / K.tex_div) * K.F * K.T * K.T * K.T * 3 * sizeof(float);
    cudaError_t e = cudaMemsetAsync(grad_textures, 0, gbytes, stream);
    if (e != cudaSuccess) return (int)e;
    const Prepared w = prep(vertices, faces, workspace, K, stream);
    if (det) {
        const long long nwarp = (long long)(K.B / K.tex_div) * K.F;
        launch(k_nmr_bwd_tex_det, (unsigned)((nwarp + DET_WARPS - 1) / DET_WARPS), DET_WARPS * 32, 0, stream, w.rec, w.box,
               face_index, grad_rgb, grad_textures, K);
    } else {
        const size_t nthr = (size_t)K.B * K.IS * K.IS;
        launch(k_nmr_bwd_tex, (unsigned)((nthr + 255) / 256), 256, 0, stream, w.rec, face_index, grad_rgb, grad_textures, K);
    }
    return (int)cudaGetLastError();
}

}  // namespace nmr
}  // namespace umr

using namespace umr::nmr;
using umr::launch;

extern "C" size_t umr_nmr_workspace_bytes(int32_t batch_size, int32_t num_faces, int32_t fill_back) {
    // 0 for the shapes check() refuses, like B <= 0
    if (batch_size <= 0 || num_faces <= 0 || batch_size > 65535) return 0;
    const long long Fc = (long long)num_faces * (fill_back ? 2 : 1);
    if (Fc > (1ll << 30)) return 0;
    return rec_bytes(batch_size, (int)Fc) + box_bytes(batch_size, (int)Fc);
}

extern "C" size_t umr_sizeof_nmr_params(void) { return sizeof(UmrNmrParams); }

extern "C" int umr_nmr_forward(const float* vertices, const int32_t* faces, const float* textures, int32_t* face_index,
                               float* raster_depth, float* rgb, float* alpha, float* depth, const UmrNmrParams* p,
                               void* workspace, void* stream_) {
    int rc = check(p, textures != nullptr);
    if (rc) return rc;
    if (!vertices || !faces || !face_index || !raster_depth || !workspace) return UMR_ERR_BAD_ARG;
    if (rgb && !textures) return UMR_ERR_BAD_ARG;
    if (((uintptr_t)workspace & 255) != 0) return UMR_ERR_BAD_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    const Consts K = make_consts(p);
    const Prepared w = prep(vertices, faces, workspace, K, stream);
    const int nb = (K.S + BIN - 1) / BIN;
    launch(k_nmr_zbuf, dim3(nb, nb, K.B), CTA, 0, stream, w.rec, w.box, face_index, raster_depth, K);
    if (rgb || alpha || depth) {
        const bool vec = (K.IS % 4) == 0 && (((uintptr_t)rgb | (uintptr_t)alpha | (uintptr_t)depth) & 15) == 0;
        const size_t nthr = (size_t)K.B * K.IS * (vec ? K.IS / 4 : K.IS);
        launch(vec ? k_nmr_shade<4> : k_nmr_shade<1>, (unsigned)((nthr + 255) / 256), 256, 0, stream, w.rec, face_index,
               raster_depth, textures, rgb, alpha, depth, K);
    }
    return (int)cudaGetLastError();
}

extern "C" int umr_nmr_backward_textures(const float* vertices, const int32_t* faces, const int32_t* face_index,
                                         const float* grad_rgb, float* grad_textures, const UmrNmrParams* p,
                                         void* workspace, void* stream_) {
    return backward_textures(vertices, faces, face_index, grad_rgb, grad_textures, p, workspace, stream_, false);
}

// Deterministic texture gradient (include/umr_b200.h)
extern "C" int umr_nmr_backward_textures_deterministic(const float* vertices, const int32_t* faces, const int32_t* face_index,
                                                       const float* grad_rgb, float* grad_textures, const UmrNmrParams* p,
                                                       void* workspace, void* stream_) {
    return backward_textures(vertices, faces, face_index, grad_rgb, grad_textures, p, workspace, stream_, true);
}

// Geometry gradient (include/umr_b200.h, DESIGN.md §14).  Workspace: the forward's record and box arrays, then the
// raster colour plane [B,S,S,3].
extern "C" size_t umr_nmr_backward_faces_workspace_bytes(int32_t batch_size, int32_t num_faces, int32_t image_size,
                                                         int32_t anti_aliasing) {
    if (batch_size <= 0 || num_faces <= 0 || image_size <= 0 || batch_size > 65535 || num_faces > (1 << 30)) return 0;
    const long long S = (long long)image_size * (anti_aliasing ? 2 : 1);
    if (S > 16384) return 0;
    return rec_bytes(batch_size, num_faces) + box_bytes(batch_size, num_faces) +
           align256((size_t)batch_size * (size_t)(S * S) * 3 * sizeof(float));
}

extern "C" int umr_nmr_backward_faces(const float* vertices, const int32_t* faces, const int32_t* face_index,
                                      const float* textures, const float* grad_rgb, const float* grad_alpha,
                                      const float* grad_depth, float* grad_face_vertices, const UmrNmrParams* p, float eps,
                                      void* workspace, void* stream_) {
    int rc = check(p, textures != nullptr);
    if (rc) return rc;
    if (!vertices || !faces || !face_index || !grad_face_vertices || !workspace) return UMR_ERR_BAD_ARG;
    if (grad_rgb && !textures) return UMR_ERR_BAD_ARG;
    if (((uintptr_t)workspace & 255) != 0 || ((uintptr_t)grad_face_vertices & 3) != 0) return UMR_ERR_BAD_ARG;
    if (!(eps >= 0.f && eps < INFINITY)) return UMR_ERR_BAD_ARG;
    // the functional rasteriser's configuration: one copy per face, light exactly 1 (no geometry-dependent shading)
    if (p->fill_back || p->light_intensity_directional != 0.f) return UMR_ERR_UNSUPPORTED;
    cudaStream_t stream = (cudaStream_t)stream_;
    const Consts K = make_consts(p);
    float* color = (float*)((char*)workspace + rec_bytes(K.B, K.Fc) + box_bytes(K.B, K.Fc));
    const Prepared w = prep(vertices, faces, workspace, K, stream);
    if (grad_rgb) {
        const size_t n = (size_t)K.B * K.S * K.S;
        launch(k_nmr_shade_raster, (unsigned)((n + 255) / 256), 256, 0, stream, w.rec, face_index, textures, color, K);
    }
    GradPlanes G{grad_rgb, grad_alpha, grad_depth, color, face_index};
    const long long nthr = (long long)K.B * K.F * 32;
    launch(k_nmr_grad_faces, (unsigned)((nthr + 255) / 256), 256, 0, stream, w.rec, w.box, G, grad_face_vertices, eps, K);
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// lighting (include/umr_b200.h, DESIGN.md §15)
// ---------------------------------------------------------------------------------------------
static int light_check(const UmrNmrLightParams* p, long long& n3, long long& N) {
    if (!p) return UMR_ERR_BAD_ARG;
    if (p->batch_size < 1 || p->num_faces < 1 || p->texture_res < 1 || p->reserved != 0) return UMR_ERR_BAD_ARG;
    if (p->dtype != UMR_DTYPE_FLOAT32 && p->dtype != UMR_DTYPE_FLOAT64) return UMR_ERR_BAD_ARG;
    for (int s : {p->color_ambient_bstride, p->color_directional_bstride, p->direction_bstride})
        if (s != 0 && s != 3) return UMR_ERR_BAD_ARG;
    const long long T = p->texture_res;
    if (T > 1024) return UMR_ERR_TOO_LARGE;
    n3 = T * T * T * 3;
    if (n3 >= (1ll << 31)) return UMR_ERR_TOO_LARGE;
    const long long BF = (long long)p->batch_size * p->num_faces;
    if (BF * 9 >= (1ll << 31) || BF * n3 >= (1ll << 31)) return UMR_ERR_TOO_LARGE;
    N = BF * n3;
    return UMR_OK;
}

static bool aligned(const void* ptr, size_t a) { return ((uintptr_t)ptr & (a - 1)) == 0; }

template <typename T>
static LightArgs<T> light_args(const void* faces, const void* textures, const void* ca, const void* cd, const void* dir,
                               const UmrNmrLightParams* p, long long n3, long long N) {
    LightArgs<T> A;
    A.faces = (const T*)faces;
    A.tex = (const T*)textures;
    A.ca = (const T*)ca;
    A.cd = (const T*)cd;
    A.dir = (const T*)dir;
    A.sca = p->color_ambient_bstride;
    A.scd = p->color_directional_bstride;
    A.sdir = p->direction_bstride;
    A.F = p->num_faces;
    A.n3 = (int)n3;
    A.N = N;
    A.Ia = (T)p->intensity_ambient;
    A.Id = (T)p->intensity_directional;
    return A;
}

template <typename T>
static int light_forward(const LightArgs<T>& A, T* out, cudaStream_t stream) {
    const unsigned grid = (unsigned)((A.N + lt_elems<T>() - 1) / lt_elems<T>());
    launch(aligned(A.tex, 16) && aligned(out, 16) ? k_nmr_light_fwd<T, true> : k_nmr_light_fwd<T, false>, grid, LT_CTA, 0,
           stream, A, out);
    return (int)cudaGetLastError();
}

template <typename T>
static int light_backward(const LightArgs<T>& A, int B, const T* g, T* grad_faces, T* grad_tex, T* grad_light, T* part,
                          cudaStream_t stream) {
    const long long nface = (long long)B * A.F;
    launch(k_nmr_light_bwd<T>, (unsigned)((nface * 32 + 255) / 256), 256, 0, stream, A, nface, g, grad_tex, grad_faces,
           grad_light ? part : nullptr);
    if (grad_light)
        launch(k_nmr_light_reduce<T>, (unsigned)(((long long)B * 9 * 32 + 127) / 128), 128, 0, stream, part, grad_light, B,
               A.F);
    return (int)cudaGetLastError();
}

extern "C" size_t umr_sizeof_nmr_light_params(void) { return sizeof(UmrNmrLightParams); }

extern "C" size_t umr_nmr_lighting_workspace_bytes(int32_t batch_size, int32_t num_faces, int32_t dtype) {
    if (batch_size < 1 || num_faces < 1 || (dtype != UMR_DTYPE_FLOAT32 && dtype != UMR_DTYPE_FLOAT64)) return 0;
    const long long BF = (long long)batch_size * num_faces;
    if (BF * 9 >= (1ll << 31)) return 0;
    return align256((size_t)BF * 9 * (dtype == UMR_DTYPE_FLOAT64 ? sizeof(double) : sizeof(float)));
}

extern "C" int umr_nmr_lighting_forward(const void* faces, const void* textures, const void* color_ambient,
                                        const void* color_directional, const void* direction, void* lit_textures,
                                        const UmrNmrLightParams* p, void* stream_) {
    long long n3 = 0, N = 0;
    int rc = light_check(p, n3, N);
    if (rc) return rc;
    const size_t es = p->dtype == UMR_DTYPE_FLOAT64 ? sizeof(double) : sizeof(float);
    for (const void* b : {faces, textures, color_ambient, color_directional, direction, (const void*)lit_textures})
        if (!b || !aligned(b, es)) return UMR_ERR_BAD_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    if (p->dtype == UMR_DTYPE_FLOAT64)
        return light_forward(light_args<double>(faces, textures, color_ambient, color_directional, direction, p, n3, N),
                             (double*)lit_textures, stream);
    return light_forward(light_args<float>(faces, textures, color_ambient, color_directional, direction, p, n3, N),
                         (float*)lit_textures, stream);
}

extern "C" int umr_nmr_lighting_backward(const void* faces, const void* textures, const void* color_ambient,
                                         const void* color_directional, const void* direction, const void* grad_lit,
                                         void* grad_faces, void* grad_textures, void* grad_light,
                                         const UmrNmrLightParams* p, void* workspace, void* stream_) {
    long long n3 = 0, N = 0;
    int rc = light_check(p, n3, N);
    if (rc) return rc;
    const size_t es = p->dtype == UMR_DTYPE_FLOAT64 ? sizeof(double) : sizeof(float);
    for (const void* b : {faces, textures, color_ambient, color_directional, direction, grad_lit})
        if (!b || !aligned(b, es)) return UMR_ERR_BAD_ARG;
    if (!grad_faces && !grad_textures && !grad_light) return UMR_ERR_BAD_ARG;
    for (const void* b : {(const void*)grad_faces, (const void*)grad_textures, (const void*)grad_light})
        if (b && !aligned(b, es)) return UMR_ERR_BAD_ARG;
    if (grad_light && (!workspace || !aligned(workspace, 256))) return UMR_ERR_BAD_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    const int B = p->batch_size;
    if (p->dtype == UMR_DTYPE_FLOAT64)
        return light_backward(light_args<double>(faces, textures, color_ambient, color_directional, direction, p, n3, N),
                              B, (const double*)grad_lit, (double*)grad_faces, (double*)grad_textures,
                              (double*)grad_light, (double*)workspace, stream);
    return light_backward(light_args<float>(faces, textures, color_ambient, color_directional, direction, p, n3, N), B,
                          (const float*)grad_lit, (float*)grad_faces, (float*)grad_textures, (float*)grad_light,
                          (float*)workspace, stream);
}
