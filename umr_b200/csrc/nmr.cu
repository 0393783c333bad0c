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
    // light from the vertices before look_at: normalize(cross(v0 - v1, v2 - v1), eps=1e-5)
    {
        const float ax = v[0][0] - v[1][0], ay = v[0][1] - v[1][1], az = v[0][2] - v[1][2];
        const float bx = v[2][0] - v[1][0], by = v[2][1] - v[1][1], bz = v[2][2] - v[1][2];
        const float c0 = ay * bz - az * by, c1 = az * bx - ax * bz, c2 = ax * by - ay * bx;
        const float den = fmaxf(sqrtf((c0 * c0 + c1 * c1) + c2 * c2), 1e-5f);
        const float n0 = c0 / den, n1 = c1 / den, n2 = c2 / den;
        float cs = (n0 * K.dir[0] + n1 * K.dir[1]) + n2 * K.dir[2];
        cs = cs < 0.f ? 0.f : cs;  // relu (NaN stays NaN)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float l = 0.f;
            if (K.Ia != 0.f) l = l + K.Ia * K.ca[c];
            if (K.Id != 0.f) l = l + K.Id * (K.cd[c] * cs);
            out[R_L + c] = l;
        }
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
                uint32_t zb = __float_as_uint(zp);
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
        }
        const size_t o = ((size_t)b * S + by0 + row) * S + bx0 + col;
        face_index[o] = fi;
        rdepth[o] = z;
    }
}

// ---------------------------------------------------------------------------------------------
// shading: texture, light, background, flip, pool
// ---------------------------------------------------------------------------------------------
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
// host side
// ---------------------------------------------------------------------------------------------
static int check(const UmrNmrParams* p, bool need_tex) {
    if (!p) return UMR_ERR_BAD_ARG;
    if (p->batch_size <= 0 || p->num_vertices <= 0 || p->num_faces <= 0 || p->image_size <= 0) return UMR_ERR_BAD_ARG;
    if (need_tex && p->texture_res < 2) return UMR_ERR_BAD_ARG;  // T = 1 indexes past the cube in NMR
    if (p->shared_textures > 1 && p->batch_size % p->shared_textures != 0) return UMR_ERR_BAD_ARG;
    const long long S = (long long)p->image_size * (p->anti_aliasing ? 2 : 1);
    const long long Fc = (long long)p->num_faces * (p->fill_back ? 2 : 1);
    if (S > 16384 || Fc > (1ll << 30) || p->batch_size > 65535 || (long long)p->texture_res * p->texture_res * p->texture_res > (1 << 20))
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

static void launch_prep(const float* vertices, const int32_t* faces, float* rec, int4* box, const Consts& K,
                        cudaStream_t stream) {
    k_nmr_prep<<<dim3((K.Fc + 127) / 128, K.B), 128, 0, stream>>>(vertices, faces, rec, box, K);
    count_launch();
}

}  // namespace nmr
}  // namespace umr

using namespace umr::nmr;

extern "C" size_t umr_nmr_workspace_bytes(int32_t batch_size, int32_t num_faces, int32_t fill_back) {
    if (batch_size <= 0 || num_faces <= 0) return 0;
    const int Fc = num_faces * (fill_back ? 2 : 1);
    return rec_bytes(batch_size, Fc) + box_bytes(batch_size, Fc);
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
    char* ws = (char*)workspace;
    float* rec = (float*)ws;
    int4* box = (int4*)(ws + rec_bytes(K.B, K.Fc));
    launch_prep(vertices, faces, rec, box, K, stream);
    const int nb = (K.S + BIN - 1) / BIN;
    k_nmr_zbuf<<<dim3(nb, nb, K.B), CTA, 0, stream>>>(rec, box, face_index, raster_depth, K);
    umr::count_launch();
    if (rgb || alpha || depth) {
        const bool vec = (K.IS % 4) == 0 && (((uintptr_t)rgb | (uintptr_t)alpha | (uintptr_t)depth) & 15) == 0;
        const size_t nthr = (size_t)K.B * K.IS * (vec ? K.IS / 4 : K.IS);
        const unsigned grid = (unsigned)((nthr + 255) / 256);
        if (vec) k_nmr_shade<4><<<grid, 256, 0, stream>>>(rec, face_index, raster_depth, textures, rgb, alpha, depth, K);
        else k_nmr_shade<1><<<grid, 256, 0, stream>>>(rec, face_index, raster_depth, textures, rgb, alpha, depth, K);
        umr::count_launch();
    }
    return (int)cudaGetLastError();
}

extern "C" int umr_nmr_backward_textures(const float* vertices, const int32_t* faces, const int32_t* face_index,
                                         const float* grad_rgb, float* grad_textures, const UmrNmrParams* p,
                                         void* workspace, void* stream_) {
    int rc = check(p, true);
    if (rc) return rc;
    if (!vertices || !faces || !face_index || !grad_rgb || !grad_textures || !workspace) return UMR_ERR_BAD_ARG;
    if (((uintptr_t)workspace & 255) != 0 || ((uintptr_t)grad_textures & 3) != 0) return UMR_ERR_BAD_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    const Consts K = make_consts(p);
    const size_t gbytes = (size_t)(K.B / K.tex_div) * K.F * K.T * K.T * K.T * 3 * sizeof(float);
    cudaError_t e = cudaMemsetAsync(grad_textures, 0, gbytes, stream);
    if (e != cudaSuccess) return (int)e;
    char* ws = (char*)workspace;
    float* rec = (float*)ws;
    int4* box = (int4*)(ws + rec_bytes(K.B, K.Fc));
    launch_prep(vertices, faces, rec, box, K, stream);
    const size_t nthr = (size_t)K.B * K.IS * K.IS;
    k_nmr_bwd_tex<<<(unsigned)((nthr + 255) / 256), 256, 0, stream>>>(rec, face_index, grad_rgb, grad_textures, K);
    umr::count_launch();
    return (int)cudaGetLastError();
}

// Deterministic texture gradient (include/umr_b200.h): the default call's arguments and workspace; k_nmr_bwd_tex_det in
// place of k_nmr_bwd_tex.
extern "C" int umr_nmr_backward_textures_deterministic(const float* vertices, const int32_t* faces, const int32_t* face_index,
                                                       const float* grad_rgb, float* grad_textures, const UmrNmrParams* p,
                                                       void* workspace, void* stream_) {
    int rc = check(p, true);
    if (rc) return rc;
    if (!vertices || !faces || !face_index || !grad_rgb || !grad_textures || !workspace) return UMR_ERR_BAD_ARG;
    if (((uintptr_t)workspace & 255) != 0 || ((uintptr_t)grad_textures & 3) != 0) return UMR_ERR_BAD_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    const Consts K = make_consts(p);
    const size_t gbytes = (size_t)(K.B / K.tex_div) * K.F * K.T * K.T * K.T * 3 * sizeof(float);
    cudaError_t e = cudaMemsetAsync(grad_textures, 0, gbytes, stream);
    if (e != cudaSuccess) return (int)e;
    char* ws = (char*)workspace;
    float* rec = (float*)ws;
    int4* box = (int4*)(ws + rec_bytes(K.B, K.Fc));
    launch_prep(vertices, faces, rec, box, K, stream);
    const long long nwarp = (long long)(K.B / K.tex_div) * K.F;
    k_nmr_bwd_tex_det<<<(unsigned)((nwarp + DET_WARPS - 1) / DET_WARPS), DET_WARPS * 32, 0, stream>>>(rec, box, face_index,
                                                                                                      grad_rgb, grad_textures, K);
    umr::count_launch();
    return (int)cudaGetLastError();
}
