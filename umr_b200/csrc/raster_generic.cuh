// raster_generic.cuh -- the soft rasteriser's per-(pixel, face) arithmetic and its deterministic gather backward, written
// once for float (raster.cu) and double (raster_f64.cu).
//
// The reference kernels (external/SoftRas/soft_renderer/cuda/soft_rasterize_cuda_kernel.cu, "kernel.cu") are one
// `template <typename scalar_t>`; every float/double promotion our float32 arithmetic reproduces (the double sigmoid, the
// double alpha quotient, the double barycentric scale) follows from the scalar type and becomes a no-op for T = double.  Both
// including translation units are compiled with -fmad=false, so every operation here is one IEEE rounding in T.
//
// What differs between the precisions is spelled out where it happens: the float32 quotient shortcuts (pixel_coord,
// depth_of), the flag word of a record (flags_of) and the float32 backward's exact-zero skips (SKIP_ZEROS).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "common.cuh"
#include "umr_b200.h"

namespace umr {

constexpr int TILE = 16;
constexpr int CTA = TILE * TILE;  // 256 threads, one pixel each
constexpr int NWARP = CTA / 32;
constexpr int REC_LEN = 32;       // elements per face record: 128 B (float), 256 B (double)

// record layout (element index)
constexpr int R_V = 0;     // 9 : x0 y0 z0 x1 y1 z1 x2 y2 z2
constexpr int R_INV = 9;   // 9 : barycentric inverse, row-major
constexpr int R_SYM = 18;  // 6 : s00 s01 s02 s11 s12 s22   (Gram + 1)
constexpr int R_BOX = 24;  // 4 : xlo xhi ylo yhi (cull box, already expanded by r)
constexpr int R_FLG = 28;  // 1 : bit0..2 obtuse corner, bit3 front-facing

// bit k of the record's flags: float records keep the bits of a uint32, double records its value
__device__ __forceinline__ uint32_t flags_of(const float* rc) { return __float_as_uint(rc[R_FLG]); }
__device__ __forceinline__ uint32_t flags_of(const double* rc) { return (uint32_t)(int)rc[R_FLG]; }

template <typename T>
struct Consts {
    T thr, sigma, gamma, near_, far_, inv_unused;
    T r_sigma, r_gamma, r_fn, r_nf;  // 1/sigma, 1/gamma, 1/(far-near), 1/(near-far): float streamed backward only
    int F, T2, R, S, IS, aa, double_side;
    int dist, alpha, tex;  // mode ids (read only by the generic-mode kernels)
    int vec_store;         // 1: float forward may use the shared-staged 128-bit store epilogue (alignment checked on host)
    size_t tex_bs;         // elements per texture (F*T2*3)
    int tex_div;           // consecutive images sharing one texture (1: per-image, B: one batch-shared texture)
};
// the float kernels' parameter blocks keep their layout
static_assert(sizeof(Consts<float>) == 104, "Consts<float> layout");

// RGB mode of the float UMR-configuration kernels that form the alpha plane and nothing else (the silhouette render,
// DESIGN.md §12): no softmax weight, no texel, no colour, no p2f.  Alpha, the pair records and the alpha terms of the
// vertex gradients are those of the softmax / hard render.
constexpr int RGB_SIL = 3;

// Per-pixel planes the float backward stages for a pixel: g[NC], g_alpha, C[NC], alpha, ssum, smax -- or, for a silhouette,
// g_alpha and alpha only.  NPL: planes of the image gradient and of the full-resolution image; GA / AL: plane of g_alpha /
// alpha in the staged set.
template <int RGB, int NC>
struct PixPlanes {
    static constexpr bool SIL = RGB == RGB_SIL;
    static constexpr int NPL = SIL ? 1 : NC + 1;
    static constexpr int NV = SIL ? 2 : 2 * NPL + 2;
    static constexpr int GA = SIL ? 0 : NC, AL = SIL ? 1 : 2 * NC + 1;
};

template <typename T>
struct Frag {
    T w0, w1, w2;  // unclipped barycentrics
    T t0, t1, t2;  // closest-point barycentrics minus w (barycentric / hard distance: the unclipped w)
    T sign, dx, dy, dis, D;
};

// kernel.cu:325-326 evaluates (2.*i + 1. - S) / S in double.  For float the result is stored as float: numerator and
// denominator are integers < 2^24 (exact in float), and rounding a correctly rounded binary64 quotient to binary32 equals
// the correctly rounded binary32 quotient whenever the wide format carries at least 2p+2 = 50 bits (Figueroa's
// double-rounding theorem; binary64 has 53).  So one IEEE float division is bit-identical and ~4x cheaper.
template <typename T = float>
__device__ __forceinline__ T pixel_coord(int i, int S) {
    if constexpr (std::is_same_v<T, float>) return __fdiv_rn((float)(2 * i + 1 - S), (float)S);
    else return (2. * i + 1. - S) / S;
}

template <typename T>
__device__ __forceinline__ bool inside_closed(const Frag<T>& fr) {  // kernel.cu:48-50
    return fr.w0 <= 1 && fr.w0 >= 0 && fr.w1 <= 1 && fr.w1 >= 0 && fr.w2 <= 1 && fr.w2 >= 0;
}

// euclidean signed distance + sigmoid: kernel.cu:62-152, 380-383.  `rc` points at a staged record.
// Returns false when the pair is culled (outside and farther than the threshold).
template <typename T>
__device__ __forceinline__ bool fragment(const T* __restrict__ rc, T xp, T yp, T thr, T sigma, Frag<T>& fr) {
    const T w0 = rc[R_INV + 0] * xp + rc[R_INV + 1] * yp + rc[R_INV + 2];
    const T w1 = rc[R_INV + 3] * xp + rc[R_INV + 4] * yp + rc[R_INV + 5];
    const T w2 = rc[R_INV + 6] * xp + rc[R_INV + 7] * yp + rc[R_INV + 8];
    fr.w0 = w0; fr.w1 = w1; fr.w2 = w2;
    const T fx0 = rc[0], fy0 = rc[1], fx1 = rc[3], fy1 = rc[4], fx2 = rc[6], fy2 = rc[7];
    const T s00 = rc[R_SYM + 0], s01 = rc[R_SYM + 1], s02 = rc[R_SYM + 2];
    const T s11 = rc[R_SYM + 3], s12 = rc[R_SYM + 4], s22 = rc[R_SYM + 5];
    // inside pixels (kernel.cu:76-110) keep the nearest of the three edges; outside pixels (:111-147) project on the ONE
    // edge selected by the sign pattern of w (with the obtuse-corner correction) and clamp
    T dx, dy, t0, t1, t2;
    if (w0 > 0 && w1 > 0 && w2 > 0 && w0 < 1 && w1 < 1 && w2 < 1) {
        T best = 100000000;
        // edge k=0: v0=0,v1=1,v2=2    a = sym[0,:] - sym[1,:]
        {
            const T a0 = s00 - s01, a1 = s01 - s11, a2 = s02 - s12;
            T u0 = (w0 * a0 + w1 * a1 + w2 * a2 - a1) / (a0 - a1);
            T u1 = 1 - u0;
            T u2 = 0;
            u0 -= w0; u1 -= w1; u2 -= w2;
            const T ex = u0 * fx0 + u1 * fx1 + u2 * fx2;
            const T ey = u0 * fy0 + u1 * fy1 + u2 * fy2;
            const T d = ex * ex + ey * ey;
            dx = 0; dy = 0; t0 = t1 = t2 = 0;
            if (d < best) { best = d; dx = ex; dy = ey; t0 = u0; t1 = u1; t2 = u2; }
        }
        // edge k=1: v0=1,v1=2,v2=0    a = sym[1,:] - sym[2,:]
        {
            const T a0 = s01 - s02, a1 = s11 - s12, a2 = s12 - s22;
            T u1 = (w0 * a0 + w1 * a1 + w2 * a2 - a2) / (a1 - a2);
            T u2 = 1 - u1;
            T u0 = 0;
            u0 -= w0; u1 -= w1; u2 -= w2;
            const T ex = u0 * fx0 + u1 * fx1 + u2 * fx2;
            const T ey = u0 * fy0 + u1 * fy1 + u2 * fy2;
            const T d = ex * ex + ey * ey;
            if (d < best) { best = d; dx = ex; dy = ey; t0 = u0; t1 = u1; t2 = u2; }
        }
        // edge k=2: v0=2,v1=0,v2=1    a = sym[2,:] - sym[0,:]
        {
            const T a0 = s02 - s00, a1 = s12 - s01, a2 = s22 - s02;
            T u2 = (w0 * a0 + w1 * a1 + w2 * a2 - a0) / (a2 - a0);
            T u0 = 1 - u2;
            T u1 = 0;
            u0 -= w0; u1 -= w1; u2 -= w2;
            const T ex = u0 * fx0 + u1 * fx1 + u2 * fx2;
            const T ey = u0 * fy0 + u1 * fy1 + u2 * fy2;
            const T d = ex * ex + ey * ey;
            if (d < best) { best = d; dx = ex; dy = ey; t0 = u0; t1 = u1; t2 = u2; }
        }
        fr.sign = 1;
    } else {
        const uint32_t flg = flags_of(rc);
        int v0 = -1;
        if (w1 <= 0 && w2 <= 0) {
            v0 = 0;
            if ((flg & 1u) && (xp - fx0) * (fx2 - fx0) + (yp - fy0) * (fy2 - fy0) > 0) v0 = 2;
        } else if (w2 <= 0 && w0 <= 0) {
            v0 = 1;
            if ((flg & 2u) && (xp - fx1) * (fx0 - fx1) + (yp - fy1) * (fy0 - fy1) > 0) v0 = 0;
        } else if (w0 <= 0 && w1 <= 0) {
            v0 = 2;
            if ((flg & 4u) && (xp - fx2) * (fx1 - fx2) + (yp - fy2) * (fy1 - fy2) > 0) v0 = 1;
        } else if (w0 <= 0) v0 = 1;
        else if (w1 <= 0) v0 = 2;
        else if (w2 <= 0) v0 = 0;
        // all w > 0 but some w >= 1 (rounding): undefined in the reference (kernel.cu:128-139 runs
        // with v0 = -1).  Defined as "corner with the largest barycentric", like oracle B.
        if (v0 < 0) v0 = w0 >= w1 ? (w0 >= w2 ? 0 : 2) : (w1 >= w2 ? 1 : 2);
        T u0, u1, u2;
        if (v0 == 0) {  // v1 = 1, v2 = 2
            const T a0 = s00 - s01, a1 = s01 - s11, a2 = s02 - s12;
            u0 = (w0 * a0 + w1 * a1 + w2 * a2 - a1) / (a0 - a1);
            u1 = 1 - u0;
            u2 = 0;
        } else if (v0 == 1) {  // v1 = 2, v2 = 0
            const T a0 = s01 - s02, a1 = s11 - s12, a2 = s12 - s22;
            u1 = (w0 * a0 + w1 * a1 + w2 * a2 - a2) / (a1 - a2);
            u2 = 1 - u1;
            u0 = 0;
        } else {  // v0 = 2, v1 = 0, v2 = 1
            const T a0 = s02 - s00, a1 = s12 - s01, a2 = s22 - s02;
            u2 = (w0 * a0 + w1 * a1 + w2 * a2 - a0) / (a2 - a0);
            u0 = 1 - u2;
            u1 = 0;
        }
        // min(max(t, 0.), 1.) in double then float == float clamp (values are only selected)
        t0 = fmin(fmax(u0, (T)0), (T)1) - w0;
        t1 = fmin(fmax(u1, (T)0), (T)1) - w1;
        t2 = fmin(fmax(u2, (T)0), (T)1) - w2;
        dx = t0 * fx0 + t1 * fx1 + t2 * fx2;
        dy = t0 * fy0 + t1 * fy1 + t2 * fy2;
        fr.sign = -1;
    }
    const T dis = dx * dx + dy * dy;
    if (fr.sign < 0 && dis >= thr) return false;
    fr.t0 = t0; fr.t1 = t1; fr.t2 = t2;
    fr.dx = dx; fr.dy = dy; fr.dis = dis;
    // 1. / (1. + exp(-sign * dis / sigma)): exp in T, double add + divide, T result (:383)
    const T e = exp(-fr.sign * dis / sigma);
    fr.D = (T)(1. / (1. + (double)e));
    return true;
}

// Cull boxes (k_prep, k_prep_f64) take the box of a face's finite coordinates, as the reference's max / min do on the
// device (CUDA's fmaxf / fmax drop a NaN operand): a face with a NaN vertex turns the pixels of that box NaN.

// Modes UMR does not exercise (SURVEY.md §8f-3): hard / barycentric distance, hard / sum alpha, per-vertex textures.  The
// generic kernels read the mode ids from Consts at run time; the float UMR configuration (euclidean, prod, surface) has its
// own kernels.
template <typename T>
__device__ __forceinline__ bool fragment_any(const T* __restrict__ rc, T xp, T yp, const Consts<T>& K, Frag<T>& fr) {
    if (K.dist == UMR_DIST_EUCLIDEAN) return fragment(rc, xp, yp, K.thr, K.sigma, fr);
    const T w0 = rc[R_INV + 0] * xp + rc[R_INV + 1] * yp + rc[R_INV + 2];
    const T w1 = rc[R_INV + 3] * xp + rc[R_INV + 4] * yp + rc[R_INV + 5];
    const T w2 = rc[R_INV + 6] * xp + rc[R_INV + 7] * yp + rc[R_INV + 8];
    fr.w0 = w0; fr.w1 = w1; fr.w2 = w2;
    fr.t0 = w0; fr.t1 = w1; fr.t2 = w2;  // kernel.cu:551 (barycentric backward uses the unclipped w)
    fr.sign = 0; fr.dx = 0; fr.dy = 0; fr.dis = 0;
    if (K.dist == UMR_DIST_HARD) {  // kernel.cu:370-372
        const bool inside = inside_closed(fr);
        fr.D = inside ? 1 : 0;
        return inside;
    }
    // barycentric distance, kernel.cu:156-159, 374-377
    T m = w0 > w1 ? (w1 > w2 ? w2 : w1) : (w0 > w2 ? w2 : w0);
    const T dis = m > 0 ? m * m : -(m * m);
    if (-dis >= K.thr) return false;
    fr.dis = dis;
    fr.D = (T)(1. / (1. + (double)exp(-dis / K.sigma)));
    return true;
}

template <typename T>
__device__ __forceinline__ void clip_bary(T& w0, T& w1, T& w2) {  // kernel.cu:54-59
    const T hi = (T)(1 - 1e-5), lo = (T)1e-5;
    w0 = fmax(fmin(w0, hi), lo);
    w1 = fmax(fmin(w1, hi), lo);
    w2 = fmax(fmin(w2, hi), lo);
    const T s = fmax(w0 + w1 + w2, lo);
    w0 /= s; w1 /= s; w2 /= s;
}

// kernel.cu:403: 1. / (sum) in double.  For float the sum is a float and the result is stored as float, which equals
// 1.f / sum in float (the theorem of pixel_coord: both operands are floats, the binary64 quotient is rounded once more).
__device__ __forceinline__ float depth_of(const float* __restrict__ rc, float c0, float c1, float c2) {
    return __fdiv_rn(1.f, c0 / rc[2] + c1 / rc[5] + c2 / rc[8]);
}
__device__ __forceinline__ double depth_of(const double* __restrict__ rc, double c0, double c1, double c2) {
    return 1. / (c0 / rc[2] + c1 / rc[5] + c2 / rc[8]);
}

template <typename T>
__device__ __forceinline__ int texel_index(T c0, T c1, int R) {  // kernel.cu:180-190
    const int wx = (int)(c0 * R);
    const int wy = (int)(c1 * R);
    if ((c0 + c1) * R - wx - wy <= 1) return wy * R + wx;
    return (R - 1 - wy) * R + (R - 1 - wx);
}

// colour of face texture `tx` (surface: [T2,3] texels; vertex: [3,3] corner colours), kernel.cu:179-195
template <typename T>
__device__ __forceinline__ void sample_texture(const T* __restrict__ tx, T c0, T c1, T c2, const Consts<T>& K, T& r, T& g,
                                               T& b) {
    if (K.tex == UMR_TEX_SURFACE) {
        const T* t = tx + (size_t)texel_index(c0, c1, K.R) * 3;
        r = __ldg(t); g = __ldg(t + 1); b = __ldg(t + 2);
    } else {
        r = c0 * __ldg(tx + 0) + c1 * __ldg(tx + 3) + c2 * __ldg(tx + 6);
        g = c0 * __ldg(tx + 1) + c1 * __ldg(tx + 4) + c2 * __ldg(tx + 7);
        b = c0 * __ldg(tx + 2) + c1 * __ldg(tx + 5) + c2 * __ldg(tx + 8);
    }
}

// Texel-gradient sinks: the float recompute backward adds a pair's texel gradient with REDs; the deterministic gather takes it
// out (address and values) and combines the warp's lanes in a fixed order instead.
struct TexRedSink {
    __device__ __forceinline__ void add3(float* p, float a, float b, float c) const { red_add3_global(p, a, b, c); }
    __device__ __forceinline__ void add(float* p, float v) const { red_add_global(p, v); }
};
// A pair adds to at most 9 consecutive elements (a surface texel's 3 channels, or a vertex texture's 3 corner colours) at
// ascending addresses: *addr = the first, val[k] = the value for *addr + k.
template <typename T>
struct TexTakeSink {
    T** addr;
    T* val;
    __device__ __forceinline__ void add3(T* p, T a, T b, T c) const {
        *addr = p; val[0] = a; val[1] = b; val[2] = c;
    }
    __device__ __forceinline__ void add(T* p, T v) const {
        if (*addr == nullptr) *addr = p;
        val[p - *addr] = v;
    }
};

// texture gradient of one pair: adds wgt * (g0,g1,g2) to the sampled texel (surface) or w_j * wgt * g to the
// three corner colours (vertex), kernel.cu:597-601 / 610-616 with the intended texel semantics (App. B-1)
template <class Sink, typename T>
__device__ __forceinline__ void add_texture_grad(T* __restrict__ gt, T c0, T c1, T c2, const Consts<T>& K, T wgt, T g0, T g1,
                                                 T g2, bool weighted, Sink sink) {
    if (K.tex == UMR_TEX_SURFACE) {
        T* t = gt + (size_t)texel_index(c0, c1, K.R) * 3;
        sink.add(t + 0, weighted ? wgt * g0 : g0);
        sink.add(t + 1, weighted ? wgt * g1 : g1);
        sink.add(t + 2, weighted ? wgt * g2 : g2);
    } else {
        const T w[3] = {c0, c1, c2};
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            sink.add(gt + 3 * j + 0, weighted ? wgt * (w[j] * g0) : w[j] * g0);
            sink.add(gt + 3 * j + 1, weighted ? wgt * (w[j] * g1) : w[j] * g1);
            sink.add(gt + 3 * j + 2, weighted ? wgt * (w[j] * g2) : w[j] * g2);
        }
    }
}

// Conservative index range [i0, i1] of the pixels whose centre coordinate pixel_coord(i, S) lies in [lo, hi] (monotone in i;
// one index of slack on each side, the exact test runs per pixel).  NaN bounds keep every index, as the tile tests do.
template <typename T>
__device__ __forceinline__ void pixel_span(T lo, T hi, int S, int& i0, int& i1) {
    const double a = ((double)lo * S + (S - 1)) * 0.5, c = ((double)hi * S + (S - 1)) * 0.5;
    i0 = a > 0.0 ? (a < (double)S ? (int)a - 1 : S) : 0;
    i1 = c < (double)(S - 1) ? (c > -1.0 ? (int)c + 1 : -1) : S - 1;  // c in (-1, 0): pixel 0 may still lie in the box
    i0 = max(i0, 0);
    i1 = min(i1, S - 1);
}

// One (pixel, face) pair of the generic-mode backward (kernel.cu:577-654), with the texture gradient going to `sink`; writes
// the 9 vertex gradients to gv (zeroed by the caller) and sets `contrib` for a pair inside the depth range.  face_of() yields
// the face index (read only for pairs inside the depth range); pix(k) the pixel's inputs g0 g1 g2 g3 C0 C1 C2 C3 ssum smax.  k_raster_bwd (raster.cu) keeps an inline copy of this body:
// calling it from there changes that kernel's instruction mix and register use, and the default kernels stay bit-for-bit what
// they were.  The GPU tests hold both to oracle B.
template <int RGB, bool TEXGRAD, class Sink = TexRedSink, typename T, class FaceOf, class Pix>
__device__ __forceinline__ void bwd_pair_generic(const T* __restrict__ rc, T xp, T yp, const Consts<T>& K, FaceOf face_of, Pix pix,
                                                 const T* __restrict__ tex_img, T* __restrict__ gtex_img, T* gv, bool& contrib,
                                                 Sink sink = Sink()) {
    // float skips terms that are exactly zero (a zero operand would take the divisions' slow special-operand path); double
    // evaluates every operation, so NaN and inf propagate as in the reference
    constexpr bool SKIP_ZEROS = std::is_same_v<T, float>;
    Frag<T> fr;
    if (fragment_any(rc, xp, yp, K, fr)) {
        // alpha: kernel.cu:577-585 (hard alpha passes the raw gradient through, as the reference does).  x * 0 answers the
        // zero cases with the sign rules of the quotient.
        const T g3 = pix(3), one_m_a = 1 - pix(7);
        T Cxy;
        if (K.alpha == UMR_ALPHA_PROD) {
            Cxy = (one_m_a == 0 || g3 == 0)
                      ? g3 * one_m_a
                      : (T)((double)g3 * ((double)one_m_a / fmax((double)(1 - fr.D), 1e-6)));
        } else if (K.alpha == UMR_ALPHA_SUM) {
            Cxy = g3 / K.F;
        } else {
            Cxy = g3;
        }
        T k0 = fr.w0, k1 = fr.w1, k2 = fr.w2;
        clip_bary(k0, k1, k2);
        const T zp = depth_of(rc, k0, k1, k2);
        if (!(zp < K.near_ || zp > K.far_)) {  // :592 drops the alpha gradient as well
            contrib = true;
            const bool front = (flags_of(rc) & 8u) != 0;
            const int f = face_of();
            const T g0 = pix(0), g1 = pix(1), g2 = pix(2), smax = pix(9);
            T gz0 = 0, gz1 = 0, gz2 = 0;
            if (RGB == 0) {
                if ((T)f == smax) {  // aggrs[1] = winning face id (:596)
                    if (TEXGRAD)
                        add_texture_grad(gtex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, (T)1, g0, g1, g2, false, sink);
                }
            } else if ((front || K.double_side) && (!SKIP_ZEROS || g0 != 0 || g1 != 0 || g2 != 0)) {
                const T zn = (K.far_ - zp) / (K.far_ - K.near_);
                const T s = fr.D * exp((zn - smax) / K.gamma) / pix(8);  // :608
                if (!SKIP_ZEROS || s != 0) {
                    if (TEXGRAD)
                        add_texture_grad(gtex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, s, g0, g1, g2, true, sink);
                    T t0, t1, t2;
                    sample_texture(tex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, t0, t1, t2);
                    T Crgb = 0;
                    Crgb += g0 * (t0 - pix(4));
                    Crgb += g1 * (t1 - pix(5));
                    Crgb += g2 * (t2 - pix(6));
                    Crgb *= s;
                    if (!SKIP_ZEROS || Crgb != 0) {
                        Cxy += Crgb / fr.D;
                        const T Cz = Crgb / K.gamma / (K.near_ - K.far_) * zp * zp;  // :624
                        gz0 = Cz * k0 / rc[2] / rc[2];
                        gz1 = Cz * k1 / rc[5] / rc[5];
                        gz2 = Cz * k2 / rc[8] / rc[8];
                    }
                }
            }
            Cxy *= fr.D * (1 - fr.D) / K.sigma;  // :632
            gv[2] = gz0; gv[5] = gz1; gv[8] = gz2;
            if (K.dist == UMR_DIST_EUCLIDEAN) {
                const T q = 2 * fr.sign * Cxy;  // :640
                gv[0] = q * (fr.t0 + fr.w0) * fr.dx;
                gv[1] = q * (fr.t0 + fr.w0) * fr.dy;
                gv[3] = q * (fr.t1 + fr.w1) * fr.dx;
                gv[4] = q * (fr.t1 + fr.w1) * fr.dy;
                gv[6] = q * (fr.t2 + fr.w2) * fr.dx;
                gv[7] = q * (fr.t2 + fr.w2) * fr.dy;
            } else if (K.dist == UMR_DIST_BARYCENTRIC) {  // kernel.cu:162-176
                const T w0 = fr.t0, w1 = fr.t1, w2 = fr.t2;  // unclipped barycentrics
                const int pidx = w0 > w1 ? (w1 > w2 ? 2 : 1) : (w0 > w2 ? 2 : 0);
                const double scale = fr.dis > 0 ? (2. * (double)sqrt(fr.dis)) : (2. * (double)sqrt(-fr.dis));
#pragma unroll
                for (int l = 0; l < 2; ++l) {
                    const T ip = rc[R_INV + 3 * pidx + l];
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        T gkl = 0;
                        gkl += -ip * rc[R_INV + 3 * k + 0] * xp;
                        gkl += -ip * rc[R_INV + 3 * k + 1] * yp;
                        gkl += -ip * rc[R_INV + 3 * k + 2] * (T)1;
                        gv[3 * k + l] = (T)((double)(gkl * Cxy) * scale);
                    }
                }
            }
        }
    }
}

// The float UMR-configuration pair (raster.cu), evaluated by the gather when GEN is false.
template <int RGB, bool TEXGRAD, int NC = 3, class Sink = TexRedSink, bool SPLIT = false>
__device__ __forceinline__ bool bwd_pair_acc(const float* __restrict__ rc, float xp, float yp, const Consts<float>& K,
                                             const float* __restrict__ sp, int f, const float* __restrict__ tex_img,
                                             float* __restrict__ gtex_img, float* acc, Sink sink = Sink());

// Face-parallel backward without atomics.  A (pixel, face) pair's gradient depends only on per-pixel constants and the face
// record, so every output gets exactly one writer: one warp owns a (texture group, face) pair and walks the group's images in
// ascending order and, in each, the face's cull box row by row (lanes across a row segment of 32 pixels).  Vertex gradients: a
// fixed shuffle tree, one plain store per image.  Texel gradients: lanes that hit the same texel are summed in ascending lane
// order, and the lowest of them adds the sum into the warp-owned texels of the face (plain load / store; __syncwarp orders the
// steps); grad_tex is zero-filled by the caller.  Every output is therefore bitwise reproducible.
// GEN: the generic modes (distance, alpha and texture mode read at run time), evaluated with bwd_pair_generic; a
// vertex-texture pair adds to the face's 9 corner colours, which the warp sums the same way.  Otherwise (float only) UMR's
// configuration, evaluated with bwd_pair_acc -- the recompute backward's arithmetic; SPLIT: see bwd_pair_acc.  RGB_SIL: the
// silhouette backward (colors_hi = the full-resolution alpha plane, grad_images = the alpha gradient; aggrs is not read).
template <typename T, int RGB, bool TEXGRAD, int NC = 3, bool GEN = false, bool SPLIT = false>
__global__ void __launch_bounds__(CTA) k_raster_bwd_det(const T* __restrict__ rec_all, const T* __restrict__ textures,
                                                        const T* __restrict__ colors_hi, const T* __restrict__ aggrs,
                                                        const T* __restrict__ grad_images, T* __restrict__ grad_faces,
                                                        T* __restrict__ grad_tex, Consts<T> K) {
    static_assert(std::is_same_v<T, float> || (GEN && NC == 3 && !SPLIT), "double runs the generic modes, 3 channels");
    static_assert(RGB != RGB_SIL || (!GEN && !TEXGRAD), "the silhouette backward is UMR's configuration, vertex gradients only");
    using PP = PixPlanes<RGB, NC>;
    constexpr int NPL = PP::NPL, NV = PP::NV, NP = CTA;  // planes: g[NC], g_alpha, C[NC], alpha, ssum, smax (PixPlanes)
    __shared__ T s_pix[NV][NP];
    __shared__ __align__(16) T s_rc[NWARP][REC_LEN];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int f = blockIdx.x * NWARP + warp;
    if (f >= K.F) return;  // warp-uniform; the warps share no memory
    const int grp = blockIdx.y, S = K.S, F = K.F;
    const T* tex_img = textures + (size_t)grp * K.tex_bs;
    T* gtex_img = TEXGRAD ? grad_tex + (size_t)grp * K.tex_bs : nullptr;
    T* sp = &s_pix[0][threadIdx.x];
    const T* rc = s_rc[warp];
    const size_t np = (size_t)S * S;
    for (int i = 0; i < K.tex_div; ++i) {
        const int b = grp * K.tex_div + i;
        __syncwarp();
        s_rc[warp][lane] = __ldg(rec_all + ((size_t)b * F + f) * REC_LEN + lane);
        __syncwarp();
        const T xlo = rc[R_BOX + 0], xhi = rc[R_BOX + 1], ylo = rc[R_BOX + 2], yhi = rc[R_BOX + 3];
        int c0, c1, j0, j1;
        pixel_span(xlo, xhi, S, c0, c1);
        pixel_span(ylo, yhi, S, j0, j1);  // j = S - 1 - row
        T acc[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) acc[k] = 0;
        for (int py = S - 1 - j1; py <= S - 1 - j0; ++py) {
            const T yp = pixel_coord<T>(S - 1 - py, S);
            if (yp > yhi || yp < ylo) continue;  // uniform
            for (int x0 = c0; x0 <= c1; x0 += 32) {
                const int px = x0 + lane;
                const T xp = pixel_coord<T>(px, S);
                T* taddr = nullptr;
                T tval[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
                if (px <= c1 && !(xp > xhi || xp < xlo)) {
                    const size_t p = (size_t)py * S + px;
                    if (K.aa) {  // avg_pool2d backward: g / 4
                        const size_t nq = (size_t)K.IS * K.IS;
                        const size_t q = (size_t)(py >> 1) * K.IS + (px >> 1);
#pragma unroll
                        for (int k = 0; k < NPL; ++k) sp[k * NP] = __ldg(grad_images + ((size_t)b * NPL + k) * nq + q) * (T)0.25;
                    } else {
#pragma unroll
                        for (int k = 0; k < NPL; ++k) sp[k * NP] = __ldg(grad_images + ((size_t)b * NPL + k) * np + p);
                    }
#pragma unroll
                    for (int k = 0; k < NPL; ++k) sp[(NPL + k) * NP] = __ldg(colors_hi + ((size_t)b * NPL + k) * np + p);
                    if (!PP::SIL) {
                        sp[(NV - 2) * NP] = __ldg(aggrs + ((size_t)b * 2 + 0) * np + p);
                        sp[(NV - 1) * NP] = __ldg(aggrs + ((size_t)b * 2 + 1) * np + p);
                    }
                    if constexpr (GEN) {
                        T gv[9];
#pragma unroll
                        for (int k = 0; k < 9; ++k) gv[k] = 0;
                        bool hit = false;
                        // float reads the pixel's inputs before the pair, double where the pair uses them (fewer live
                        // registers across the double fragment)
                        auto pix = [&] {
                            if constexpr (std::is_same_v<T, float>) {
                                const T v[NV] = {sp[0],      sp[NP],     sp[2 * NP], sp[3 * NP], sp[4 * NP],
                                                 sp[5 * NP], sp[6 * NP], sp[7 * NP], sp[8 * NP], sp[9 * NP]};
                                return [=](int k) { return v[k]; };
                            } else {
                                return [=](int k) { return sp[k * NP]; };
                            }
                        }();
                        bwd_pair_generic<RGB, TEXGRAD, TexTakeSink<T>>(rc, xp, yp, K, [=] { return f; }, pix, tex_img, gtex_img,
                                                                       gv, hit, TexTakeSink<T>{&taddr, tval});
                        if (hit) {
#pragma unroll
                            for (int k = 0; k < 9; ++k) acc[k] += gv[k];
                        }
                    } else {
                        bwd_pair_acc<RGB, TEXGRAD, NC, TexTakeSink<T>, SPLIT>(rc, xp, yp, K, sp, f, tex_img, gtex_img, acc,
                                                                               TexTakeSink<T>{&taddr, tval});
                    }
                }
                if (TEXGRAD) {
                    const bool has = taddr != nullptr;
                    uint32_t rem = __ballot_sync(0xffffffffu, has);
                    if (rem) {  // uniform
                        const uint32_t peers = __match_any_sync(0xffffffffu, (unsigned long long)(uintptr_t)taddr);
                        const bool vtx = GEN && K.tex != UMR_TEX_SURFACE;  // 9 corner-colour values instead of 3 texel channels
                        T sum[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
                        while (rem) {  // ascending lane order
                            const int o = __ffs(rem) - 1;
                            rem &= rem - 1u;
                            const bool mine = (peers >> o) & 1u;
#pragma unroll
                            for (int k = 0; k < 9; ++k) {
                                if (k < 3 || vtx) {
                                    const T v = __shfl_sync(0xffffffffu, tval[k], o);
                                    if (mine) sum[k] += v;
                                }
                            }
                        }
                        if (has && lane == __ffs(peers) - 1) {
#pragma unroll
                            for (int k = 0; k < 9; ++k)
                                if (k < 3 || vtx) taddr[k] = taddr[k] + sum[k];
                        }
                        __syncwarp();
                    }
                }
            }
        }
#pragma unroll
        for (int k = 0; k < 9; ++k) acc[k] = warp_sum(acc[k]);
        if (grad_faces != nullptr && lane < 9) {
            T v = acc[0];
#pragma unroll
            for (int k = 1; k < 9; ++k) v = (lane == k) ? acc[k] : v;
            grad_faces[((size_t)b * F + f) * 9 + lane] = v;
        }
    }
}

}  // namespace umr
