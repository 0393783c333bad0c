// raster_f64.cu -- the soft rasteriser in double precision (forward + backward) for sm_90a.
//
// An operation-for-operation twin of the `scalar_t = double` instantiation of the reference kernels
// external/SoftRas/soft_renderer/cuda/soft_rasterize_cuda_kernel.cu:22-659 ("kernel.cu"): same expression order, every
// operation one IEEE binary64 rounding (this translation unit is compiled with -fmad=false).  The scalar arguments are
// float, as in the reference binding (soft_rasterize_cuda.cpp:62-97), and are widened where they are used; the two
// float-typed expressions of the reference stay float: `dist_eps * sigma_val` (kernel.cu:333) and `exp(eps / gamma_val)`
// (:337, expf of a float quotient).  The two undefined corners of the reference keep the definitions of raster.cu
// (DESIGN.md §2).  Only exp() may differ from a CPU libm, by an ulp.
//
// All modes in one family, read at run time: hard / barycentric / euclidean distance, hard / sum / prod alpha, hard /
// softmax RGB, surface / vertex textures, single / double sided, 3 colour channels.
//
//   k_prep_f64         one thread per face -> a 256-byte record (vertices, barycentric inverse, Gram matrix + 1, cull box,
//                      obtuse / front flags) and the 32-byte cull box used for binning.  The cull box is the bound of the
//                      reference's bounding-box test (kernel.cu:32-38, :355), so "outside" is decided exactly as there.
//   k_raster_fwd_f64   one CTA per 16x16 pixel tile (a warp = an 8x4 block).  Windows of 1024 faces are tested against the
//                      tile and ballot-compacted into an ascending list of 32-bit face indices; the listed records are
//                      staged 32 at a time through shared memory and every pixel walks them in face order (running depth
//                      max, strict `<` z-test).  Fuses the background fill, the 2x2 average pool and the p2f sums.
//   k_raster_bwd_f64   face-parallel gather without atomics: one warp owns a (texture group, face), walks the group's
//                      images in ascending order and the face's cull box row by row; vertex gradients go through a fixed
//                      shuffle tree to one plain store, texel gradients are combined in ascending lane order.
//
// p2f: every per-pair term is bounded (a = exp_z * D <= 1, |grid| <= 1), so the sums are accumulated as fixed point with
// integer REDs, which are associative: a warp's 32 terms of one face are added in a fixed shuffle tree (|partial| <= 32),
// the partial is rounded to a multiple of 2^-P2F_FRAC_BITS and its 26-bit limbs are added into int64 words.  Rounding
// loses at most 2^-129 per partial; a face collects fewer than 2^36 partials (one per warp of a raster the grid can
// launch), so the accumulated error stays below 2^-93, which is under 2^-53 relative -- half an ulp -- of every sum that
// survives the clamp_min(1e-12) ~ 2^-40 of the finalize.  Every output of this file is therefore bitwise reproducible.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "common.cuh"
#include "umr_b200.h"

namespace umr {
namespace f64 {

constexpr int TILE = 16;
constexpr int CTA = TILE * TILE;
constexpr int NWARP = CTA / 32;
constexpr int CHUNK = 32;                // face records per shared-memory stage
constexpr int REC_D = 32;                // doubles per record (256 B)
constexpr int R_V = 0;                   // 9 : x0 y0 z0 x1 y1 z1 x2 y2 z2
constexpr int R_INV = 9;                 // 9 : barycentric inverse, row-major (faces_info[0..8])
constexpr int R_SYM = 18;                // 6 : s00 s01 s02 s11 s12 s22 (faces_info[9..17] is symmetric)
constexpr int R_BOX = 24;                // 4 : xlo xhi ylo yhi
constexpr int R_FLG = 28;                // 1 : bit0..2 obtuse corner, bit3 front-facing (an integer stored as double)
constexpr int WINDOW = 4 * CTA;          // faces tested per binning round (4 per thread)
constexpr int LIST_CAP = 2 * WINDOW;     // tile-list entries held before they are consumed

constexpr int P2F_LIMBS = 6;
constexpr int P2F_LIMB_BITS = 26;
constexpr int P2F_FRAC_BITS = 128;
constexpr int P2F_WORDS = 3 * P2F_LIMBS + 1;  // x, y, w limbs, then a word set when a partial was not finite
// the 16x16-tile grid (gridDim.y <= 65535) bounds the raster side, and with it the partials per face (see the header)
constexpr int MAX_RASTER = 65535 * TILE;

struct Consts {
    double thr, r, sigma, gamma, near_, far_;
    int F, T2, R, S, IS, aa, double_side;
    int dist, alpha, tex;
    size_t tex_bs;  // elements per texture (F * T2 * 3)
    int tex_div;    // consecutive images sharing one texture
};

__host__ __device__ inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
struct Layout { size_t rec_off, box_off, acc_off, total; };
inline Layout ws_layout(int B, int F) {
    const size_t n = (size_t)B * F;
    Layout L;
    L.rec_off = 0;
    L.box_off = align256(n * REC_D * sizeof(double));
    L.acc_off = L.box_off + align256(n * 4 * sizeof(double));
    L.total = L.acc_off + align256(n * P2F_WORDS * sizeof(unsigned long long));
    return L;
}

// the reference's max / min chains are comparisons (kernel.cu:32-38); a NaN operand propagates as they do there
__device__ __forceinline__ double sel_max(double a, double b) { return a > b ? a : b; }
__device__ __forceinline__ double sel_min(double a, double b) { return a < b ? a : b; }

// kernel.cu:222-282 and the per-face parts of :32-44
__global__ void __launch_bounds__(256) k_prep_f64(const double* __restrict__ fv, double* __restrict__ rec,
                                                  double* __restrict__ box, int F, double r) {
    const int fidx = blockIdx.x * blockDim.x + threadIdx.x;
    if (fidx >= F) return;
    const size_t i = (size_t)blockIdx.y * F + fidx;
    double v[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) v[k] = __ldg(fv + i * 9 + k);
    const double x0 = v[0], y0 = v[1], x1 = v[3], y1 = v[4], x2 = v[6], y2 = v[7];
    const double star[9] = {y1 - y2, x2 - x1, x1 * y2 - x2 * y1,  //
                            y2 - y0, x0 - x2, x2 * y0 - x0 * y2,  //
                            y0 - y1, x1 - x0, x0 * y1 - x1 * y0};
    double det = x2 * (y0 - y1) + x0 * (y1 - y2) + x1 * (y2 - y0);
    det = det > 0 ? fmax(det, 1e-10) : fmin(det, -1e-10);  // :259
    double* o = rec + i * REC_D;
#pragma unroll
    for (int k = 0; k < 9; ++k) o[R_V + k] = v[k];
#pragma unroll
    for (int k = 0; k < 9; ++k) o[R_INV + k] = star[k] / det;
    o[R_SYM + 0] = x0 * x0 + y0 * y0 + 1;
    o[R_SYM + 1] = x0 * x1 + y0 * y1 + 1;
    o[R_SYM + 2] = x0 * x2 + y0 * y2 + 1;
    o[R_SYM + 3] = x1 * x1 + y1 * y1 + 1;
    o[R_SYM + 4] = x1 * x2 + y1 * y2 + 1;
    o[R_SYM + 5] = x2 * x2 + y2 * y2 + 1;
    const double xlo = sel_min(sel_min(x0, x1), x2) - r, xhi = sel_max(sel_max(x0, x1), x2) + r;
    const double ylo = sel_min(sel_min(y0, y1), y2) - r, yhi = sel_max(sel_max(y0, y1), y2) + r;
    o[R_BOX + 0] = xlo; o[R_BOX + 1] = xhi; o[R_BOX + 2] = ylo; o[R_BOX + 3] = yhi;
    int flags = 0;  // first obtuse corner only, :273-281
    if ((x1 - x0) * (x2 - x0) + (y1 - y0) * (y2 - y0) < 0) flags = 1;
    else if ((x2 - x1) * (x0 - x1) + (y2 - y1) * (y0 - y1) < 0) flags = 2;
    else if ((x0 - x2) * (x1 - x2) + (y0 - y2) * (y1 - y2) < 0) flags = 4;
    if ((y2 - y0) * (x1 - x0) < (y1 - y0) * (x2 - x0)) flags |= 8;  // :42-44
    o[R_FLG] = (double)flags;
    o[R_FLG + 1] = 0.0; o[R_FLG + 2] = 0.0; o[R_FLG + 3] = 0.0;
    double* bx = box + i * 4;
    bx[0] = xlo; bx[1] = xhi; bx[2] = ylo; bx[3] = yhi;
}

struct Frag {
    double w0, w1, w2;  // unclipped barycentrics
    double t0, t1, t2;  // closest-point barycentrics minus w (barycentric distance: the unclipped w)
    double sign, dx, dy, dis, D;
};

__device__ __forceinline__ double pixel_coord(int i, int S) { return (2. * i + 1. - S) / S; }  // :325-326

__device__ __forceinline__ bool inside_closed(const Frag& fr) {  // :48-50
    return fr.w0 <= 1 && fr.w0 >= 0 && fr.w1 <= 1 && fr.w1 >= 0 && fr.w2 <= 1 && fr.w2 >= 0;
}

// distance + probability of one (pixel, face) pair past the bounding-box test: kernel.cu:25-29, :62-159, :368-384.
// Returns false when the pair is culled.
__device__ __forceinline__ bool fragment(const double* __restrict__ rc, double xp, double yp, const Consts& K, Frag& fr) {
    const double w0 = rc[R_INV + 0] * xp + rc[R_INV + 1] * yp + rc[R_INV + 2];
    const double w1 = rc[R_INV + 3] * xp + rc[R_INV + 4] * yp + rc[R_INV + 5];
    const double w2 = rc[R_INV + 6] * xp + rc[R_INV + 7] * yp + rc[R_INV + 8];
    fr.w0 = w0; fr.w1 = w1; fr.w2 = w2;
    fr.sign = 0.; fr.dx = 0.; fr.dy = 0.; fr.dis = 0.;
    if (K.dist == UMR_DIST_HARD) {  // :370-372
        fr.t0 = w0; fr.t1 = w1; fr.t2 = w2;
        fr.D = inside_closed(fr) ? 1. : 0.;
        return fr.D != 0.;
    }
    if (K.dist == UMR_DIST_BARYCENTRIC) {  // :156-159, :374-377
        const double m = w0 > w1 ? (w1 > w2 ? w2 : w1) : (w0 > w2 ? w2 : w0);
        const double dis = m > 0 ? m * m : -(m * m);
        fr.t0 = w0; fr.t1 = w1; fr.t2 = w2;
        fr.dis = dis;
        if (-dis >= K.thr) return false;
        fr.D = 1. / (1. + exp(-dis / K.sigma));
        return true;
    }
    const double fx0 = rc[0], fy0 = rc[1], fx1 = rc[3], fy1 = rc[4], fx2 = rc[6], fy2 = rc[7];
    const double s00 = rc[R_SYM + 0], s01 = rc[R_SYM + 1], s02 = rc[R_SYM + 2];
    const double s11 = rc[R_SYM + 3], s12 = rc[R_SYM + 4], s22 = rc[R_SYM + 5];
    double dx = 0., dy = 0., t0 = 0., t1 = 0., t2 = 0.;
    if (w0 > 0 && w1 > 0 && w2 > 0 && w0 < 1 && w1 < 1 && w2 < 1) {  // inside: the nearest of the three edges, :76-110
        double best = 100000000;
        {   // edge 0: v0 = 0, v1 = 1, v2 = 2
            const double a0 = s00 - s01, a1 = s01 - s11, a2 = s02 - s12;
            double u0 = (w0 * a0 + w1 * a1 + w2 * a2 - a1) / (a0 - a1);
            double u1 = 1 - u0;
            double u2 = 0;
            u0 -= w0; u1 -= w1; u2 -= w2;
            const double ex = u0 * fx0 + u1 * fx1 + u2 * fx2;
            const double ey = u0 * fy0 + u1 * fy1 + u2 * fy2;
            const double d = ex * ex + ey * ey;
            if (d < best) { best = d; dx = ex; dy = ey; t0 = u0; t1 = u1; t2 = u2; }
        }
        {   // edge 1: v0 = 1, v1 = 2, v2 = 0
            const double a0 = s01 - s02, a1 = s11 - s12, a2 = s12 - s22;
            double u1 = (w0 * a0 + w1 * a1 + w2 * a2 - a2) / (a1 - a2);
            double u2 = 1 - u1;
            double u0 = 0;
            u0 -= w0; u1 -= w1; u2 -= w2;
            const double ex = u0 * fx0 + u1 * fx1 + u2 * fx2;
            const double ey = u0 * fy0 + u1 * fy1 + u2 * fy2;
            const double d = ex * ex + ey * ey;
            if (d < best) { best = d; dx = ex; dy = ey; t0 = u0; t1 = u1; t2 = u2; }
        }
        {   // edge 2: v0 = 2, v1 = 0, v2 = 1
            const double a0 = s02 - s00, a1 = s12 - s01, a2 = s22 - s02;
            double u2 = (w0 * a0 + w1 * a1 + w2 * a2 - a0) / (a2 - a0);
            double u0 = 1 - u2;
            double u1 = 0;
            u0 -= w0; u1 -= w1; u2 -= w2;
            const double ex = u0 * fx0 + u1 * fx1 + u2 * fx2;
            const double ey = u0 * fy0 + u1 * fy1 + u2 * fy2;
            const double d = ex * ex + ey * ey;
            if (d < best) { best = d; dx = ex; dy = ey; t0 = u0; t1 = u1; t2 = u2; }
        }
        fr.sign = 1.;
    } else {  // outside: project on the one edge the sign pattern of w selects, with the obtuse-corner correction, :111-147
        const int flg = (int)rc[R_FLG];
        int v0 = -1;
        if (w1 <= 0 && w2 <= 0) {
            v0 = 0;
            if ((flg & 1) && (xp - fx0) * (fx2 - fx0) + (yp - fy0) * (fy2 - fy0) > 0) v0 = 2;
        } else if (w2 <= 0 && w0 <= 0) {
            v0 = 1;
            if ((flg & 2) && (xp - fx1) * (fx0 - fx1) + (yp - fy1) * (fy0 - fy1) > 0) v0 = 0;
        } else if (w0 <= 0 && w1 <= 0) {
            v0 = 2;
            if ((flg & 4) && (xp - fx2) * (fx1 - fx2) + (yp - fy2) * (fy1 - fy2) > 0) v0 = 1;
        } else if (w0 <= 0) v0 = 1;
        else if (w1 <= 0) v0 = 2;
        else if (w2 <= 0) v0 = 0;
        // every w > 0 but some w >= 1: undefined in the reference (:128-139 runs with v0 = -1); defined as "the corner
        // with the largest barycentric", as in raster.cu
        if (v0 < 0) v0 = w0 >= w1 ? (w0 >= w2 ? 0 : 2) : (w1 >= w2 ? 1 : 2);
        double u0, u1, u2;
        if (v0 == 0) {
            const double a0 = s00 - s01, a1 = s01 - s11, a2 = s02 - s12;
            u0 = (w0 * a0 + w1 * a1 + w2 * a2 - a1) / (a0 - a1);
            u1 = 1 - u0;
            u2 = 0;
        } else if (v0 == 1) {
            const double a0 = s01 - s02, a1 = s11 - s12, a2 = s12 - s22;
            u1 = (w0 * a0 + w1 * a1 + w2 * a2 - a2) / (a1 - a2);
            u2 = 1 - u1;
            u0 = 0;
        } else {
            const double a0 = s02 - s00, a1 = s12 - s01, a2 = s22 - s02;
            u2 = (w0 * a0 + w1 * a1 + w2 * a2 - a0) / (a2 - a0);
            u0 = 1 - u2;
            u1 = 0;
        }
        t0 = fmin(fmax(u0, 0.), 1.) - w0;  // :142-145
        t1 = fmin(fmax(u1, 0.), 1.) - w1;
        t2 = fmin(fmax(u2, 0.), 1.) - w2;
        dx = t0 * fx0 + t1 * fx1 + t2 * fx2;
        dy = t0 * fy0 + t1 * fy1 + t2 * fy2;
        fr.sign = -1.;
    }
    const double dis = dx * dx + dy * dy;
    fr.t0 = t0; fr.t1 = t1; fr.t2 = t2;
    fr.dx = dx; fr.dy = dy; fr.dis = dis;
    if (fr.sign < 0 && dis >= K.thr) return false;
    fr.D = 1. / (1. + exp(-fr.sign * dis / K.sigma));  // :383
    return true;
}

__device__ __forceinline__ void clip_bary(double& w0, double& w1, double& w2) {  // :54-59
    w0 = fmax(fmin(w0, 1 - 1e-5), 1e-5);
    w1 = fmax(fmin(w1, 1 - 1e-5), 1e-5);
    w2 = fmax(fmin(w2, 1 - 1e-5), 1e-5);
    const double s = fmax(w0 + w1 + w2, 1e-5);
    w0 /= s; w1 /= s; w2 /= s;
}

__device__ __forceinline__ int texel_index(double c0, double c1, int R) {  // :180-190
    const int wx = (int)(c0 * R);
    const int wy = (int)(c1 * R);
    if ((c0 + c1) * R - wx - wy <= 1) return wy * R + wx;
    return (R - 1 - wy) * R + (R - 1 - wx);
}

// colour of face texture `tx` (surface: [T2,3] texels; vertex: [3,3] corner colours), :179-195
__device__ __forceinline__ void sample_texture(const double* __restrict__ tx, double c0, double c1, double c2, const Consts& K,
                                               double& r, double& g, double& b) {
    if (K.tex == UMR_TEX_SURFACE) {
        const double* t = tx + (size_t)texel_index(c0, c1, K.R) * 3;
        r = __ldg(t); g = __ldg(t + 1); b = __ldg(t + 2);
    } else {
        r = c0 * __ldg(tx + 0) + c1 * __ldg(tx + 3) + c2 * __ldg(tx + 6);
        g = c0 * __ldg(tx + 1) + c1 * __ldg(tx + 4) + c2 * __ldg(tx + 7);
        b = c0 * __ldg(tx + 2) + c1 * __ldg(tx + 5) + c2 * __ldg(tx + 8);
    }
}

__device__ __forceinline__ void red_add_u64(unsigned long long* addr, unsigned long long v) {
    asm volatile("red.global.add.u64 [%0], %1;" ::"l"(addr), "l"(v) : "memory");
}

// adds round(|v| * 2^P2F_FRAC_BITS), with the sign of v, to the limb words (|v| <= 32 unless it is not finite)
__device__ __forceinline__ void red_fixed(unsigned long long* limbs, unsigned long long* bad, double v) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(v);
    const int e = (int)((u >> 52) & 0x7ffull);
    const int s = (e ? e : 1) - (1075 - P2F_FRAC_BITS);  // |v| * 2^128 = m * 2^s
    if (e == 0x7ff || s > P2F_LIMBS * P2F_LIMB_BITS - 53) {
        atomicOr(bad, 1ull);
        return;
    }
    unsigned long long m = (u & 0xfffffffffffffull) | (e ? (1ull << 52) : 0ull);
    int up = s;  // the integer is m * 2^up (up to 134 bits: its limbs are cut from the 53-bit m directly)
    if (s < 0) {
        if (s <= -54) return;
        m = (m + (1ull << (-s - 1))) >> (-s);  // round half away from zero
        up = 0;
    }
    const bool neg = (u >> 63) != 0;
#pragma unroll
    for (int k = 0; k < P2F_LIMBS; ++k) {
        const int d = k * P2F_LIMB_BITS - up;  // limb k = bits [d, d + 26) of m
        unsigned long long l = 0ull;
        if (d >= 0) l = d < 64 ? m >> d : 0ull;
        else if (-d < P2F_LIMB_BITS) l = m << -d;
        l &= (1ull << P2F_LIMB_BITS) - 1ull;
        if (l != 0ull) red_add_u64(limbs + k, neg ? 0ull - l : l);
    }
}

// The exact value of the limb words, rounded once to double (nearest even): carries are propagated upwards so every limb
// but the top one lies in [0, 2^26), the magnitude's leading 64 bits are taken with a sticky bit, and the hardware
// converts those to double.
__device__ __forceinline__ double fixed_value(const unsigned long long* words) {
    long long l[P2F_LIMBS];
    long long carry = 0;
#pragma unroll
    for (int k = 0; k < P2F_LIMBS; ++k) {
        const long long t = (long long)words[k] + carry;
        if (k < P2F_LIMBS - 1) {
            carry = t >> P2F_LIMB_BITS;  // arithmetic shift: floor
            l[k] = t - (carry << P2F_LIMB_BITS);
        } else {
            l[k] = t;
        }
    }
    const bool neg = l[P2F_LIMBS - 1] < 0;
    if (neg) {  // negate: limb-wise two's complement in base 2^26
        long long borrow = 0;
#pragma unroll
        for (int k = 0; k < P2F_LIMBS; ++k) {
            long long t = -l[k] - borrow;
            if (k < P2F_LIMBS - 1) {
                borrow = t < 0 ? 1 : 0;
                t += borrow << P2F_LIMB_BITS;
            }
            l[k] = t;
        }
    }
    int h = P2F_LIMBS - 1;
    while (h > 0 && l[h] == 0) --h;
    // four limbs from the leading one: at least 79 significant bits when the value is not tiny, and fewer than 2^127
    unsigned __int128 m = 0;
    bool sticky = false;
    for (int k = P2F_LIMBS - 1; k >= 0; --k) {
        if (k <= h && k > h - 4) m = (m << P2F_LIMB_BITS) | (unsigned __int128)(unsigned long long)l[k];
        else if (k <= h - 4 && l[k] != 0) sticky = true;
    }
    int expo = (h > 3 ? h - 3 : 0) * P2F_LIMB_BITS - P2F_FRAC_BITS;  // weight of bit 0 of m
    const unsigned long long hi = (unsigned long long)(m >> 64), lo = (unsigned long long)m;
    unsigned long long top;
    if (hi != 0ull) {
        const int sh = 64 - __clzll((long long)hi);  // bits to drop
        top = (unsigned long long)(m >> sh);
        if ((m & (((unsigned __int128)1 << sh) - 1)) != 0) sticky = true;
        expo += sh;
    } else {
        top = lo;
    }
    if (sticky) top |= 1ull;
    const double v = ldexp(__ull2double_rn(top), expo);
    return neg ? -v : v;
}

__global__ void k_p2f_finalize_f64(const unsigned long long* __restrict__ acc, double* __restrict__ p2f, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long* a = acc + i * P2F_WORDS;
    if (a[3 * P2F_LIMBS] != 0ull) {
        const double nan = __longlong_as_double(0x7ff8000000000000ll);
        p2f[2 * i] = nan; p2f[2 * i + 1] = nan;
        return;
    }
    const double x = fixed_value(a), y = fixed_value(a + P2F_LIMBS), w = fixed_value(a + 2 * P2F_LIMBS);
    const double d = fmax(w, 1e-12);  // soft_rasterize.py:73 clamp_min(1e-12)
    p2f[2 * i] = x / d;
    p2f[2 * i + 1] = y / d;
}

// =============================================================================================
// forward (kernel.cu:285-476, soft_rasterize.py:47-73, rasterizer.py:52-53)
// =============================================================================================
template <int RGB>
__global__ void __launch_bounds__(CTA, 2) k_raster_fwd_f64(const double* __restrict__ rec_all, const double* __restrict__ box_all,
                                                        const double* __restrict__ textures, double* __restrict__ images,
                                                        double* __restrict__ colors_hi, double* __restrict__ aggrs,
                                                        unsigned long long* __restrict__ p2f_acc, Consts K, float eps,
                                                        float bg0, float bg1, float bg2) {
    __shared__ __align__(16) double s_rec[CHUNK * REC_D];
    __shared__ uint32_t s_list[LIST_CAP];
    __shared__ int s_warp_cnt[NWARP];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z, S = K.S, F = K.F;
    const int px = blockIdx.x * TILE + (warp & 1) * 8 + (lane & 7);
    const int py = blockIdx.y * TILE + (warp >> 1) * 4 + (lane >> 3);  // image row (0 = top)
    const bool live = px < S && py < S;
    const double xp = pixel_coord(px, S), yp = pixel_coord(S - 1 - py, S);
    // tile extents in pixel-centre coordinates (monotone in the index, so the tile test is conservative)
    const double tx_first = pixel_coord(blockIdx.x * TILE, S), tx_last = pixel_coord(min((int)blockIdx.x * TILE + TILE - 1, S - 1), S);
    const double ty_top = pixel_coord(S - 1 - blockIdx.y * TILE, S);
    const double ty_bot = pixel_coord(S - 1 - min((int)blockIdx.y * TILE + TILE - 1, S - 1), S);

    // pixel state (:335-348)
    double acc_a = K.alpha == UMR_ALPHA_PROD ? 1. : 0.;
    double ssum = (double)expf(eps / (float)K.gamma);  // :337 is a float expression
    double smax = (double)eps;
    double c0 = bg0, c1 = bg1, c2 = bg2;
    if (RGB == 1) { c0 = c0 * ssum; c1 = c1 * ssum; c2 = c2 * ssum; }
    double zmin = 10000000;
    int fid = -1;

    const double* tex_img = textures + (size_t)(b / K.tex_div) * K.tex_bs;
    // the float32 affine_grid (align_corners=True) coordinates of this pixel, widened: soft_rasterize.py:58-62 builds
    // the grid from a float theta
    // S = 1: torch 1.1's affine_grid takes linspace(-1, 1, 1) = [-1] (DESIGN.md §2), where 2 / 0 would give -1 + inf * 0 = NaN
    const float gstep = S > 1 ? 2.f / (float)(S - 1) : 0.f;
    const double gx = (double)((px * 2 < S) ? (-1.f + gstep * px) : (1.f - gstep * (S - 1 - px)));
    const double gy = (double)((py * 2 < S) ? (-1.f + gstep * py) : (1.f - gstep * (S - 1 - py)));

    const double* box = box_all + (size_t)b * F * 4;
    const double* rec_img = rec_all + (size_t)b * F * REC_D;
    int n = 0;  // listed faces not consumed yet (uniform)
    for (int base = 0; base < F; base += WINDOW) {
        {
            // ordered compaction of the window's faces whose cull box touches the tile: warp w owns faces
            // [128 w, 128 w + 128) of the window, 32 per round
            uint32_t masks[WINDOW / CTA];
            int cnt = 0;
#pragma unroll
            for (int r = 0; r < WINDOW / CTA; ++r) {
                const int f = base + warp * (WINDOW / NWARP) + r * 32 + lane;
                bool hit = false;
                if (f < F) {
                    const double2 lo = __ldg(reinterpret_cast<const double2*>(box + (size_t)f * 4));
                    const double2 hi = __ldg(reinterpret_cast<const double2*>(box + (size_t)f * 4) + 1);
                    hit = !(tx_first > lo.y || tx_last < lo.x || ty_bot > hi.y || ty_top < hi.x);
                }
                masks[r] = __ballot_sync(0xffffffffu, hit);
                cnt += __popc(masks[r]);
            }
            if (lane == 0) s_warp_cnt[warp] = cnt;
            __syncthreads();
            int off = n, total = 0;
#pragma unroll
            for (int w = 0; w < NWARP; ++w) {
                const int c = s_warp_cnt[w];
                if (w < warp) off += c;
                total += c;
            }
            const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
            for (int r = 0; r < WINDOW / CTA; ++r) {
                if ((masks[r] >> lane) & 1u)
                    s_list[off + __popc(masks[r] & lt)] = (uint32_t)(base + warp * (WINDOW / NWARP) + r * 32 + lane);
                off += __popc(masks[r]);
            }
            n += total;
            __syncthreads();  // list visible; s_warp_cnt reusable
            if (n <= LIST_CAP - WINDOW && base + WINDOW < F) continue;  // room for another window
        }
        // consume the list: 32 records per stage
        for (int c = 0; c * CHUNK < n; ++c) {
            const int cnt = min(CHUNK, n - c * CHUNK);
            {
                const int j = tid >> 3, q = tid & 7;  // 8 threads copy one 256-byte record
                if (j < cnt) {
                    const double2* src = reinterpret_cast<const double2*>(rec_img + (size_t)s_list[c * CHUNK + j] * REC_D) + q * 2;
                    double2* dst = reinterpret_cast<double2*>(s_rec + j * REC_D) + q * 2;
                    dst[0] = __ldg(src);
                    dst[1] = __ldg(src + 1);
                }
            }
            __syncthreads();
            double own_x = 0., own_y = 0., own_w = 0.;  // p2f partials of this warp: lane j owns stage face j
            for (int j = 0; j < cnt; ++j) {
                const double* rc = s_rec + j * REC_D;
                double a_x = 0., a_y = 0., a_w = 0.;
                bool contrib = false;
                // :355 bounding-box test
                if (live && !(xp > rc[R_BOX + 1] || xp < rc[R_BOX + 0] || yp > rc[R_BOX + 3] || yp < rc[R_BOX + 2])) {
                    Frag fr;
                    if (fragment(rc, xp, yp, K, fr)) {
                        if (K.alpha == UMR_ALPHA_PROD) acc_a = acc_a * (1. - fr.D);  // :396
                        else if (K.alpha == UMR_ALPHA_SUM) acc_a += fr.D;           // :394
                        else if (fr.D > 0.5) acc_a = 1.;                            // :392
                        double k0 = fr.w0, k1 = fr.w1, k2 = fr.w2;
                        clip_bary(k0, k1, k2);
                        const double zp = 1. / (k0 / rc[2] + k1 / rc[5] + k2 / rc[8]);  // :403
                        if (!(zp < K.near_ || zp > K.far_)) {
                            const bool front = ((int)rc[R_FLG] & 8) != 0;
                            const uint32_t f = s_list[c * CHUNK + j];
                            if (RGB == 0) {
                                if (zp < zmin && inside_closed(fr) && (K.double_side || front)) {
                                    zmin = zp;
                                    fid = (int)f;
                                    double t0, t1, t2;
                                    sample_texture(tex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, t0, t1, t2);
                                    c0 = t0; c1 = t1; c2 = t2;
                                }
                            } else if (front || K.double_side) {
                                const double zn = (K.far_ - zp) / (K.far_ - K.near_);
                                double ed = 1.;
                                if (zn > smax) { ed = exp((smax - zn) / K.gamma); smax = zn; }
                                const double ez = exp((zn - smax) / K.gamma);
                                ssum = ed * ssum + ez * fr.D;
                                const double a = ez * fr.D;
                                a_x = a * gx; a_y = a * gy; a_w = a;
                                contrib = a != 0.;
                                double t0, t1, t2;
                                sample_texture(tex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, t0, t1, t2);
                                c0 = ed * c0 + a * t0;
                                c1 = ed * c1 + a * t1;
                                c2 = ed * c2 + a * t2;
                            }
                        }
                    }
                }
                if (RGB == 1 && p2f_acc != nullptr && __any_sync(0xffffffffu, contrib)) {
                    a_x = warp_sum(a_x); a_y = warp_sum(a_y); a_w = warp_sum(a_w);
                    if (lane == j) { own_x = a_x; own_y = a_y; own_w = a_w; }
                }
            }
            if (RGB == 1 && p2f_acc != nullptr && lane < cnt && own_w != 0.) {  // one update per (warp, face, component)
                unsigned long long* acc = p2f_acc + ((size_t)b * F + s_list[c * CHUNK + lane]) * P2F_WORDS;
                red_fixed(acc, acc + 3 * P2F_LIMBS, own_x);
                red_fixed(acc + P2F_LIMBS, acc + 3 * P2F_LIMBS, own_y);
                red_fixed(acc + 2 * P2F_LIMBS, acc + 3 * P2F_LIMBS, own_w);
            }
            __syncthreads();  // everyone is done with the stage (and, after the last one, with the list)
        }
        n = 0;
    }

    // finalise (:443-475)
    double alpha;
    if (K.alpha == UMR_ALPHA_PROD) alpha = 1. - acc_a;
    else if (K.alpha == UMR_ALPHA_SUM) alpha = acc_a / K.F;
    else alpha = acc_a;
    double v[4], g0, g1;
    if (RGB == 0) {
        v[0] = c0; v[1] = c1; v[2] = c2;  // the background where no face won
        g0 = zmin; g1 = (double)fid;
    } else {
        v[0] = c0 / ssum; v[1] = c1 / ssum; v[2] = c2 / ssum;
        g0 = ssum; g1 = smax;
    }
    v[3] = alpha;
    const size_t np = (size_t)S * S;
    if (live) {
        const size_t p = (size_t)py * S + px;
        aggrs[((size_t)b * 2 + 0) * np + p] = g0;
        aggrs[((size_t)b * 2 + 1) * np + p] = g1;
        if (colors_hi != nullptr) {
#pragma unroll
            for (int k = 0; k < 4; ++k) colors_hi[((size_t)b * 4 + k) * np + p] = v[k];
        }
    }
    if (K.aa) {
        // avg_pool2d(2, 2) = ((a00 + a01) + a10) + a11, then * 0.25 (rasterizer.py:52-53); S is even, so a live
        // (even x, even y) lane has a live quad at lanes ^1, ^8, ^9
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const double a01 = __shfl_xor_sync(0xffffffffu, v[k], 1);
            const double a10 = __shfl_xor_sync(0xffffffffu, v[k], 8);
            const double a11 = __shfl_xor_sync(0xffffffffu, v[k], 9);
            v[k] = (((v[k] + a01) + a10) + a11) * 0.25;
        }
        if (live && (lane & 1) == 0 && (lane & 8) == 0) {
            const size_t nq = (size_t)K.IS * K.IS;
            const size_t q = (size_t)(py >> 1) * K.IS + (px >> 1);
#pragma unroll
            for (int k = 0; k < 4; ++k) images[((size_t)b * 4 + k) * nq + q] = v[k];
        }
    } else if (live && images != colors_hi) {
        const size_t p = (size_t)py * S + px;
#pragma unroll
        for (int k = 0; k < 4; ++k) images[((size_t)b * 4 + k) * np + p] = v[k];
    }
}

// =============================================================================================
// backward (kernel.cu:479-656, rasterizer.py:52-53 pool backward)
// =============================================================================================
// Conservative index range [i0, i1] of the pixels whose centre coordinate lies in [lo, hi] (one index of slack on each
// side; the exact test runs per pixel).  NaN bounds keep every index, as the tile test of the forward does.
__device__ __forceinline__ void box_span(double lo, double hi, int S, int& i0, int& i1) {
    const double a = (lo * S + (S - 1)) * 0.5, c = (hi * S + (S - 1)) * 0.5;
    i0 = a > 0.0 ? (a < (double)S ? (int)a - 1 : S) : 0;
    i1 = c < (double)(S - 1) ? (c > -1.0 ? (int)c + 1 : -1) : S - 1;  // c in (-1, 0): pixel 0 may still lie in the box
    i0 = max(i0, 0);
    i1 = min(i1, S - 1);
}

// One warp per (texture group, face).  A pair's gradient depends only on per-pixel constants and the face record, so every
// output has one writer: vertex gradients are summed per lane over the face's pixels, then across the warp in a fixed
// shuffle tree and stored; the lanes of a step that hit the same texel (surface) or the face's corner colours (vertex
// textures) are summed in ascending lane order and the lowest of them adds the sum to the warp-owned texels with a plain
// load and store.  grad_tex is zero-filled by the caller.
template <int RGB, bool TEXGRAD>
__global__ void __launch_bounds__(CTA) k_raster_bwd_f64(const double* __restrict__ rec_all, const double* __restrict__ textures,
                                                        const double* __restrict__ colors_hi, const double* __restrict__ aggrs,
                                                        const double* __restrict__ grad_images, double* __restrict__ grad_faces,
                                                        double* __restrict__ grad_tex, Consts K) {
    __shared__ __align__(16) double s_rc[NWARP][REC_D];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int f = blockIdx.x * NWARP + warp;
    if (f >= K.F) return;  // warp-uniform; the warps share no memory
    const int grp = blockIdx.y, S = K.S, F = K.F;
    const double* tx = textures + (size_t)grp * K.tex_bs + (size_t)f * K.T2 * 3;
    double* gt = TEXGRAD ? grad_tex + (size_t)grp * K.tex_bs + (size_t)f * K.T2 * 3 : nullptr;
    const double* rc = s_rc[warp];
    const size_t np = (size_t)S * S;
    const bool vtx = K.tex != UMR_TEX_SURFACE;  // 9 corner-colour values per pair instead of 3 texel channels
    for (int i = 0; i < K.tex_div; ++i) {
        const int b = grp * K.tex_div + i;
        __syncwarp();
        s_rc[warp][lane] = __ldg(rec_all + ((size_t)b * F + f) * REC_D + lane);
        __syncwarp();
        const double xlo = rc[R_BOX + 0], xhi = rc[R_BOX + 1], ylo = rc[R_BOX + 2], yhi = rc[R_BOX + 3];
        const bool front = ((int)rc[R_FLG] & 8) != 0;
        int x_first, x_last, j0, j1;
        box_span(xlo, xhi, S, x_first, x_last);
        box_span(ylo, yhi, S, j0, j1);  // j = S - 1 - row
        double acc[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) acc[k] = 0.;
        for (int py = S - 1 - j1; py <= S - 1 - j0; ++py) {
            const double yp = pixel_coord(S - 1 - py, S);
            if (yp > yhi || yp < ylo) continue;  // uniform
            for (int x0 = x_first; x0 <= x_last; x0 += 32) {
                const int px = x0 + lane;
                const double xp = pixel_coord(px, S);
                long long toff = -1;  // first texture element this pair adds to, relative to the face's texture
                double tval[9] = {0., 0., 0., 0., 0., 0., 0., 0., 0.};
                Frag fr;
                if (px <= x_last && !(xp > xhi || xp < xlo) && fragment(rc, xp, yp, K, fr)) {
                    const size_t p = (size_t)py * S + px;
                    double g[4];
                    if (K.aa) {  // avg_pool2d backward: g / 4
                        const size_t nq = (size_t)K.IS * K.IS, q = (size_t)(py >> 1) * K.IS + (px >> 1);
#pragma unroll
                        for (int k = 0; k < 4; ++k) g[k] = __ldg(grad_images + ((size_t)b * 4 + k) * nq + q) / 4.;
                    } else {
#pragma unroll
                        for (int k = 0; k < 4; ++k) g[k] = __ldg(grad_images + ((size_t)b * 4 + k) * np + p);
                    }
                    const double C3 = __ldg(colors_hi + ((size_t)b * 4 + 3) * np + p);
                    const double ssum = __ldg(aggrs + ((size_t)b * 2 + 0) * np + p);
                    const double smax = __ldg(aggrs + ((size_t)b * 2 + 1) * np + p);
                    // alpha: :577-585 (hard alpha passes the raw gradient through, as the reference does)
                    double Ca = g[3];
                    if (K.alpha == UMR_ALPHA_SUM) Ca /= K.F;
                    else if (K.alpha == UMR_ALPHA_PROD) Ca = Ca * ((1 - C3) / fmax(1 - fr.D, 1e-6));
                    double Cxy = 0;
                    Cxy += Ca;
                    double k0 = fr.w0, k1 = fr.w1, k2 = fr.w2;
                    clip_bary(k0, k1, k2);
                    const double zp = 1. / (k0 / rc[2] + k1 / rc[5] + k2 / rc[8]);
                    if (!(zp < K.near_ || zp > K.far_)) {  // :592 drops the alpha gradient as well
                        double gz0 = 0., gz1 = 0., gz2 = 0.;
                        const double kw[3] = {k0, k1, k2};
                        if (RGB == 0) {
                            if ((double)f == smax) {  // aggrs[1] = winning face id (:596)
                                if (TEXGRAD) {
                                    if (!vtx) {
                                        toff = (long long)texel_index(k0, k1, K.R) * 3;
                                        tval[0] = g[0]; tval[1] = g[1]; tval[2] = g[2];
                                    } else {
                                        toff = 0;
#pragma unroll
                                        for (int j = 0; j < 3; ++j)
#pragma unroll
                                            for (int k = 0; k < 3; ++k) tval[3 * j + k] = kw[j] * g[k];
                                    }
                                }
                            }
                        } else if (front || K.double_side) {
                            const double zn = (K.far_ - zp) / (K.far_ - K.near_);
                            const double s = fr.D * exp((zn - smax) / K.gamma) / ssum;  // :608
                            if (TEXGRAD) {
                                if (!vtx) {
                                    toff = (long long)texel_index(k0, k1, K.R) * 3;
                                    tval[0] = s * g[0]; tval[1] = s * g[1]; tval[2] = s * g[2];
                                } else {
                                    toff = 0;
#pragma unroll
                                    for (int j = 0; j < 3; ++j)
#pragma unroll
                                        for (int k = 0; k < 3; ++k) tval[3 * j + k] = s * (kw[j] * g[k]);
                                }
                            }
                            double t[3];
                            sample_texture(tx, k0, k1, k2, K, t[0], t[1], t[2]);
                            double Crgb = 0.;
#pragma unroll
                            for (int k = 0; k < 3; ++k)
                                Crgb += g[k] * (t[k] - __ldg(colors_hi + ((size_t)b * 4 + k) * np + p));
                            Crgb *= s;
                            Cxy += Crgb / fr.D;
                            const double Cz = Crgb / K.gamma / (K.near_ - K.far_) * zp * zp;  // :624
                            gz0 = Cz * k0 / rc[2] / rc[2];
                            gz1 = Cz * k1 / rc[5] / rc[5];
                            gz2 = Cz * k2 / rc[8] / rc[8];
                        }
                        Cxy *= fr.D * (1 - fr.D) / K.sigma;  // :632
                        double gv[9] = {0., 0., gz0, 0., 0., gz1, 0., 0., gz2};
                        if (K.dist == UMR_DIST_EUCLIDEAN) {  // :637-642
                            const double w0[3] = {fr.w0, fr.w1, fr.w2}, t[3] = {fr.t0, fr.t1, fr.t2};
#pragma unroll
                            for (int k = 0; k < 3; ++k) {
                                gv[3 * k + 0] = 2 * fr.sign * Cxy * (t[k] + w0[k]) * fr.dx;
                                gv[3 * k + 1] = 2 * fr.sign * Cxy * (t[k] + w0[k]) * fr.dy;
                            }
                        } else if (K.dist == UMR_DIST_BARYCENTRIC) {  // :162-176, :634-635
                            const int pidx = fr.t0 > fr.t1 ? (fr.t1 > fr.t2 ? 2 : 1) : (fr.t0 > fr.t2 ? 2 : 0);
                            const double scale = fr.dis > 0 ? (2. * sqrt(fr.dis)) : (2. * sqrt(-fr.dis));
#pragma unroll
                            for (int l = 0; l < 2; ++l) {
                                const double ip = rc[R_INV + 3 * pidx + l];
#pragma unroll
                                for (int k = 0; k < 3; ++k) {
                                    double gkl = 0;
                                    gkl += -ip * rc[R_INV + 3 * k + 0] * xp;
                                    gkl += -ip * rc[R_INV + 3 * k + 1] * yp;
                                    gkl += -ip * rc[R_INV + 3 * k + 2] * 1.;
                                    gv[3 * k + l] = gkl * Cxy * scale;
                                }
                            }
                        }
#pragma unroll
                        for (int k = 0; k < 9; ++k) acc[k] += gv[k];
                    }
                }
                if (TEXGRAD) {
                    uint32_t rem = __ballot_sync(0xffffffffu, toff >= 0);
                    if (rem) {  // uniform
                        const uint32_t peers = __match_any_sync(0xffffffffu, toff);
                        double sum[9] = {0., 0., 0., 0., 0., 0., 0., 0., 0.};
                        while (rem) {  // ascending lane order
                            const int o = __ffs(rem) - 1;
                            rem &= rem - 1u;
                            const bool mine = (peers >> o) & 1u;
#pragma unroll
                            for (int k = 0; k < 9; ++k) {
                                if (k < 3 || vtx) {
                                    const double v = __shfl_sync(0xffffffffu, tval[k], o);
                                    if (mine) sum[k] += v;
                                }
                            }
                        }
                        if (toff >= 0 && lane == __ffs(peers) - 1) {
#pragma unroll
                            for (int k = 0; k < 9; ++k)
                                if (k < 3 || vtx) gt[toff + k] = gt[toff + k] + sum[k];
                        }
                        __syncwarp();
                    }
                }
            }
        }
#pragma unroll
        for (int k = 0; k < 9; ++k) acc[k] = warp_sum(acc[k]);
        if (grad_faces != nullptr && lane < 9) {
            double v = acc[0];
#pragma unroll
            for (int k = 1; k < 9; ++k) v = (lane == k) ? acc[k] : v;
            grad_faces[((size_t)b * F + f) * 9 + lane] = v;
        }
    }
}

}  // namespace f64
}  // namespace umr

// =============================================================================================
// C ABI
// =============================================================================================
using namespace umr;
using namespace umr::f64;

// the checks of umr_raster_forward / umr_raster_backward, with 3 colour channels only
static int check_params_f64(const UmrRasterParams* p) {
    if (!p) return UMR_ERR_BAD_ARG;
    if (p->batch_size <= 0 || p->num_faces <= 0 || p->texture_size <= 0 || p->image_size <= 0) return UMR_ERR_BAD_ARG;
    if (p->num_faces > UMR_RASTER_MAX_FACES || p->batch_size > 65535) return UMR_ERR_TOO_LARGE;
    if ((int64_t)p->image_size * (p->anti_aliasing ? 2 : 1) > MAX_RASTER) return UMR_ERR_TOO_LARGE;
    if (p->func_id_dist < 0 || p->func_id_dist > 2 || p->func_id_alpha < 0 || p->func_id_alpha > 2 ||
        p->texture_sample_type < 0 || p->texture_sample_type > 1)
        return UMR_ERR_UNSUPPORTED;
    if (p->texture_sample_type == UMR_TEX_VERTEX && p->texture_size != 3) return UMR_ERR_BAD_ARG;  // [B,F,3,3]
    if (p->shared_textures > 1 && p->batch_size % p->shared_textures != 0) return UMR_ERR_BAD_ARG;
    if (p->func_id_rgb != UMR_RGB_HARD && p->func_id_rgb != UMR_RGB_SOFTMAX) return UMR_ERR_UNSUPPORTED;
    if (p->color_channels != 0 && p->color_channels != 3) return UMR_ERR_BAD_ARG;
    return UMR_OK;
}

static f64::Consts make_consts_f64(const UmrRasterParams* p) {
    f64::Consts K;
    K.thr = (double)(p->dist_eps * p->sigma_val);  // kernel.cu:333: float * float, then scalar_t
    K.r = sqrt(K.thr);                             // :355
    K.sigma = p->sigma_val;
    K.gamma = p->gamma_val;
    K.near_ = p->near_plane;
    K.far_ = p->far_plane;
    K.F = p->num_faces;
    K.T2 = p->texture_size;
    K.R = (int)sqrt((double)p->texture_size);  // :685
    K.IS = p->image_size;
    K.aa = p->anti_aliasing ? 1 : 0;
    K.S = p->image_size * (K.aa ? 2 : 1);
    K.double_side = p->double_side ? 1 : 0;
    K.dist = p->func_id_dist;
    K.alpha = p->func_id_alpha;
    K.tex = p->texture_sample_type;
    K.tex_bs = (size_t)p->num_faces * p->texture_size * 3;
    K.tex_div = p->shared_textures > 1 ? p->shared_textures : 1;
    return K;
}

extern "C" size_t umr_raster_workspace_bytes_f64(int32_t B, int32_t F, int32_t image_size, int32_t anti_aliasing) {
    (void)anti_aliasing;
    if (B <= 0 || F <= 0 || image_size <= 0) return 0;
    return f64::ws_layout(B, F).total;
}

extern "C" int umr_raster_forward_f64(const double* face_vertices, const double* textures, double* images,
                                      double* soft_colors, double* aggrs_info, double* p2f_info,
                                      const UmrRasterParams* p, void* workspace, void* stream_) {
    int rc = check_params_f64(p);
    if (rc) return rc;
    if (!face_vertices || !textures || !images || !aggrs_info || !workspace) return UMR_ERR_BAD_ARG;
    if (((uintptr_t)workspace & 255) != 0) return UMR_ERR_BAD_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    const int B = p->batch_size, F = p->num_faces;
    const f64::Consts K = make_consts_f64(p);
    if (!K.aa && soft_colors == nullptr) soft_colors = images;
    const f64::Layout L = f64::ws_layout(B, F);
    char* ws = (char*)workspace;
    double* rec = (double*)(ws + L.rec_off);
    double* box = (double*)(ws + L.box_off);
    unsigned long long* acc = (unsigned long long*)(ws + L.acc_off);
    const size_t n = (size_t)B * F;
    const bool softmax = p->func_id_rgb == UMR_RGB_SOFTMAX;
    const bool want_p2f = p2f_info != nullptr;
    k_prep_f64<<<dim3((F + 255) / 256, B), 256, 0, stream>>>(face_vertices, rec, box, F, K.r);
    if (want_p2f) {
        // hard mode never accumulates p2f (kernel.cu:417-431 is softmax-only) -> zeros
        cudaError_t e = softmax ? cudaMemsetAsync(acc, 0, n * P2F_WORDS * sizeof(unsigned long long), stream)
                                : cudaMemsetAsync(p2f_info, 0, n * 2 * sizeof(double), stream);
        if (e != cudaSuccess) return (int)e;
    }
    const dim3 grid((K.S + TILE - 1) / TILE, (K.S + TILE - 1) / TILE, B);
    if (p->ev_kernel_start) cudaEventRecord((cudaEvent_t)p->ev_kernel_start, stream);
    if (softmax)
        k_raster_fwd_f64<1><<<grid, CTA, 0, stream>>>(rec, box, textures, images, soft_colors, aggrs_info,
                                                     want_p2f ? acc : nullptr, K, p->eps, p->background_color[0],
                                                     p->background_color[1], p->background_color[2]);
    else
        k_raster_fwd_f64<0><<<grid, CTA, 0, stream>>>(rec, box, textures, images, soft_colors, aggrs_info, nullptr, K, p->eps,
                                                     p->background_color[0], p->background_color[1], p->background_color[2]);
    if (p->ev_kernel_stop) cudaEventRecord((cudaEvent_t)p->ev_kernel_stop, stream);
    count_launch(2);
    if (want_p2f && softmax) {
        k_p2f_finalize_f64<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(acc, p2f_info, n);
        count_launch();
    }
    return (int)cudaGetLastError();
}

extern "C" int umr_raster_backward_f64(const double* face_vertices, const double* textures, const double* soft_colors,
                                       const double* aggrs_info, const double* grad_images, double* grad_faces,
                                       double* grad_textures, const UmrRasterParams* p, void* workspace, void* stream_) {
    int rc = check_params_f64(p);
    if (rc) return rc;
    if (!face_vertices || !textures || !soft_colors || !aggrs_info || !grad_images || !workspace) return UMR_ERR_BAD_ARG;
    if (!grad_faces && !grad_textures) return UMR_ERR_BAD_ARG;
    if (((uintptr_t)workspace & 255) != 0) return UMR_ERR_BAD_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    const int B = p->batch_size, F = p->num_faces;
    const f64::Consts K = make_consts_f64(p);
    const f64::Layout L = f64::ws_layout(B, F);
    char* ws = (char*)workspace;
    double* rec = (double*)(ws + L.rec_off);
    double* box = (double*)(ws + L.box_off);
    const size_t n = (size_t)B * F;
    k_prep_f64<<<dim3((F + 255) / 256, B), 256, 0, stream>>>(face_vertices, rec, box, F, K.r);
    if (grad_textures) {
        cudaError_t e = cudaMemsetAsync(grad_textures, 0, (n / K.tex_div) * p->texture_size * 3 * sizeof(double), stream);
        if (e != cudaSuccess) return (int)e;
    }
    const dim3 grid((unsigned)((F + NWARP - 1) / NWARP), (unsigned)(B / K.tex_div));
    const bool softmax = p->func_id_rgb == UMR_RGB_SOFTMAX;
    if (p->ev_kernel_start) cudaEventRecord((cudaEvent_t)p->ev_kernel_start, stream);
#define UMR_BWD_F64(RGBM, TG) \
    k_raster_bwd_f64<RGBM, TG><<<grid, CTA, 0, stream>>>(rec, textures, soft_colors, aggrs_info, grad_images, grad_faces, grad_textures, K)
    if (softmax) { if (grad_textures) UMR_BWD_F64(1, true); else UMR_BWD_F64(1, false); }
    else { if (grad_textures) UMR_BWD_F64(0, true); else UMR_BWD_F64(0, false); }
#undef UMR_BWD_F64
    if (p->ev_kernel_stop) cudaEventRecord((cudaEvent_t)p->ev_kernel_stop, stream);
    count_launch(2);
    return (int)cudaGetLastError();
}
