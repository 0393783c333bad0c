// raster_f64.cu -- the soft rasteriser in double precision (forward + backward) for sm_90a.
//
// The `scalar_t = double` instantiation of the reference kernels
// external/SoftRas/soft_renderer/cuda/soft_rasterize_cuda_kernel.cu:22-659 ("kernel.cu"): same expression order, every
// operation one IEEE binary64 rounding (this translation unit is compiled with -fmad=false).  The per-pair arithmetic and the
// backward are the double instantiations of raster_generic.cuh, which raster.cu instantiates for float.  The scalar arguments are
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
//   backward           k_raster_bwd_det<double, RGB, TEXGRAD, 3, GEN = true> (raster_generic.cuh): the face-parallel gather
//                      without atomics, over these records.
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
#include "raster_generic.cuh"
#include "umr_b200.h"

namespace umr {
namespace f64 {

constexpr int CHUNK = 32;                // face records per shared-memory stage
constexpr int WINDOW = 4 * CTA;          // faces tested per binning round (4 per thread)
constexpr int LIST_CAP = 2 * WINDOW;     // tile-list entries held before they are consumed

constexpr int P2F_LIMBS = 6;
constexpr int P2F_LIMB_BITS = 26;
constexpr int P2F_FRAC_BITS = 128;
constexpr int P2F_WORDS = 3 * P2F_LIMBS + 1;  // x, y, w limbs, then a word set when a partial was not finite

__host__ __device__ inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
struct Layout { size_t rec_off, box_off, acc_off, total; };
inline Layout ws_layout(int B, int F) {
    const size_t n = (size_t)B * F;
    Layout L;
    L.rec_off = 0;
    L.box_off = align256(n * REC_LEN * sizeof(double));
    L.acc_off = L.box_off + align256(n * 4 * sizeof(double));
    L.total = L.acc_off + align256(n * P2F_WORDS * sizeof(unsigned long long));
    return L;
}

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
    double* o = rec + i * REC_LEN;
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
    // the reference's max / min (kernel.cu:32-38) are CUDA's double overloads, fmax / fmin: a NaN coordinate is dropped,
    // so a face with one keeps the box of its finite coordinates.  Finite inputs: the same bits as comparisons (the +-r
    // after them removes the sign of a zero)
    const double xlo = fmin(fmin(x0, x1), x2) - r, xhi = fmax(fmax(x0, x1), x2) + r;
    const double ylo = fmin(fmin(y0, y1), y2) - r, yhi = fmax(fmax(y0, y1), y2) + r;
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
                                                        unsigned long long* __restrict__ p2f_acc, Consts<double> K, float eps,
                                                        float bg0, float bg1, float bg2) {
    __shared__ __align__(16) double s_rec[CHUNK * REC_LEN];
    __shared__ uint32_t s_list[LIST_CAP];
    __shared__ int s_warp_cnt[NWARP];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z, S = K.S, F = K.F;
    const int px = blockIdx.x * TILE + (warp & 1) * 8 + (lane & 7);
    const int py = blockIdx.y * TILE + (warp >> 1) * 4 + (lane >> 3);  // image row (0 = top)
    const bool live = px < S && py < S;
    const double xp = pixel_coord<double>(px, S), yp = pixel_coord<double>(S - 1 - py, S);
    // tile extents in pixel-centre coordinates (monotone in the index, so the tile test is conservative)
    const double tx_first = pixel_coord<double>(blockIdx.x * TILE, S), tx_last = pixel_coord<double>(min((int)blockIdx.x * TILE + TILE - 1, S - 1), S);
    const double ty_top = pixel_coord<double>(S - 1 - blockIdx.y * TILE, S);
    const double ty_bot = pixel_coord<double>(S - 1 - min((int)blockIdx.y * TILE + TILE - 1, S - 1), S);

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
    const double* rec_img = rec_all + (size_t)b * F * REC_LEN;
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
                    const double2* src = reinterpret_cast<const double2*>(rec_img + (size_t)s_list[c * CHUNK + j] * REC_LEN) + q * 2;
                    double2* dst = reinterpret_cast<double2*>(s_rec + j * REC_LEN) + q * 2;
                    dst[0] = __ldg(src);
                    dst[1] = __ldg(src + 1);
                }
            }
            __syncthreads();
            double own_x = 0., own_y = 0., own_w = 0.;  // p2f partials of this warp: lane j owns stage face j
            for (int j = 0; j < cnt; ++j) {
                const double* rc = s_rec + j * REC_LEN;
                double a_x = 0., a_y = 0., a_w = 0.;
                bool contrib = false;
                // :355 bounding-box test
                if (live && !(xp > rc[R_BOX + 1] || xp < rc[R_BOX + 0] || yp > rc[R_BOX + 3] || yp < rc[R_BOX + 2])) {
                    Frag<double> fr;
                    if (fragment_any(rc, xp, yp, K, fr)) {
                        if (K.alpha == UMR_ALPHA_PROD) acc_a = acc_a * (1. - fr.D);  // :396
                        else if (K.alpha == UMR_ALPHA_SUM) acc_a += fr.D;           // :394
                        else if (fr.D > 0.5) acc_a = 1.;                            // :392
                        double k0 = fr.w0, k1 = fr.w1, k2 = fr.w2;
                        clip_bary(k0, k1, k2);
                        const double zp = depth_of(rc, k0, k1, k2);  // :403
                        if (!(zp < K.near_ || zp > K.far_)) {
                            const bool front = (flags_of(rc) & 8u) != 0;
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

}  // namespace f64
}  // namespace umr

#include "raster_host.cuh"

// =============================================================================================
// C ABI
// =============================================================================================
using namespace umr;
using namespace umr::f64;

extern "C" size_t umr_raster_workspace_bytes_f64(int32_t B, int32_t F, int32_t image_size, int32_t anti_aliasing) {
    (void)anti_aliasing;
    if (B <= 0 || F <= 0 || image_size <= 0) return 0;
    return f64::ws_layout(B, F).total;
}

extern "C" int umr_raster_forward_f64(const double* face_vertices, const double* textures, double* images,
                                      double* soft_colors, double* aggrs_info, double* p2f_info,
                                      const UmrRasterParams* p, void* workspace, void* stream_) {
    int rc = check_params<double>(p);
    if (rc) return rc;
    if (!face_vertices || !textures || !images || !aggrs_info || !workspace) return UMR_ERR_BAD_ARG;
    if (misaligned(workspace, 256)) return UMR_ERR_BAD_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    const int B = p->batch_size, F = p->num_faces;
    const Consts<double> K = make_consts<double>(p);
    if (!K.aa && soft_colors == nullptr) soft_colors = images;
    const f64::Layout L = f64::ws_layout(B, F);
    char* ws = (char*)workspace;
    double* rec = (double*)(ws + L.rec_off);
    double* box = (double*)(ws + L.box_off);
    unsigned long long* acc = (unsigned long long*)(ws + L.acc_off);
    const size_t n = (size_t)B * F;
    const bool sums = p->func_id_rgb == UMR_RGB_SOFTMAX && p2f_info;  // p2f accumulated and finalized
    launch(k_prep_f64, dim3((F + 255) / 256, B), 256, 0, stream, face_vertices, rec, box, F, sqrt(K.thr));  // r: kernel.cu:355
    if (p2f_info) {
        // hard mode never accumulates p2f (kernel.cu:417-431 is softmax-only) -> zeros
        cudaError_t e = sums ? cudaMemsetAsync(acc, 0, n * P2F_WORDS * sizeof(unsigned long long), stream)
                             : cudaMemsetAsync(p2f_info, 0, n * 2 * sizeof(double), stream);
        if (e != cudaSuccess) return (int)e;
    }
    record(p->ev_kernel_start, stream);
    launch(p->func_id_rgb == UMR_RGB_SOFTMAX ? k_raster_fwd_f64<1> : k_raster_fwd_f64<0>,
           dim3((K.S + TILE - 1) / TILE, (K.S + TILE - 1) / TILE, B), CTA, 0, stream, rec, box, textures, images, soft_colors,
           aggrs_info, sums ? acc : nullptr, K, p->eps, p->background_color[0], p->background_color[1], p->background_color[2]);
    record(p->ev_kernel_stop, stream);
    if (sums) launch(k_p2f_finalize_f64, (unsigned)((n + 255) / 256), 256, 0, stream, acc, p2f_info, n);
    return (int)cudaGetLastError();
}

extern "C" int umr_raster_backward_f64(const double* face_vertices, const double* textures, const double* soft_colors,
                                       const double* aggrs_info, const double* grad_images, double* grad_faces,
                                       double* grad_textures, const UmrRasterParams* p, void* workspace, void* stream_) {
    int rc = check_params<double>(p);
    if (rc) return rc;
    if (!face_vertices || !textures || !soft_colors || !aggrs_info || !grad_images || !workspace) return UMR_ERR_BAD_ARG;
    if (!grad_faces && !grad_textures) return UMR_ERR_BAD_ARG;
    if (misaligned(workspace, 256)) return UMR_ERR_BAD_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    const int B = p->batch_size, F = p->num_faces;
    const Consts<double> K = make_consts<double>(p);
    const f64::Layout L = f64::ws_layout(B, F);
    char* ws = (char*)workspace;
    double* rec = (double*)(ws + L.rec_off);
    double* box = (double*)(ws + L.box_off);
    const size_t n = (size_t)B * F;
    launch(k_prep_f64, dim3((F + 255) / 256, B), 256, 0, stream, face_vertices, rec, box, F, sqrt(K.thr));  // r: kernel.cu:355
    if (grad_textures) {
        cudaError_t e = cudaMemsetAsync(grad_textures, 0, (n / K.tex_div) * p->texture_size * 3 * sizeof(double), stream);
        if (e != cudaSuccess) return (int)e;
    }
    const bool softmax = p->func_id_rgb == UMR_RGB_SOFTMAX;
    record(p->ev_kernel_start, stream);
    launch(softmax ? (grad_textures ? k_raster_bwd_det<double, 1, true, 3, true> : k_raster_bwd_det<double, 1, false, 3, true>)
                   : (grad_textures ? k_raster_bwd_det<double, 0, true, 3, true> : k_raster_bwd_det<double, 0, false, 3, true>),
           gather_grid(K, B), CTA, 0, stream, rec, textures, soft_colors, aggrs_info, grad_images, grad_faces, grad_textures, K);
    record(p->ev_kernel_stop, stream);
    return (int)cudaGetLastError();
}
