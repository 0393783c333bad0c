// oracle/softras_oracle.cpp -- TEST INFRASTRUCTURE ONLY (never imported by the product path).
//
// "Oracle B": an independent CPU restatement of the reference soft rasteriser
//   NVlabs/UMR  external/SoftRas/soft_renderer/cuda/soft_rasterize_cuda_kernel.cu  ("kernel.cu")
// written from the behavioural specification in SURVEY.md App. A, with the SAME IEEE operation
// order and float/double promotions as the reference's float instantiation, so that, compiled with
// -ffp-contract=off, every discrete decision (cull, region, near/far, running max, z-test) is
// bit-identical to the reference's own code compiled for the host (oracle A, ref_host_shim.cpp).
//
// Pinning: the reference has no tests or golden vectors for this path (SURVEY.md §4), so this
// restatement is pinned against OUTPUTS OF THE REFERENCE ITSELF RUN HERE (oracle A) by
// tests/test_oracle.py, and against tests/golden/*.npz generated from oracle A by
// tests/golden/make_golden.py.
//
// ONE deliberate difference (SURVEY.md App. B-1): kernel.cu:199-218 `backward_sample_texture`
// returns an uninitialised value for non-matching texels (undefined behaviour; both nvcc and g++
// resolve it as "every texel of the face gets the gradient").  Here only the sampled texel
// receives the gradient (the intended semantics, confirmed by finite differences).  `ub_texgrad=1`
// switches to the as-compiled behaviour so the restatement can be compared with oracle A.
//
// Layouts (all row-major fp32 unless templated on double):
//   faces[B,F,9] = (x0,y0,z0,x1,y1,z1,x2,y2,z2)   textures[B,F,T2,3]   faces_info[B,F,27]
//   soft_colors[B,4,S,S]   aggrs_info[B,2,S,S]   grid[S,S,2]   p2f_info/p2f_sum[B,F,2]
#include <cmath>
#include <cstdint>
#include <cstring>
#include <omp.h>
#include <vector>

namespace {

// mixed-precision select helpers: CUDA's max/min(float,double) return double (kernel.cu:56-57,143,259,584)
template <class S> inline double dmax(S a, double b) { return (double)a > b ? (double)a : b; }
template <class S> inline double dmin(S a, double b) { return (double)a < b ? (double)a : b; }
// CUDA's max / min(S, S) at kernel.cu:32-38: fmax / fmin, which drop a NaN operand (the box of the finite coordinates)
template <class S> inline S smax(S a, S b) { return std::fmax(a, b); }
template <class S> inline S smin(S a, S b) { return std::fmin(a, b); }

struct Params {
    int B, F, IS, T2, R;
    float near_, far_, eps, sigma, dist_eps, gamma;
    int dist, rgb, alpha, tex, double_side;
};

// kernel.cu:222-282  per-face preprocessing -> faces_info[27] = inv[9] | sym[9] | obt[3] | 0[6]
template <class S>
void prep_face(const S* face, S* info) {
    const S x0 = face[0], y0 = face[1], x1 = face[3], y1 = face[4], x2 = face[6], y2 = face[7];
    const S star[9] = {y1 - y2, x2 - x1, x1 * y2 - x2 * y1,   // kernel.cu:250-253
                       y2 - y0, x0 - x2, x2 * y0 - x0 * y2,
                       y0 - y1, x1 - x0, x0 * y1 - x1 * y0};
    S det = x2 * (y0 - y1) + x0 * (y1 - y2) + x1 * (y2 - y0);  // kernel.cu:254-258
    det = det > 0 ? (S)dmax(det, 1e-10) : (S)dmin(det, -1e-10);  // :259
    for (int k = 0; k < 9; ++k) info[k] = star[k] / det;
    for (int j = 0; j < 3; ++j)
        for (int k = 0; k < 3; ++k)  // Gram matrix + 1, kernel.cu:265-271
            info[9 + 3 * j + k] = face[3 * j] * face[3 * k] + face[3 * j + 1] * face[3 * k + 1] + 1;
    const S px[3] = {x0, x1, x2}, py[3] = {y0, y1, y2};
    for (int k = 0; k < 3; ++k) {  // first obtuse corner only, kernel.cu:273-281
        const int a = (k + 1) % 3, b = (k + 2) % 3;
        if ((px[a] - px[k]) * (px[b] - px[k]) + (py[a] - py[k]) * (py[b] - py[k]) < 0) {
            info[18 + k] = 1;
            break;
        }
    }
}

template <class S>
inline bool outside_bbox(S x, S y, const S* f, S r) {  // kernel.cu:32-38
    return x > smax(smax(f[0], f[3]), f[6]) + r || x < smin(smin(f[0], f[3]), f[6]) - r ||
           y > smax(smax(f[1], f[4]), f[7]) + r || y < smin(smin(f[1], f[4]), f[7]) - r;
}
template <class S>
inline bool frontside(const S* f) {  // kernel.cu:42-44
    return (f[7] - f[1]) * (f[3] - f[0]) < (f[4] - f[1]) * (f[6] - f[0]);
}
template <class S>
inline bool inside_closed(const S* w) {  // kernel.cu:48-50
    return w[0] <= 1 && w[0] >= 0 && w[1] <= 1 && w[1] >= 0 && w[2] <= 1 && w[2] >= 0;
}
inline double dmax(double a, double b) { return a > b ? a : b; }
template <class S>
inline void clip_bary(S* w) {  // kernel.cu:54-59: max(min(w, 1 - 1e-5), 1e-5) evaluated in double, stored as S
    for (int k = 0; k < 3; ++k) w[k] = (S)dmax(dmin(w[k], 1 - 1e-5), 1e-5);
    const S s = (S)dmax((S)(w[0] + w[1] + w[2]), 1e-5);
    for (int k = 0; k < 3; ++k) w[k] /= s;
}

// kernel.cu:62-152  euclidean pixel-to-triangle distance.  Outputs sign, (dx,dy), t[3] (= closest-
// point barycentrics minus w).
template <class S>
inline void euclid(S& sign, S& dx, S& dy, const S* w, S* t, const S* f, const S* info, S xp, S yp) {
    const S* sym = info + 9;
    const S* obt = info + 18;
    if (w[0] > 0 && w[1] > 0 && w[2] > 0 && w[0] < 1 && w[1] < 1 && w[2] < 1) {
        S best = 100000000, bx = 0, by = 0;
        S t0[3];
        for (int k = 0; k < 3; ++k) {
            const int v0 = k, v1 = (k + 1) % 3, v2 = (k + 2) % 3;
            const S a0 = sym[3 * v0 + 0] - sym[3 * v1 + 0];
            const S a1 = sym[3 * v0 + 1] - sym[3 * v1 + 1];
            const S a2 = sym[3 * v0 + 2] - sym[3 * v1 + 2];
            const S a[3] = {a0, a1, a2};
            // NOTE: t0 persists across k (kernel.cu:79 declares it outside the loop body's
            // assignments); every entry is rewritten each iteration so there is no carry-over.
            t0[v0] = (w[0] * a0 + w[1] * a1 + w[2] * a2 - a[v1]) / (a[v0] - a[v1]);
            t0[v1] = 1 - t0[v0];
            t0[v2] = 0;
            t0[0] -= w[0];
            t0[1] -= w[1];
            t0[2] -= w[2];
            dx = t0[0] * f[0] + t0[1] * f[3] + t0[2] * f[6];
            dy = t0[0] * f[1] + t0[1] * f[4] + t0[2] * f[7];
            const S d = dx * dx + dy * dy;
            if (d < best) {
                best = d; bx = dx; by = dy;
                t[0] = t0[0]; t[1] = t0[1]; t[2] = t0[2];
            }
        }
        dx = bx; dy = by; sign = 1;
    } else {
        int v0 = -1;
        if (w[1] <= 0 && w[2] <= 0) {
            v0 = 0;
            if (obt[0] == 1 && (xp - f[0]) * (f[6] - f[0]) + (yp - f[1]) * (f[7] - f[1]) > 0) v0 = 2;
        } else if (w[2] <= 0 && w[0] <= 0) {
            v0 = 1;
            if (obt[1] == 1 && (xp - f[3]) * (f[0] - f[3]) + (yp - f[4]) * (f[1] - f[4]) > 0) v0 = 0;
        } else if (w[0] <= 0 && w[1] <= 0) {
            v0 = 2;
            if (obt[2] == 1 && (xp - f[6]) * (f[3] - f[6]) + (yp - f[7]) * (f[4] - f[7]) > 0) v0 = 1;
        } else if (w[0] <= 0) v0 = 1;
        else if (w[1] <= 0) v0 = 2;
        else if (w[2] <= 0) v0 = 0;
        if (v0 < 0) {
            // Reached only when every w_k > 0 but some w_k >= 1 (rounding).  The reference then runs
            // with v0 = -1 (kernel.cu:128-139): it writes t[-1] and reads a0[-1] -- undefined
            // behaviour that cannot be restated.  DEFINED HERE (and in the CUDA kernel) as: start from
            // the corner with the largest barycentric.  tests/test_oracle.py counts how often oracle A
            // and B disagree because of it (never, on the committed scenes).
            v0 = w[0] >= w[1] ? (w[0] >= w[2] ? 0 : 2) : (w[1] >= w[2] ? 1 : 2);
        }
        const int v1 = (v0 + 1) % 3, v2 = (v0 + 2) % 3;
        S a[3];
        a[0] = sym[3 * v0 + 0] - sym[3 * v1 + 0];
        a[1] = sym[3 * v0 + 1] - sym[3 * v1 + 1];
        a[2] = sym[3 * v0 + 2] - sym[3 * v1 + 2];
        S tp[3];
        tp[v0] = (w[0] * a[0] + w[1] * a[1] + w[2] * a[2] - a[v1]) / (a[v0] - a[v1]);
        tp[v1] = 1 - tp[v0];
        tp[v2] = 0;
        for (int k = 0; k < 3; ++k) {  // kernel.cu:142-145
            tp[k] = (S)dmin((S)dmax(tp[k], 0.), 1.);  // min(max(t, 0.), 1.) in double
            tp[k] -= w[k];
            t[k] = tp[k];
        }
        dx = t[0] * f[0] + t[1] * f[3] + t[2] * f[6];
        dy = t[0] * f[1] + t[1] * f[4] + t[2] * f[7];
        sign = -1;
    }
}

template <class S>
inline int texel_index(const S* w, int R) {  // kernel.cu:180-190 (surface sampling)
    const int wx = (int)(w[0] * R);
    const int wy = (int)(w[1] * R);
    if ((w[0] + w[1]) * R - wx - wy <= 1) return wy * R + wx;
    return (R - 1 - wy) * R + (R - 1 - wx);
}
template <class S>
inline S sample_tex(const S* tex, const S* w, int R, int k, int mode) {  // kernel.cu:179-195
    if (mode == 0) return tex[texel_index(w, R) * 3 + k];
    return w[0] * tex[k] + w[1] * tex[3 + k] + w[2] * tex[6 + k];
}

template <class S>
inline void pixel_xy(int pn, int IS, S& xp, S& yp) {  // kernel.cu:323-326
    const int yi = IS - 1 - (pn / IS);
    const int xi = pn % IS;
    yp = (S)((2. * yi + 1. - IS) / IS);
    xp = (S)((2. * xi + 1. - IS) / IS);
}

// Distance/probability stage shared by forward and backward (kernel.cu:355-384 / 536-563).
// Returns false when the pair is culled.
template <class S>
inline bool fragment(const Params& P, const S* f, const S* info, S xp, S yp, S thr, S r, S* w, S* t,
                     S& sign, S& dx, S& dy, S& dis, S& D) {
    if (outside_bbox(xp, yp, f, r)) return false;
    w[0] = info[0] * xp + info[1] * yp + info[2];  // kernel.cu:25-29
    w[1] = info[3] * xp + info[4] * yp + info[5];
    w[2] = info[6] * xp + info[7] * yp + info[8];
    sign = 0; dx = dy = 0; dis = 0;
    if (P.dist == 0) {
        D = inside_closed(w) ? (S)1. : (S)0.;
        if (D == 0.) return false;
    } else if (P.dist == 1) {  // kernel.cu:156-159
        S m = w[0] > w[1] ? (w[1] > w[2] ? w[2] : w[1]) : (w[0] > w[2] ? w[2] : w[0]);
        dis = m > 0 ? m * m : -(m * m);
        t[0] = w[0]; t[1] = w[1]; t[2] = w[2];
        if (-dis >= thr) return false;
        D = (S)(1. / (1. + (double)std::exp(-dis / (S)P.sigma)));
    } else {
        euclid(sign, dx, dy, w, t, f, info, xp, yp);
        dis = dx * dx + dy * dy;
        if (sign < 0 && dis >= thr) return false;
        D = (S)(1. / (1. + (double)std::exp(-sign * dis / (S)P.sigma)));
    }
    return true;
}

template <class S>
void forward(const Params& P, const S* faces, const S* textures, S* faces_info, S* aggrs, const S* grid,
             S* p2f, S* p2f_sum, S* colors, int nthreads) {
    const int B = P.B, F = P.F, IS = P.IS, T2 = P.T2, NP = IS * IS;
#pragma omp parallel for num_threads(nthreads)
    for (long i = 0; i < (long)B * F; ++i) prep_face(faces + i * 9, faces_info + i * 27);

    const S thr = (S)(P.dist_eps * P.sigma);  // kernel.cu:333: float*float, then scalar_t
    const S r = std::sqrt(thr);
#pragma omp parallel for schedule(dynamic, 64) num_threads(nthreads)
    for (long i = 0; i < (long)B * NP; ++i) {
        const int b = (int)(i / NP), pn = (int)(i % NP);
        S xp, yp;
        pixel_xy(pn, IS, xp, yp);
        S c[4] = {1., 1., 1., 0.};
        if (P.alpha == 2) c[3] = 1.;
        S ssum = (S)std::exp(P.eps / P.gamma);  // kernel.cu:337: expf(float/float)
        S smaxv = (S)P.eps;
        for (int k = 0; k < 3; ++k) {
            const S bg = colors[((long)b * 4 + k) * NP + pn];
            c[k] = P.rgb == 0 ? bg : bg * ssum;
        }
        S zmin = 10000000;
        int fid = -1;
        for (int fn = 0; fn < F; ++fn) {
            const S* f = faces + ((long)b * F + fn) * 9;
            const S* info = faces_info + ((long)b * F + fn) * 27;
            const S* tex = textures + ((long)b * F + fn) * T2 * 3;
            S w[3], t[3], sign, dx, dy, dis, D;
            if (!fragment(P, f, info, xp, yp, thr, r, w, t, sign, dx, dy, dis, D)) continue;
            if (P.alpha == 0) { if (D > 0.5) c[3] = 1.; }
            else if (P.alpha == 1) c[3] += D;
            else c[3] = (S)((double)c[3] * (1. - (double)D));  // kernel.cu:396
            S wc[3] = {w[0], w[1], w[2]};
            clip_bary(wc);
            const S zp = (S)(1. / (double)(wc[0] / f[2] + wc[1] / f[5] + wc[2] / f[8]));  // :403
            if (zp < (S)P.near_ || zp > (S)P.far_) continue;
            if (P.rgb == 0) {
                if (zp < zmin && inside_closed(w) && (P.double_side || frontside(f))) {
                    zmin = zp; fid = fn;
                    for (int k = 0; k < 3; ++k) c[k] = sample_tex(tex, wc, P.R, k, P.tex);
                }
            } else if (frontside(f) || P.double_side) {
                const S zn = ((S)P.far_ - zp) / ((S)P.far_ - (S)P.near_);
                S ed = 1.;
                if (zn > smaxv) { ed = std::exp((smaxv - zn) / (S)P.gamma); smaxv = zn; }
                const S ez = std::exp((zn - smaxv) / (S)P.gamma);
                ssum = ed * ssum + ez * D;
                const long q = ((long)b * F + fn) * 2;
                const S a0 = ez * D * grid[pn * 2 + 0], a1 = ez * D * grid[pn * 2 + 1], a2 = ez * D;
#pragma omp atomic
                p2f[q + 0] += a0;
#pragma omp atomic
                p2f[q + 1] += a1;
#pragma omp atomic
                p2f_sum[q + 0] += a2;
#pragma omp atomic
                p2f_sum[q + 1] += a2;
                for (int k = 0; k < 3; ++k) c[k] = ed * c[k] + ez * D * sample_tex(tex, wc, P.R, k, P.tex);
            }
        }
        S* ca = colors + ((long)b * 4 + 3) * NP + pn;
        if (P.alpha == 0) *ca = c[3];
        else if (P.alpha == 1) *ca = c[3] / F;
        else *ca = (S)(1. - (double)c[3]);
        if (P.rgb == 0) {
            if (fid != -1) for (int k = 0; k < 3; ++k) colors[((long)b * 4 + k) * NP + pn] = c[k];
            aggrs[((long)b * 2 + 0) * NP + pn] = zmin;
            aggrs[((long)b * 2 + 1) * NP + pn] = (S)fid;
        } else {
            for (int k = 0; k < 3; ++k) colors[((long)b * 4 + k) * NP + pn] = c[k] / ssum;
            aggrs[((long)b * 2 + 0) * NP + pn] = ssum;
            aggrs[((long)b * 2 + 1) * NP + pn] = smaxv;
        }
    }
}

template <class S>
void backward(const Params& P, const S* faces, const S* textures, const S* colors, const S* faces_info,
              const S* aggrs, S* gfaces, S* gtex, const S* gcolors, int ub_texgrad, int nthreads) {
    const int B = P.B, F = P.F, IS = P.IS, T2 = P.T2, NP = IS * IS;
    const S thr = (S)(P.dist_eps * P.sigma);
    const S r = std::sqrt(thr);
#pragma omp parallel for schedule(dynamic, 64) num_threads(nthreads)
    for (long i = 0; i < (long)B * NP; ++i) {
        const int b = (int)(i / NP), pn = (int)(i % NP);
        S xp, yp;
        pixel_xy(pn, IS, xp, yp);
        const S ssum = aggrs[((long)b * 2 + 0) * NP + pn];
        const S smaxv = aggrs[((long)b * 2 + 1) * NP + pn];
        const S g[4] = {gcolors[((long)b * 4 + 0) * NP + pn], gcolors[((long)b * 4 + 1) * NP + pn],
                        gcolors[((long)b * 4 + 2) * NP + pn], gcolors[((long)b * 4 + 3) * NP + pn]};
        const S C[4] = {colors[((long)b * 4 + 0) * NP + pn], colors[((long)b * 4 + 1) * NP + pn],
                        colors[((long)b * 4 + 2) * NP + pn], colors[((long)b * 4 + 3) * NP + pn]};
        for (int fn = 0; fn < F; ++fn) {
            const S* f = faces + ((long)b * F + fn) * 9;
            const S* info = faces_info + ((long)b * F + fn) * 27;
            const S* tex = textures + ((long)b * F + fn) * T2 * 3;
            S w[3], t[3], sign, dx, dy, dis, D;
            if (!fragment(P, f, info, xp, yp, thr, r, w, t, sign, dx, dy, dis, D)) continue;
            S* gf = gfaces + ((long)b * F + fn) * 9;
            S* gt = gtex + ((long)b * F + fn) * T2 * 3;
            S gv[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
            S Cxy = 0;
            S Ca = g[3];  // kernel.cu:577-585
            if (P.alpha == 1) Ca /= F;
            else if (P.alpha == 2) Ca = (S)((double)Ca * ((double)(1 - C[3]) / dmax((S)(1 - D), 1e-6)));
            Cxy += Ca;
            const S w0[3] = {w[0], w[1], w[2]};
            clip_bary(w);
            const S zp = (S)(1. / (double)(w[0] / f[2] + w[1] / f[5] + w[2] / f[8]));
            if (zp < (S)P.near_ || zp > (S)P.far_) continue;  // drops the alpha gradient too (:592)
            if (P.rgb == 0) {
                if ((S)fn == smaxv) {  // aggrs[1] holds the winning face id as a float (:596)
                    for (int k = 0; k < 3; ++k) {
                        if (P.tex == 0) {
                            const int hit = texel_index(w, P.R);
                            for (int j = 0; j < T2; ++j)
                                if (ub_texgrad || j == hit) {
#pragma omp atomic
                                    gt[3 * j + k] += g[k];
                                }
                        } else {
                            // reference loops j over texture_size (=3 corner colours) with w[j]*grad
                            for (int j = 0; j < T2; ++j) {
#pragma omp atomic
                                gt[3 * j + k] += w[j] * g[k];
                            }
                        }
                    }
                }
            } else if (P.rgb == 1 && (frontside(f) || P.double_side)) {
                S Crgb = 0.;
                const S zn = ((S)P.far_ - zp) / ((S)P.far_ - (S)P.near_);
                const S s = D * std::exp((zn - smaxv) / (S)P.gamma) / ssum;  // :608
                for (int k = 0; k < 3; ++k) {
                    if (P.tex == 0) {
                        const int hit = texel_index(w, P.R);
                        for (int j = 0; j < T2; ++j)
                            if (ub_texgrad || j == hit) {
                                const S add = s * g[k];
#pragma omp atomic
                                gt[3 * j + k] += add;
                            }
                    } else {
                        for (int j = 0; j < T2; ++j) {
                            const S add = s * (w[j] * g[k]);
#pragma omp atomic
                            gt[3 * j + k] += add;
                        }
                    }
                    const S ck = sample_tex(tex, w, P.R, k, P.tex);
                    Crgb += g[k] * (ck - C[k]);
                }
                Crgb *= s;
                Cxy += Crgb / D;
                const S Cz = Crgb / (S)P.gamma / ((S)P.near_ - (S)P.far_) * zp * zp;  // :624
                gv[0][2] = Cz * w[0] / f[2] / f[2];
                gv[1][2] = Cz * w[1] / f[5] / f[5];
                gv[2][2] = Cz * w[2] / f[8] / f[8];
            }
            Cxy *= D * (1 - D) / (S)P.sigma;  // :632
            if (P.dist == 1) {  // kernel.cu:162-176 with w := t (unclipped w copy), :634-635
                const int p = t[0] > t[1] ? (t[1] > t[2] ? 2 : 1) : (t[0] > t[2] ? 2 : 0);
                for (int l = 0; l < 2; ++l)
                    for (int k = 0; k < 3; ++k) {
                        S gkl = 0;
                        for (int q = 0; q < 3; ++q)
                            gkl += -info[3 * p + l] * info[3 * k + q] * (q == 0 ? xp : (q == 1 ? yp : (S)1));
                        gv[k][l] = gkl * Cxy;
                        gv[k][l] = (S)((double)gv[k][l] *
                                       (dis > 0 ? (2. * (double)std::sqrt(dis)) : (2. * (double)std::sqrt(-dis))));
                    }
            } else if (P.dist == 2) {  // :637-642
                for (int k = 0; k < 3; ++k)
                    for (int l = 0; l < 2; ++l) gv[k][l] = 2 * sign * Cxy * (t[k] + w0[k]) * (l == 0 ? dx : dy);
            }
            for (int k = 0; k < 3; ++k)
                for (int l = 0; l < 3; ++l) {
#pragma omp atomic
                    gf[3 * k + l] += gv[k][l];
                }
        }
    }
}

Params mk(int B, int F, int IS, int T2, float near_, float far_, float eps, float sigma, int dist,
          float dist_eps, float gamma, int rgb, int alpha, int tex, int double_side) {
    Params P;
    P.B = B; P.F = F; P.IS = IS; P.T2 = T2; P.R = (int)std::sqrt((double)T2);
    P.near_ = near_; P.far_ = far_; P.eps = eps; P.sigma = sigma; P.dist_eps = dist_eps; P.gamma = gamma;
    P.dist = dist; P.rgb = rgb; P.alpha = alpha; P.tex = tex; P.double_side = double_side;
    return P;
}
}  // namespace

// Same argument order as the reference binding cuda/soft_rasterize_cuda.cpp:62-138.
extern "C" {
int oracle_forward_soft_rasterize_f32(const float* faces, const float* textures, float* faces_info,
                                      float* aggrs_info, const float* grid, float* p2f_info, float* p2f_sum,
                                      float* soft_colors, int B, int F, int IS, int T2, float near_, float far_,
                                      float eps, float sigma, int dist, float dist_eps, float gamma, int rgb,
                                      int alpha, int texmode, int double_side, int nthreads) {
    if (nthreads <= 0) nthreads = omp_get_max_threads();
    forward<float>(mk(B, F, IS, T2, near_, far_, eps, sigma, dist, dist_eps, gamma, rgb, alpha, texmode, double_side),
                   faces, textures, faces_info, aggrs_info, grid, p2f_info, p2f_sum, soft_colors, nthreads);
    return 0;
}
int oracle_backward_soft_rasterize_f32(const float* faces, const float* textures, const float* soft_colors,
                                       const float* faces_info, const float* aggrs_info, float* grad_faces,
                                       float* grad_textures, const float* grad_soft_colors, int B, int F, int IS,
                                       int T2, float near_, float far_, float eps, float sigma, int dist,
                                       float dist_eps, float gamma, int rgb, int alpha, int texmode,
                                       int double_side, int ub_texgrad, int nthreads) {
    if (nthreads <= 0) nthreads = omp_get_max_threads();
    backward<float>(mk(B, F, IS, T2, near_, far_, eps, sigma, dist, dist_eps, gamma, rgb, alpha, texmode, double_side),
                    faces, textures, soft_colors, faces_info, aggrs_info, grad_faces, grad_textures,
                    grad_soft_colors, ub_texgrad, nthreads);
    return 0;
}
int oracle_forward_soft_rasterize_f64(const double* faces, const double* textures, double* faces_info,
                                      double* aggrs_info, const double* grid, double* p2f_info, double* p2f_sum,
                                      double* soft_colors, int B, int F, int IS, int T2, float near_, float far_,
                                      float eps, float sigma, int dist, float dist_eps, float gamma, int rgb,
                                      int alpha, int texmode, int double_side, int nthreads) {
    if (nthreads <= 0) nthreads = omp_get_max_threads();
    forward<double>(mk(B, F, IS, T2, near_, far_, eps, sigma, dist, dist_eps, gamma, rgb, alpha, texmode, double_side),
                    faces, textures, faces_info, aggrs_info, grid, p2f_info, p2f_sum, soft_colors, nthreads);
    return 0;
}
int oracle_backward_soft_rasterize_f64(const double* faces, const double* textures, const double* soft_colors,
                                       const double* faces_info, const double* aggrs_info, double* grad_faces,
                                       double* grad_textures, const double* grad_soft_colors, int B, int F, int IS,
                                       int T2, float near_, float far_, float eps, float sigma, int dist,
                                       float dist_eps, float gamma, int rgb, int alpha, int texmode,
                                       int double_side, int ub_texgrad, int nthreads) {
    if (nthreads <= 0) nthreads = omp_get_max_threads();
    backward<double>(mk(B, F, IS, T2, near_, far_, eps, sigma, dist, dist_eps, gamma, rgb, alpha, texmode, double_side),
                     faces, textures, soft_colors, faces_info, aggrs_info, grad_faces, grad_textures,
                     grad_soft_colors, ub_texgrad, nthreads);
    return 0;
}
int oracle_max_threads(void) { return omp_get_max_threads(); }
}
