// oracle/ref_host_shim.cpp -- TEST INFRASTRUCTURE ONLY (never imported by the product path).
//
// "Oracle A": the reference's OWN rasteriser device code, compiled for the host.
//
// The reference (NVlabs/UMR, external/SoftRas/soft_renderer/cuda/soft_rasterize_cuda_kernel.cu)
// ships no CPU path (functional/soft_rasterize.py:117-118, cuda/soft_rasterize_cuda.cpp:57-59).
// Its anonymous namespace (kernel.cu:22-659: helpers :24-218, prep kernel :222-282, forward
// :285-476, backward :479-656) is plain C++ apart from CUDA qualifiers.  oracle/build_oracle.py
// extracts that namespace verbatim from /root/reference into a temporary ref_device_code.inc
// (temp dir, generated, NEVER committed) and this file textually includes it behind a small
// qualifier shim, emulating the <<<ceil(n/512),512>>> launches of kernel.cu:688-697,704-732,768-797
// with an OpenMP loop over blocks.
//
// Build (done by oracle/build_oracle.py):
//   g++ -O2 -ffp-contract=off -fopenmp -std=c++17 -shared -fPIC ref_host_shim.cpp -I<tmp> -o _ref/libsoftras_ref_host.so
// -ffp-contract=off: no FMA contraction, so the float instantiation is a fixed IEEE op sequence.
//
// Known property inherited from the reference: backward_sample_texture (kernel.cu:199-218) returns
// an uninitialised value for non-matching texels; g++ resolves it like nvcc does (every texel of the
// face receives the gradient).  grad_textures for T2>1 must therefore be pinned on oracle B.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <omp.h>

#define __global__
#define __device__
#define __forceinline__ inline
#define __restrict__

namespace {
struct idx3 { int x, y, z; };
thread_local idx3 blockIdx{0, 0, 0};
thread_local idx3 threadIdx{0, 0, 0};
idx3 blockDim{512, 1, 1};
}  // namespace

using std::exp;
using std::pow;
using std::sqrt;

// CUDA's mixed float/double min/max overload set (used at kernel.cu:56-57, 143, 259, 584).
inline double max(float a, double b) { return (double)a > b ? (double)a : b; }
inline double max(double a, float b) { return a > (double)b ? a : (double)b; }
inline double min(float a, double b) { return (double)a < b ? (double)a : b; }
inline double min(double a, float b) { return a < (double)b ? a : (double)b; }
// CUDA's max / min(float, float) and (double, double) are fmaxf / fminf and fmax / fmin (crt/math_functions.hpp): a NaN
// operand is dropped, so kernel.cu:32-38 tests the box of a face's finite coordinates
inline float max(float a, float b) { return std::fmax(a, b); }
inline float min(float a, float b) { return std::fmin(a, b); }
inline double max(double a, double b) { return std::fmax(a, b); }
inline double min(double a, double b) { return std::fmin(a, b); }

template <class T>
inline T atomicAdd(T* p, T v) {
    T old;
#pragma omp atomic capture
    {
        old = *p;
        *p += v;
    }
    return old;
}

#include "ref_device_code.inc"  // generated from the reference; see header comment

namespace {
template <class K>
void launch512(long n, int nthreads, K body) {
    const int T = 512;
    const long nb = (n + T - 1) / T;
#pragma omp parallel for schedule(dynamic, 4) num_threads(nthreads)
    for (long b = 0; b < nb; ++b) {
        for (int t = 0; t < T; ++t) {
            blockIdx = {(int)b, 0, 0};
            threadIdx = {t, 0, 0};
            body();
        }
    }
}

template <class S>
int fwd(const S* faces, const S* textures, S* faces_info, S* aggrs_info, S* grid, S* p2f_info,
        S* p2f_sum, S* soft_colors, int B, int F, int IS, int T2, float near_, float far_,
        float eps, float sigma, int dist, float dist_eps, float gamma, int rgb, int alpha,
        int texmode, int double_side, int nthreads) {
    if (nthreads <= 0) nthreads = omp_get_max_threads();
    const int R = (int)std::sqrt((double)T2);  // kernel.cu:685 `int(sqrt(texture_size))`
    launch512((long)B * F, nthreads, [&] {
        forward_soft_rasterize_inv_cuda_kernel<S>(faces, faces_info, B, F, IS);
    });
    launch512((long)B * IS * IS, nthreads, [&] {
        forward_soft_rasterize_cuda_kernel<S>(faces, textures, faces_info, aggrs_info, grid,
                                              p2f_info, p2f_sum, soft_colors, B, F, IS, T2, R,
                                              near_, far_, eps, sigma, dist, dist_eps, gamma, rgb,
                                              alpha, texmode, double_side != 0);
    });
    return 0;
}

template <class S>
int bwd(const S* faces, const S* textures, const S* soft_colors, const S* faces_info,
        const S* aggrs_info, S* grad_faces, S* grad_textures, S* grad_soft_colors, int B, int F,
        int IS, int T2, float near_, float far_, float eps, float sigma, int dist, float dist_eps,
        float gamma, int rgb, int alpha, int texmode, int double_side, int nthreads) {
    if (nthreads <= 0) nthreads = omp_get_max_threads();
    const int R = (int)std::sqrt((double)T2);
    launch512((long)B * IS * IS, nthreads, [&] {
        backward_soft_rasterize_cuda_kernel<S>(faces, textures, soft_colors, faces_info,
                                               aggrs_info, grad_faces, grad_textures,
                                               grad_soft_colors, B, F, IS, T2, R, near_, far_, eps,
                                               sigma, dist, dist_eps, gamma, rgb, alpha, texmode,
                                               double_side != 0);
    });
    return 0;
}
}  // namespace

// C entry points mirror the pybind functions of cuda/soft_rasterize_cuda.cpp:62-138 (same argument
// order; tensors become host pointers + explicit B/F/T2).  All buffers are caller-allocated and
// pre-filled exactly as functional/soft_rasterize.py:47-55,94-95 does.
extern "C" {
int ref_forward_soft_rasterize_f32(const float* faces, const float* textures, float* faces_info,
                                   float* aggrs_info, float* grid, float* p2f_info, float* p2f_sum,
                                   float* soft_colors, int B, int F, int IS, int T2, float near_,
                                   float far_, float eps, float sigma, int dist, float dist_eps,
                                   float gamma, int rgb, int alpha, int texmode, int double_side,
                                   int nthreads) {
    return fwd<float>(faces, textures, faces_info, aggrs_info, grid, p2f_info, p2f_sum, soft_colors,
                      B, F, IS, T2, near_, far_, eps, sigma, dist, dist_eps, gamma, rgb, alpha,
                      texmode, double_side, nthreads);
}
int ref_backward_soft_rasterize_f32(const float* faces, const float* textures,
                                    const float* soft_colors, const float* faces_info,
                                    const float* aggrs_info, float* grad_faces,
                                    float* grad_textures, float* grad_soft_colors, int B, int F,
                                    int IS, int T2, float near_, float far_, float eps, float sigma,
                                    int dist, float dist_eps, float gamma, int rgb, int alpha,
                                    int texmode, int double_side, int nthreads) {
    return bwd<float>(faces, textures, soft_colors, faces_info, aggrs_info, grad_faces,
                      grad_textures, grad_soft_colors, B, F, IS, T2, near_, far_, eps, sigma, dist,
                      dist_eps, gamma, rgb, alpha, texmode, double_side, nthreads);
}
int ref_forward_soft_rasterize_f64(const double* faces, const double* textures, double* faces_info,
                                   double* aggrs_info, double* grid, double* p2f_info,
                                   double* p2f_sum, double* soft_colors, int B, int F, int IS,
                                   int T2, float near_, float far_, float eps, float sigma,
                                   int dist, float dist_eps, float gamma, int rgb, int alpha,
                                   int texmode, int double_side, int nthreads) {
    return fwd<double>(faces, textures, faces_info, aggrs_info, grid, p2f_info, p2f_sum,
                       soft_colors, B, F, IS, T2, near_, far_, eps, sigma, dist, dist_eps, gamma,
                       rgb, alpha, texmode, double_side, nthreads);
}
int ref_backward_soft_rasterize_f64(const double* faces, const double* textures,
                                    const double* soft_colors, const double* faces_info,
                                    const double* aggrs_info, double* grad_faces,
                                    double* grad_textures, double* grad_soft_colors, int B, int F,
                                    int IS, int T2, float near_, float far_, float eps,
                                    float sigma, int dist, float dist_eps, float gamma, int rgb,
                                    int alpha, int texmode, int double_side, int nthreads) {
    return bwd<double>(faces, textures, soft_colors, faces_info, aggrs_info, grad_faces,
                       grad_textures, grad_soft_colors, B, F, IS, T2, near_, far_, eps, sigma, dist,
                       dist_eps, gamma, rgb, alpha, texmode, double_side, nthreads);
}
int ref_host_max_threads(void) { return omp_get_max_threads(); }
}
