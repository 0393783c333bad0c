// raster_host.cuh -- host side shared by the rasteriser's C entry points (raster.cu, raster_f64.cu): the parameter checks
// and the kernel constants.  Kernels are launched through launch() (common.cuh).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <type_traits>

#include "common.cuh"
#include "raster_generic.cuh"
#include "umr_b200.h"

namespace umr {

// one of the profiling events of UmrRasterParams (NULL: off)
inline void record(void* event, cudaStream_t stream) {
    if (event) cudaEventRecord((cudaEvent_t)event, stream);
}

inline bool misaligned(const void* ptr, uintptr_t alignment) { return ((uintptr_t)ptr & (alignment - 1)) != 0; }

// raster side S: the image side, doubled by anti-aliasing
inline int64_t raster_side(const UmrRasterParams* p) { return (int64_t)p->image_size * (p->anti_aliasing ? 2 : 1); }

// Raster sides past the launch limit of the 16x16-tile grid (gridDim.y <= 65535) are refused by the entry points whose
// backward is the face-parallel gather (deterministic float32, float64); the bounds of their fixed-point p2f sums hold
// below it.
constexpr int64_t GATHER_MAX_RASTER = 65535 * TILE;

// the UMR configuration has specialised kernels; every other mode combination takes the generic ones
inline bool is_generic(const UmrRasterParams* p) {
    return p->func_id_dist != UMR_DIST_EUCLIDEAN || p->func_id_alpha != UMR_ALPHA_PROD ||
           p->texture_sample_type != UMR_TEX_SURFACE;
}

// The checks every raster entry point starts with, for float (T = float) or double buffers.  Double buffers take 3 colour
// channels only and have their raster-side limit checked right after the other size limits; float buffers take 3, or 4 in
// UMR's softmax configuration, and their deterministic entry points check the limit after all of these.
template <typename T>
int check_params(const UmrRasterParams* p) {
    constexpr bool F64 = std::is_same_v<T, double>;
    if (!p) return UMR_ERR_BAD_ARG;
    if (p->batch_size <= 0 || p->num_faces <= 0 || p->texture_size <= 0 || p->image_size <= 0) return UMR_ERR_BAD_ARG;
    if (p->num_faces > UMR_RASTER_MAX_FACES || p->batch_size > 65535) return UMR_ERR_TOO_LARGE;
    if (F64 && raster_side(p) > GATHER_MAX_RASTER) return UMR_ERR_TOO_LARGE;
    if (p->func_id_dist < 0 || p->func_id_dist > 2 || p->func_id_alpha < 0 || p->func_id_alpha > 2 ||
        p->texture_sample_type < 0 || p->texture_sample_type > 1)
        return UMR_ERR_UNSUPPORTED;
    if (p->texture_sample_type == UMR_TEX_VERTEX && p->texture_size != 3) return UMR_ERR_BAD_ARG;  // [B,F,3,3]
    if (p->shared_textures > 1 && p->batch_size % p->shared_textures != 0) return UMR_ERR_BAD_ARG;
    if (p->func_id_rgb != UMR_RGB_HARD && p->func_id_rgb != UMR_RGB_SOFTMAX) return UMR_ERR_UNSUPPORTED;
    if (p->color_channels != 0 && p->color_channels != 3 && (F64 || p->color_channels != 4)) return UMR_ERR_BAD_ARG;
    // 4 colour channels (the part-map render): UMR's own configuration only
    if (p->color_channels == 4 && (is_generic(p) || p->func_id_rgb != UMR_RGB_SOFTMAX)) return UMR_ERR_UNSUPPORTED;
    return UMR_OK;
}

template <typename T>
Consts<T> make_consts(const UmrRasterParams* p) {
    Consts<T> K = {};
    K.thr = p->dist_eps * p->sigma_val;  // kernel.cu:333 (float * float)
    K.sigma = p->sigma_val;
    K.gamma = p->gamma_val;
    K.near_ = p->near_plane;
    K.far_ = p->far_plane;
    if constexpr (std::is_same_v<T, float>) {  // the float streamed backward's reciprocals
        K.r_sigma = (float)(1.0 / (double)p->sigma_val);
        K.r_gamma = (float)(1.0 / (double)p->gamma_val);
        K.r_fn = (float)(1.0 / ((double)p->far_plane - (double)p->near_plane));
        K.r_nf = (float)(1.0 / ((double)p->near_plane - (double)p->far_plane));
    }
    K.F = p->num_faces;
    K.T2 = p->texture_size;
    K.R = (int)sqrt((double)p->texture_size);  // kernel.cu:685
    K.IS = p->image_size;
    K.aa = p->anti_aliasing ? 1 : 0;
    K.S = p->image_size * (K.aa ? 2 : 1);
    K.double_side = p->double_side ? 1 : 0;
    K.dist = p->func_id_dist;
    K.alpha = p->func_id_alpha;
    K.tex = p->texture_sample_type;
    K.tex_bs = (size_t)p->num_faces * p->texture_size * (p->color_channels == 4 ? 4 : 3);
    K.tex_div = p->shared_textures > 1 ? p->shared_textures : 1;
    return K;
}

// grid of the face-parallel gather backward k_raster_bwd_det: one warp per (texture group, face)
template <typename T>
dim3 gather_grid(const Consts<T>& K, int B) {
    return dim3((unsigned)((K.F + NWARP - 1) / NWARP), (unsigned)(B / K.tex_div));
}

}  // namespace umr
