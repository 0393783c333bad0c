// losses.cu -- geometric-loss kernels around the rasteriser (sm_90a): bilinear texture-flow
// sampler, silhouette IoU, O(N*M) chamfer, texture-cycle.  All HBM/L2-bound gather/reduce work; no
// tensor cores (none of these is a dense contraction -- chamfer's inner dimension is 2 or 3).
//
// Reference entry points replaced (file:line under the reference tree):
//   nnutils/geom_utils.py:41-59 `sample_textures`, nnutils/loss_utils.py:59-64 (texture_dt_loss)
//   nnutils/loss_utils.py:41-48 `neg_iou_loss`
//   nnutils/chamfer_python.py:43-64 `distChamfer`
//   nnutils/loss_utils.py:152-182 `TexCycle.forward`
//
// The kernels are written once on the scalar type in losses.cuh; this unit instantiates them for float, with FMA
// contraction, and holds the float32 entry points.  The kernels used only by float32 (the atomic chamfer backward, the
// non-deterministic IoU finalize, the face-visibility bitmap that float64 shares) are here.  The reductions and the
// chamfer backward also have deterministic variants (DET template parameter / gather kernels, `*_deterministic` entry
// points at the end of this file; DESIGN.md §2): no atomics reach their outputs.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <climits>

#include "common.cuh"
#include "losses.cuh"
#include "umr_b200.h"

namespace umr {

__global__ void k_iou_finalize(const float* __restrict__ inter, float* __restrict__ uni, float* __restrict__ loss, int B) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float u = uni[b] + 1e-6f;
    uni[b] = u;
    loss[b] = 1.f - inter[b] / u;
}

template <int D>
__global__ void __launch_bounds__(256) k_chamfer_bwd(const float* __restrict__ q, const float* __restrict__ k,
                                                     const int32_t* __restrict__ idx, const float* __restrict__ gd,
                                                     float* __restrict__ gq, float* __restrict__ gk, int NQ, int NK) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (i >= NQ) return;
    const float g = __ldg(gd + (size_t)b * NQ + i);
    const int j = __ldg(idx + (size_t)b * NQ + i);
#pragma unroll
    for (int d = 0; d < D; ++d) {
        const float diff = __ldg(q + ((size_t)b * NQ + i) * D + d) - __ldg(k + ((size_t)b * NK + j) * D + d);
        atomicAdd(gq + ((size_t)b * NQ + i) * D + d, 2.f * g * diff);
        atomicAdd(gk + ((size_t)b * NK + j) * D + d, -2.f * g * diff);
    }
}

// Visibility bitmap of the face-id plane (replaces the per-sample torch.unique + host sync of loss_utils.py:174-179).
// Almost every pixel carries the background id or the id of its neighbour: a thread only touches the bitmap when the id
// differs from the previous pixel it saw AND the byte is not set yet (test-before-set through L2), so the plane is
// streamed at HBM speed instead of serialising millions of stores on a handful of bytes.
__global__ void __launch_bounds__(256) k_visible(const float* __restrict__ ids, uint8_t* __restrict__ vis, int F, int64_t P) {
    const int b = blockIdx.y;
    const float* src = ids + (size_t)b * P;
    uint8_t* v = vis + (size_t)b * F;
    int last = INT_MIN;
    auto mark = [&](float id) {
        int f = (int)id;
        if (f == last) return;
        last = f;
        if (f < 0) f += F;  // python negative index: -1 (background) marks the LAST face (loss_utils.py:175-177)
        if (f >= 0 && f < F && __ldcg(v + f) == 0) v[f] = 1;
    };
    const bool vec = ((P & 3) == 0) && ((((uintptr_t)src) & 15) == 0);
    if (vec) {
        const int64_t n4 = P >> 2;
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(src) + i);
            mark(q.x); mark(q.y); mark(q.z); mark(q.w);
        }
    } else {
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < P; i += (int64_t)gridDim.x * blockDim.x)
            mark(__ldg(src + i));
    }
}

}  // namespace umr

using namespace umr;

extern "C" int umr_bilinear_sample_forward(const float* image, const float* flow, float* out, int32_t B,
                                           int32_t C, int32_t H, int32_t W, int32_t N, void* stream_) {
    return sample_forward(image, flow, out, B, C, H, W, N, stream_);
}

extern "C" int umr_bilinear_sample_backward(const float* image, const float* flow, const float* grad_out,
                                            float* grad_flow, float* grad_image, int32_t B, int32_t C,
                                            int32_t H, int32_t W, int32_t N, void* stream_) {
    if (!image || !flow || !grad_out || !grad_flow || B <= 0 || C <= 0 || H <= 0 || W <= 0 || N <= 0 ||
        vec2_misaligned(flow) || vec2_misaligned(grad_flow))
        return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (C > 4) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    if (grad_image) {
        cudaError_t e = cudaMemsetAsync(grad_image, 0, (size_t)B * C * H * W * sizeof(float), st);
        if (e != cudaSuccess) return (int)e;
    }
    with_channels(C, [&](auto c) {
        launch(k_sample_bwd<float, c>, dim3((N + 255) / 256, B), 256, 0, st, image, reinterpret_cast<const float2*>(flow),
               grad_out, reinterpret_cast<float2*>(grad_flow), grad_image, H, W, N);
    });
    return (int)cudaGetLastError();
}

extern "C" int umr_iou_forward(const float* predict, int64_t predict_bstride, const float* target, float* inter,
                               float* uni, float* loss, int32_t B, int64_t N, void* stream_) {
    if (!predict || !target || !inter || !uni || !loss || B <= 0 || N <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(inter, 0, (size_t)B * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    e = cudaMemsetAsync(uni, 0, (size_t)B * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    const dim3 grid(iou_slots<float>(N), B);
    launch(k_iou_partial<float, false>, grid, IOU_THREADS<float>, 0, st, predict, target, inter, uni, N, predict_bstride);
    launch(k_iou_finalize, (B + 127) / 128, 128, 0, st, inter, uni, loss, B);
    return (int)cudaGetLastError();
}

extern "C" int umr_iou_backward(const float* target, const float* inter, const float* uni, const float* grad_loss,
                                float* grad_predict, int32_t B, int64_t N, void* stream_) {
    return iou_backward(target, inter, uni, grad_loss, grad_predict, B, N, stream_);
}

extern "C" int umr_chamfer_forward(const float* a, const float* b, float* dist_ab, float* dist_ba, int32_t* idx_ab,
                                   int32_t* idx_ba, int32_t B, int32_t N, int32_t M, int32_t D, void* stream_) {
    return chamfer_forward(a, b, dist_ab, dist_ba, idx_ab, idx_ba, B, N, M, D, stream_);
}

extern "C" int umr_chamfer_backward(const float* a, const float* b, const int32_t* idx_ab, const int32_t* idx_ba,
                                    const float* grad_dist_ab, const float* grad_dist_ba, float* grad_a, float* grad_b,
                                    int32_t B, int32_t N, int32_t M, int32_t D, void* stream_) {
    if (!a || !b || !grad_a || !grad_b || B <= 0 || N <= 0 || M <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (D != 2 && D != 3) return UMR_ERR_UNSUPPORTED;
    if ((grad_dist_ab && !idx_ab) || (grad_dist_ba && !idx_ba)) return UMR_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(grad_a, 0, (size_t)B * N * D * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    e = cudaMemsetAsync(grad_b, 0, (size_t)B * M * D * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    auto bwd = D == 2 ? k_chamfer_bwd<2> : k_chamfer_bwd<3>;
    if (grad_dist_ab) launch(bwd, dim3((N + 255) / 256, B), 256, 0, st, a, b, idx_ab, grad_dist_ab, grad_a, grad_b, N, M);
    if (grad_dist_ba) launch(bwd, dim3((M + 255) / 256, B), 256, 0, st, b, a, idx_ba, grad_dist_ba, grad_b, grad_a, M, N);
    return (int)cudaGetLastError();
}

extern "C" int umr_texcycle_forward(const float* flow, const float* prob, const float* face_ids, uint8_t* visible,
                                    float* loss, int32_t B, int32_t F, int32_t T2, int64_t P, void* stream_) {
    // face_ids == NULL: `visible` was already filled by umr_raster_visibility (its visible_faces output)
    if (!flow || !prob || !visible || !loss || B <= 0 || F <= 0 || T2 <= 0 || (face_ids && P <= 0) ||
        vec2_misaligned(flow) || vec2_misaligned(prob))
        return UMR_ERR_BAD_ARG;
    if (B > 65535 || (int64_t)B * F > INT_MAX) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(loss, 0, sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    if (face_ids) {
        e = cudaMemsetAsync(visible, 0, (size_t)B * F, st);
        if (e != cudaSuccess) return (int)e;
        const int64_t blocks = (P / 4 + 255) / 256 + 1;
        launch(k_visible, dim3((unsigned)(blocks > 1024 ? 1024 : blocks), B), 256, 0, st, face_ids, visible, F, P);
    }
    const int n = B * F;
    const float scale = 1.f / ((float)n * 2.f);  // MSELoss mean over B*F*2 elements
    launch(k_texcycle_fwd<float, false>, (n + 255) / 256, 256, 0, st, reinterpret_cast<const float2*>(flow),
           reinterpret_cast<const float2*>(prob), visible, loss, n, T2, scale);
    return (int)cudaGetLastError();
}

extern "C" int umr_texcycle_backward(const float* flow, const float* prob, const uint8_t* visible, const float* grad_loss,
                                     float* grad_flow, int32_t B, int32_t F, int32_t T2, void* stream_) {
    if (!flow || !prob || !visible || !grad_loss || !grad_flow || B <= 0 || F <= 0 || T2 <= 0 || vec2_misaligned(flow) ||
        vec2_misaligned(prob) || vec2_misaligned(grad_flow))
        return UMR_ERR_BAD_ARG;
    if ((int64_t)B * F > INT_MAX) return UMR_ERR_TOO_LARGE;
    return texcycle_backward(flow, prob, visible, grad_loss, grad_flow, B, F, T2, stream_);
}

extern "C" int umr_masked_l1_forward(const float* pred, int64_t pred_bstride, const float* mask_pred,
                                     int64_t mask_pred_bstride, const float* gt, const float* mask_gt, float* loss,
                                     int32_t B, int32_t C, int64_t HW, void* stream_) {
    if (!pred || !mask_pred || !gt || !mask_gt || !loss || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    if (C != 3 && C != 1) return UMR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(loss, 0, (size_t)B * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    const dim3 grid(ml1_slots(HW), B);
    const float inv_n = 1.f / ((float)C * (float)HW);
    launch(C == 3 ? k_masked_l1_fwd<float, 3, false> : k_masked_l1_fwd<float, 1, false>, grid, ML1_THREADS, 0, st, pred,
           pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, loss, HW, inv_n);
    return (int)cudaGetLastError();
}

extern "C" int umr_masked_l1_backward(const float* pred, int64_t pred_bstride, const float* mask_pred,
                                      int64_t mask_pred_bstride, const float* gt, const float* mask_gt,
                                      const float* grad_loss, float* grad_pred, float* grad_mask_pred, int32_t B,
                                      int32_t C, int64_t HW, void* stream_) {
    return masked_l1_backward(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, grad_loss, grad_pred,
                              grad_mask_pred, B, C, HW, stream_);
}

extern "C" int umr_loss_head_forward(const float* rgba, const float* gt, const float* mask_gt, float* stats,
                                     float* per_image, float* loss, int32_t B, int64_t HW, float w_iou, float w_tex,
                                     void* stream_) {
    if (!rgba || !gt || !mask_gt || !stats || !per_image || !loss || B <= 0 || HW <= 0) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    cudaError_t e = cudaMemsetAsync(stats, 0, (size_t)B * 3 * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    launch(k_losshead_partial<float, false>, dim3(lh_slots(HW), B), LH_THREADS, 0, st, rgba, gt, mask_gt, stats, HW);
    launch(k_losshead_finalize<float>, 1, 32, 0, st, stats, per_image, loss, B, 1.f / (3.f * (float)HW), w_iou, w_tex);
    return (int)cudaGetLastError();
}

extern "C" int umr_loss_head_backward(const float* rgba, const float* gt, const float* mask_gt, const float* stats,
                                      const float* grad_loss, float* grad_rgba, int32_t B, int64_t HW, float w_iou,
                                      float w_tex, void* stream_) {
    return loss_head_backward(rgba, gt, mask_gt, stats, grad_loss, grad_rgba, B, HW, w_iou, w_tex, stream_);
}

// ---------------------------------------------------------------------------------------------
// deterministic mode (include/umr_b200.h, DESIGN.md §2): each reduction CTA stores its partial into a workspace slot
// (grids sized from the shapes only, so the slot layout is fixed) and a finalize kernel sums every image's slots in
// ascending CTA order; the chamfer backward is a gather with one writer per gradient element.  The launchers are the
// float64 entry points' (losses.cuh).
// ---------------------------------------------------------------------------------------------
extern "C" size_t umr_iou_workspace_bytes_deterministic(int32_t B, int64_t N) { return iou_workspace_bytes<float>(B, N); }
extern "C" int umr_iou_forward_deterministic(const float* predict, int64_t predict_bstride, const float* target, float* inter,
                                             float* uni, float* loss, int32_t B, int64_t N, void* workspace, void* stream_) {
    return iou_forward_slots(predict, predict_bstride, target, inter, uni, loss, B, N, workspace, stream_);
}

extern "C" int umr_chamfer_backward_deterministic(const float* a, const float* b, const int32_t* idx_ab, const int32_t* idx_ba,
                                                  const float* grad_dist_ab, const float* grad_dist_ba, float* grad_a,
                                                  float* grad_b, int32_t B, int32_t N, int32_t M, int32_t D, void* stream_) {
    return chamfer_backward_gather(a, b, idx_ab, idx_ba, grad_dist_ab, grad_dist_ba, grad_a, grad_b, B, N, M, D, stream_);
}

extern "C" size_t umr_texcycle_workspace_bytes_deterministic(int32_t B, int32_t F) { return texcycle_workspace_bytes<float>(B, F); }
extern "C" int umr_texcycle_forward_deterministic(const float* flow, const float* prob, const float* face_ids, uint8_t* visible,
                                                  float* loss, int32_t B, int32_t F, int32_t T2, int64_t P, void* workspace,
                                                  void* stream_) {
    return texcycle_forward_slots(flow, prob, face_ids, visible, loss, B, F, T2, P, workspace, stream_);
}

extern "C" size_t umr_masked_l1_workspace_bytes_deterministic(int32_t B, int64_t HW) { return masked_l1_workspace_bytes<float>(B, HW); }
extern "C" int umr_masked_l1_forward_deterministic(const float* pred, int64_t pred_bstride, const float* mask_pred,
                                                   int64_t mask_pred_bstride, const float* gt, const float* mask_gt, float* loss,
                                                   int32_t B, int32_t C, int64_t HW, void* workspace, void* stream_) {
    return masked_l1_forward_slots(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, loss, B, C, HW, workspace,
                                   stream_);
}

extern "C" size_t umr_loss_head_workspace_bytes_deterministic(int32_t B, int64_t HW) { return loss_head_workspace_bytes<float>(B, HW); }
extern "C" int umr_loss_head_forward_deterministic(const float* rgba, const float* gt, const float* mask_gt, float* stats,
                                                   float* per_image, float* loss, int32_t B, int64_t HW, float w_iou,
                                                   float w_tex, void* workspace, void* stream_) {
    return loss_head_forward_slots(rgba, gt, mask_gt, stats, per_image, loss, B, HW, w_iou, w_tex, workspace, stream_);
}

// Sampler (include/umr_b200.h): grad_flow from k_sample_bwd itself (one writer per element, no image gradient there), the
// image gradient from a per-pixel gather over the cell table.
extern "C" int umr_bilinear_sample_cells(const float* flow, int32_t* cells, int32_t B, int32_t H, int32_t W, int32_t N,
                                         void* stream_) {
    return sample_cells(flow, cells, B, H, W, N, stream_);
}
extern "C" int umr_bilinear_sample_backward_deterministic(const float* image, const float* flow, const float* grad_out,
                                                          float* grad_flow, float* grad_image, int32_t B, int32_t C, int32_t H,
                                                          int32_t W, int32_t N, const int32_t* cell_rowptr,
                                                          const int32_t* cell_samples, void* stream_) {
    return sample_backward_gather(image, flow, grad_out, grad_flow, grad_image, B, C, H, W, N, cell_rowptr, cell_samples,
                                  stream_);
}

// part_matching_loss head (include/umr_b200.h, DESIGN.md §13): one entry point per operation for both precisions (the
// double instantiations live in losses_f64.cu).  Slot reductions only, so there is no _deterministic form.
extern "C" size_t umr_part_head_workspace_bytes(int32_t B, int32_t H, int32_t dtype) {
    if (dtype == UMR_DTYPE_FLOAT32) return part_head_workspace_bytes<float>(B, H);
    if (dtype == UMR_DTYPE_FLOAT64) return part_head_workspace_bytes<double>(B, H);
    return 0;
}
extern "C" int umr_part_head_forward(const void* const* maps, const int64_t* map_bstrides, const void* c0, int64_t c0_bstride,
                                     const void* part_segs, int64_t segs_bstride, const void* weights, void* terms, int32_t B,
                                     int32_t H, int32_t kld, int32_t dtype, void* workspace, void* stream_) {
    if (dtype == UMR_DTYPE_FLOAT64)
        return part_head_forward_f64(maps, map_bstrides, c0, c0_bstride, part_segs, segs_bstride, weights, terms, B, H, kld,
                                     workspace, stream_);
    if (dtype != UMR_DTYPE_FLOAT32) return UMR_ERR_BAD_ARG;
    return part_head_forward(reinterpret_cast<const float* const*>(maps), map_bstrides, (const float*)c0, c0_bstride,
                             (const float*)part_segs, segs_bstride, (const float*)weights, (float*)terms, B, H, kld, workspace,
                             stream_);
}
extern "C" int umr_part_head_backward(const void* const* maps, const int64_t* map_bstrides, const void* c0, int64_t c0_bstride,
                                      const void* part_segs, int64_t segs_bstride, const void* weights, const void* workspace,
                                      const void* grad_terms, void* grad_maps, int32_t B, int32_t H, int32_t kld, int32_t dtype,
                                      void* stream_) {
    if (dtype == UMR_DTYPE_FLOAT64)
        return part_head_backward_f64(maps, map_bstrides, c0, c0_bstride, part_segs, segs_bstride, weights, workspace,
                                      grad_terms, grad_maps, B, H, kld, stream_);
    if (dtype != UMR_DTYPE_FLOAT32) return UMR_ERR_BAD_ARG;
    return part_head_backward(reinterpret_cast<const float* const*>(maps), map_bstrides, (const float*)c0, c0_bstride,
                              (const float*)part_segs, segs_bstride, (const float*)weights, workspace, (const float*)grad_terms,
                              (float*)grad_maps, B, H, kld, stream_);
}
