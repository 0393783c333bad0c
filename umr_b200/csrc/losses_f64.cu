// losses_f64.cu -- the float64 entry points of the loss kernels of losses.cuh (sampler, IoU, masked L1, loss head, chamfer,
// TexCycle), behind the `umr_*_f64` entry points of include/umr_b200.h.  ops.py takes them when any floating-point input
// of an op is float64 (DESIGN.md §10).  The float64 Laplacian, flatten and CorrLossChamfer entry points sit next to their
// float32 ones in mesh_ops.cu and vertex.cu.
//
// This unit instantiates the kernels for double and is compiled with -fmad=false: each product and sum is rounded once,
// in the written order (the float32 instantiations in losses.cu keep FMA contraction, hence two units).  The float64 path
// is the deterministic structure: every reduction CTA stores its partial into a workspace slot (grids sized from the
// shapes only) and a finalize kernel sums each row's slots in ascending order; every gradient element has exactly one
// writer.  There are no atomics, so every output is bitwise reproducible for identical inputs on the same device type and
// library build, with no separate deterministic variant.
#include <cuda_runtime.h>
#include <stdint.h>

#include <climits>

#include "common.cuh"
#include "losses.cuh"
#include "umr_b200.h"

using namespace umr;

extern "C" int umr_bilinear_sample_forward_f64(const double* image, const double* flow, double* out, int32_t B, int32_t C,
                                               int32_t H, int32_t W, int32_t N, void* stream_) {
    return sample_forward(image, flow, out, B, C, H, W, N, stream_);
}

extern "C" int umr_bilinear_sample_cells_f64(const double* flow, int32_t* cells, int32_t B, int32_t H, int32_t W, int32_t N,
                                             void* stream_) {
    return sample_cells(flow, cells, B, H, W, N, stream_);
}

extern "C" int umr_bilinear_sample_backward_f64(const double* image, const double* flow, const double* grad_out,
                                                double* grad_flow, double* grad_image, int32_t B, int32_t C, int32_t H,
                                                int32_t W, int32_t N, const int32_t* cell_rowptr,
                                                const int32_t* cell_samples, void* stream_) {
    return sample_backward_gather(image, flow, grad_out, grad_flow, grad_image, B, C, H, W, N, cell_rowptr, cell_samples,
                                  stream_);
}

extern "C" size_t umr_iou_workspace_bytes_f64(int32_t B, int64_t N) { return iou_workspace_bytes<double>(B, N); }
extern "C" int umr_iou_forward_f64(const double* predict, int64_t predict_bstride, const double* target, double* inter,
                                   double* uni, double* loss, int32_t B, int64_t N, void* workspace, void* stream_) {
    return iou_forward_slots(predict, predict_bstride, target, inter, uni, loss, B, N, workspace, stream_);
}
extern "C" int umr_iou_backward_f64(const double* target, const double* inter, const double* uni, const double* grad_loss,
                                    double* grad_predict, int32_t B, int64_t N, void* stream_) {
    return iou_backward(target, inter, uni, grad_loss, grad_predict, B, N, stream_);
}

extern "C" size_t umr_masked_l1_workspace_bytes_f64(int32_t B, int64_t HW) { return masked_l1_workspace_bytes<double>(B, HW); }
extern "C" int umr_masked_l1_forward_f64(const double* pred, int64_t pred_bstride, const double* mask_pred,
                                         int64_t mask_pred_bstride, const double* gt, const double* mask_gt, double* loss,
                                         int32_t B, int32_t C, int64_t HW, void* workspace, void* stream_) {
    return masked_l1_forward_slots(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, loss, B, C, HW, workspace,
                                   stream_);
}
extern "C" int umr_masked_l1_backward_f64(const double* pred, int64_t pred_bstride, const double* mask_pred,
                                          int64_t mask_pred_bstride, const double* gt, const double* mask_gt,
                                          const double* grad_loss, double* grad_pred, double* grad_mask_pred, int32_t B,
                                          int32_t C, int64_t HW, void* stream_) {
    return masked_l1_backward(pred, pred_bstride, mask_pred, mask_pred_bstride, gt, mask_gt, grad_loss, grad_pred,
                              grad_mask_pred, B, C, HW, stream_);
}

extern "C" size_t umr_loss_head_workspace_bytes_f64(int32_t B, int64_t HW) { return loss_head_workspace_bytes<double>(B, HW); }
extern "C" int umr_loss_head_forward_f64(const double* rgba, const double* gt, const double* mask_gt, double* stats,
                                         double* per_image, double* loss, int32_t B, int64_t HW, double w_iou, double w_tex,
                                         void* workspace, void* stream_) {
    return loss_head_forward_slots(rgba, gt, mask_gt, stats, per_image, loss, B, HW, w_iou, w_tex, workspace, stream_);
}
extern "C" int umr_loss_head_backward_f64(const double* rgba, const double* gt, const double* mask_gt, const double* stats,
                                          const double* grad_loss, double* grad_rgba, int32_t B, int64_t HW, double w_iou,
                                          double w_tex, void* stream_) {
    return loss_head_backward(rgba, gt, mask_gt, stats, grad_loss, grad_rgba, B, HW, w_iou, w_tex, stream_);
}

extern "C" int umr_chamfer_forward_f64(const double* a, const double* b, double* dist_ab, double* dist_ba, int32_t* idx_ab,
                                       int32_t* idx_ba, int32_t B, int32_t N, int32_t M, int32_t D, void* stream_) {
    return chamfer_forward(a, b, dist_ab, dist_ba, idx_ab, idx_ba, B, N, M, D, stream_);
}
extern "C" int umr_chamfer_backward_f64(const double* a, const double* b, const int32_t* idx_ab, const int32_t* idx_ba,
                                        const double* grad_dist_ab, const double* grad_dist_ba, double* grad_a, double* grad_b,
                                        int32_t B, int32_t N, int32_t M, int32_t D, void* stream_) {
    return chamfer_backward_gather(a, b, idx_ab, idx_ba, grad_dist_ab, grad_dist_ba, grad_a, grad_b, B, N, M, D, stream_);
}

extern "C" size_t umr_texcycle_workspace_bytes_f64(int32_t B, int32_t F) { return texcycle_workspace_bytes<double>(B, F); }
extern "C" int umr_texcycle_forward_f64(const double* flow, const double* prob, const float* face_ids, uint8_t* visible,
                                        double* loss, int32_t B, int32_t F, int32_t T2, int64_t P, void* workspace,
                                        void* stream_) {
    return texcycle_forward_slots(flow, prob, face_ids, visible, loss, B, F, T2, P, workspace, stream_);
}
extern "C" int umr_texcycle_backward_f64(const double* flow, const double* prob, const uint8_t* visible, const double* grad_loss,
                                         double* grad_flow, int32_t B, int32_t F, int32_t T2, void* stream_) {
    if (!flow || !prob || !visible || !grad_loss || !grad_flow || B <= 0 || F <= 0 || T2 <= 0 || vec2_misaligned(flow) ||
        vec2_misaligned(prob) || vec2_misaligned(grad_flow))
        return UMR_ERR_BAD_ARG;
    if (B > 65535 || (int64_t)B * F > INT_MAX) return UMR_ERR_TOO_LARGE;
    return texcycle_backward(flow, prob, visible, grad_loss, grad_flow, B, F, T2, stream_);
}

// the double half of umr_part_head_forward / _backward (losses.cu), instantiated in this -fmad=false unit
int umr::part_head_forward_f64(const void* const* maps, const int64_t* map_bstrides, const void* c0, int64_t c0_bstride,
                               const void* part_segs, int64_t segs_bstride, const void* weights, void* terms, int32_t B,
                               int32_t H, int32_t kld, void* workspace, void* stream_) {
    return part_head_forward(reinterpret_cast<const double* const*>(maps), map_bstrides, (const double*)c0, c0_bstride,
                             (const double*)part_segs, segs_bstride, (const double*)weights, (double*)terms, B, H, kld,
                             workspace, stream_);
}
int umr::part_head_backward_f64(const void* const* maps, const int64_t* map_bstrides, const void* c0, int64_t c0_bstride,
                                const void* part_segs, int64_t segs_bstride, const void* weights, const void* workspace,
                                const void* grad_terms, void* grad_maps, int32_t B, int32_t H, int32_t kld, void* stream_) {
    return part_head_backward(reinterpret_cast<const double* const*>(maps), map_bstrides, (const double*)c0, c0_bstride,
                              (const double*)part_segs, segs_bstride, (const double*)weights, workspace,
                              (const double*)grad_terms, (double*)grad_maps, B, H, kld, stream_);
}
