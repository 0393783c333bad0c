/* umr_kp_transfer.h -- keypoint transfer of UMR's keypoint evaluation (experiments/test_kp.py:125-193), part of the C ABI
 * of libumr_b200.so and included by umr_b200.h, whose conventions hold here (caller-allocated device buffers, work
 * enqueued on `stream`, 0 / positive cudaError_t / negative UMR_ERR_* return).  Declared apart from umr_b200.h's own list
 * and bound by _lib.KP_EXPORTS, with their refusals tested beside them (DESIGN.md §16).
 *
 * Both entry points: float32, contiguous buffers, one result per (pair, keypoint) in out [P,K,2] (fully written), no
 * atomics (bitwise reproducible), one kernel launch, no host synchronisation (CUDA-graph capturable).  kps [P,K,2] are
 * keypoints in [-1, 1] image coordinates (x, y).  grid [S] is the identity grid's coordinate table, torch.linspace(-1, 1,
 * S): the outputs are grid coordinates.  Refused before any device work: a NULL buffer, P, K, F, T2, V, S or sigma
 * <= 0, kps / flows / projections / out not 8-byte aligned or gauss / grid / mask_tgt not 4-byte aligned ->
 * UMR_ERR_BAD_ARG; sigma > 18 (the table exceeds 48 KB of shared memory), P * K, F * T2, V or S * S >= 2^30 ->
 * UMR_ERR_TOO_LARGE.  Contract and deviations: DESIGN.md §16. */
#ifndef UMR_KP_TRANSFER_H_
#define UMR_KP_TRANSFER_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Flow mode (test_kp.py:125-158, kp_utils.py:42-69).  Per (pair, keypoint): the Gaussian heat map of draw_labelmap at
 * pt = (kp + 1) / 2 * 256 (256 whatever S, as the reference writes it) on an S x S image, from gauss [(6 sigma + 1)^2]
 * (the reference's unnormalised Gaussian, float32), its window clamped to the table where float32 rounding widens it;
 * sampled bilinearly (align_corners=True, zeros padding) at the T2 points of each face of flow_src [P,F,T2,2] and averaged (summed in order, divided by T2); the first face of largest mean
 * (NaN first, as torch.max); out = the identity grid sampled at that face's T2 points of flow_tgt [P,F,T2,2], averaged. */
int umr_kp_transfer_flow(const float* kps, const float* flow_src, const float* flow_tgt, const float* gauss,
                         const float* grid, float* out, int32_t P, int32_t K, int32_t F, int32_t T2, int32_t S,
                         int32_t sigma, void* stream);

/* Camera mode (test_kp.py:160-193).  Per (pair, keypoint): the nearest source vertex of proj_src [P,V,2] to the keypoint,
 * then the nearest foreground pixel (mask_tgt [P,S,S] != 0) of the target to that vertex's proj_tgt [P,V,2]; out = the
 * pixel's (grid[x], grid[y]).  Distances and ties as umr_chamfer_forward (lowest index).  An empty mask, or no finite
 * distance, gives (NaN, NaN). */
int umr_kp_transfer_cam(const float* kps, const float* proj_src, const float* proj_tgt, const float* mask_tgt,
                        const float* grid, float* out, int32_t P, int32_t K, int32_t V, int32_t S, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* UMR_KP_TRANSFER_H_ */
