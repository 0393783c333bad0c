/* umr_b200.h -- C ABI of libumr_b200.so: H100 (sm_90a) soft rasteriser + geometric-loss kernels.
 *
 * This is the drop-in boundary for the hot path of NVlabs/UMR (SURVEY.md §8b).  Each entry point
 * replaces a reference interface, cited as file:line under the reference tree:
 *
 *   umr_raster_forward / umr_raster_backward
 *       replace the pybind functions `forward_soft_rasterize` / `backward_soft_rasterize` of
 *       external/SoftRas/soft_renderer/cuda/soft_rasterize_cuda.cpp:62-97 / :100-138 (kernels
 *       soft_rasterize_cuda_kernel.cu:222-282, :285-476, :479-656) AND the host work around them in
 *       functional/soft_rasterize.py:41-73,94-106 (buffer fills, `grid`, p2f normalisation) and
 *       rasterizer.py:52-53 (2x2 average pool), which are fused into the kernels.
 *   umr_bilinear_sample_forward / _backward
 *       replace `F.grid_sample` (+permute) at nnutils/geom_utils.py:41-59 and
 *       nnutils/loss_utils.py:59-64 (torch-1.1 semantics == align_corners=True, zeros padding).
 *   umr_iou_forward / _backward      replace nnutils/loss_utils.py:41-48 (`neg_iou_loss`).
 *   umr_chamfer_forward / _backward  replace nnutils/chamfer_python.py:43-64 (`distChamfer`).
 *   umr_texcycle_forward / _backward replace nnutils/loss_utils.py:152-182 (`TexCycle.forward`).
 *   umr_corr_chamfer_forward / _backward replace nnutils/loss_utils.py:218-248 (`CorrLossChamfer.forward`).
 *   umr_nmr_forward / umr_nmr_backward_textures replace the render of `neural_renderer.Renderer` (driven by
 *       nnutils/nmr_pytorch.py; the upstream package is not vendored, its contract is DESIGN.md §7).
 *
 * Conventions: plain device pointers + sizes, no torch types.  Every buffer is CALLER-allocated
 * (torch owns all memory); the library keeps no global mutable state and is re-entrant across host
 * threads and devices (the device is the current CUDA device of the calling thread).  All work is
 * enqueued asynchronously on `stream` (a cudaStream_t passed as void*).  Return value: 0 on success,
 * a positive cudaError_t, or a negative UMR_ERR_* code; umr_error_string() decodes both.  Nothing
 * is ever printed (the reference only printf()s launch failures, kernel.cu:700-702,734-736,799-801).
 */
#ifndef UMR_B200_H_
#define UMR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UMR_OK 0
#define UMR_ERR_UNSUPPORTED (-1) /* mode combination not built into the sm_90a kernels        */
#define UMR_ERR_BAD_ARG (-2)     /* null pointer / non-positive size / misaligned buffer       */
#define UMR_ERR_TOO_LARGE (-3)   /* size beyond a compiled limit (e.g. num_faces > UMR_RASTER_MAX_FACES) */

/* Largest num_faces of the soft rasteriser: 2^24.  The hard render's face-index plane holds face ids as float, exact
 * below 2^24, and the pair-block headers of meshes above 65535 faces keep 24 face bits. */
#define UMR_RASTER_MAX_FACES 16777216

/* mode ids: same numbering as functional/soft_rasterize.py:22-25 */
enum { UMR_DIST_HARD = 0, UMR_DIST_BARYCENTRIC = 1, UMR_DIST_EUCLIDEAN = 2 };
enum { UMR_RGB_HARD = 0, UMR_RGB_SOFTMAX = 1 };
enum { UMR_ALPHA_HARD = 0, UMR_ALPHA_SUM = 1, UMR_ALPHA_PROD = 2 };
enum { UMR_TEX_SURFACE = 0, UMR_TEX_VERTEX = 1 };

/* Scalar arguments of soft_rasterize (soft_rasterize_cuda.cpp:71-82), plus the fused-host-work
 * fields.  `dist_eps` is the ALREADY TRANSFORMED value log(1/dist_eps - 1) the reference binding
 * receives (functional/soft_rasterize.py:35). */
typedef struct UmrRasterParams {
    int32_t batch_size;    /* B */
    int32_t num_faces;     /* F (<= UMR_RASTER_MAX_FACES); F <= 65535 keeps 16-bit face indices, larger meshes take
                            * the 32-bit-index instantiations of the same kernels */
    int32_t texture_size;  /* T2 = texture_res^2 (surface textures [B,F,T2,3]) */
    int32_t image_size;    /* output image side `is`; raster side S = is * (anti_aliasing ? 2 : 1) */
    int32_t anti_aliasing; /* 1: rasterise at 2*is and 2x2 average-pool (rasterizer.py:43,52-53) */
    float near_plane, far_plane, eps, sigma_val, dist_eps, gamma_val;
    int32_t func_id_dist, func_id_rgb, func_id_alpha, texture_sample_type, double_side;
    float background_color[3];
    /* optional profiling hooks: two cudaEvent_t (from umr_event_create) recorded on `stream`
     * immediately before / after the main raster kernel of the call (NULL = off).  Used by bench.py
     * to time the dominant kernel alone, live, without a profiler. */
    void* ev_kernel_start;
    void* ev_kernel_stop;
    /* optional PAIR BUFFER (device memory, 256-byte aligned, caller-allocated like every other buffer): when given,
     * the forward saves one 32-byte record per surviving (pixel, face) pair and the backward streams them instead
     * of re-deriving the geometry (the role `faces_info`/`soft_colors` play as saved tensors in the reference,
     * functional/soft_rasterize.py:75).  It must be the SAME memory, untouched, in the matching backward call.
     * Tiles whose records do not fit are recomputed in the backward -- results are identical, only slower -- so any
     * size is valid; umr_raster_pair_buffer_bytes() sizes it.  After the forward, the first uint32 of the buffer
     * holds the number of 32-record blocks the render wanted, the second the number of tiles left unsaved.
     * A record keeps the sampled texel's index in a bit field of 23 bits with 16x16 tiles and 21 bits with 32x32 tiles;
     * a texture_size above 2^23 (2^21) saves nothing and the backward recomputes every tile.
     * NULL / 0: nothing is saved (forward-only renders, generic modes). */
    void* pair_buffer;
    uint64_t pair_buffer_bytes;
    /* Texture sharing: G = shared_textures consecutive images use ONE [F,T2,3] texture -- `textures` (and `grad_textures`,
     * summed over each group) are [B/G,F,T2,3].  G == B: one batch-shared parameter; G == 8: the camera hypotheses of a
     * sample (the reference materialises repeat(...) copies, loss_utils.py:305: 70.8 MB at batch 16).  0 or 1: per-image. */
    int32_t shared_textures;
    /* forward tiling: 0 = automatic (by grid size), 16 = 16x16 tiles with one warp per 8x4 pixel block, 32 = 32x32 tiles
     * whose warps grab pixel blocks dynamically (F <= 2048).  Must be the same in the matching backward call. */
    int32_t tile_mode;
    /* colour channels C of `textures` [..,F,T2,C]: 0 or 3 = RGB.  4 = the part-map render of part_matching_loss
     * (loss_utils.py:385-399 renders its four one-hot part maps as four 3-identical-channel images; colour channels
     * never interact in the rasteriser, so ONE render with C = 4 carries all of them): images / soft_colors /
     * grad_images are then [B,5,..] = (c0..c3, alpha), the 4th background value is `background_extra`.  C = 4 is built
     * for UMR's own configuration only (euclidean / softmax / prod, surface textures, no texture gradient). */
    int32_t color_channels;
    float background_extra;
} UmrRasterParams;

const char* umr_error_string(int code);
int umr_version(void);
/* sizeof() of the parameter structs as compiled into the library (binding self-check). */
size_t umr_sizeof_raster_params(void);
size_t umr_sizeof_project_params(void);
/* Number of kernels this library has launched in this process (all entry points, all threads). */
uint64_t umr_launch_count(void);
/* Thin event helpers so callers without a CUDA runtime binding can time on the launch stream. */
int umr_event_create(void** event);
int umr_event_destroy(void* event);
int umr_event_record(void* event, void* stream);
int umr_event_elapsed_ms(void* start, void* stop, float* ms); /* synchronises on `stop` */

/* Bytes of scratch `workspace` umr_raster_forward/backward need (256-byte aligned device memory).  F > 65535: the
 * coarse-bin lists share a pool of 8 entries per face (DESIGN.md §3); bins that overflow it stay correct. */
size_t umr_raster_workspace_bytes(int32_t batch_size, int32_t num_faces, int32_t image_size, int32_t anti_aliasing);
/* Bytes of a pair buffer (UmrRasterParams.pair_buffer) holding at least `capacity_blocks` blocks of 32 pair records
 * plus the per-tile headers.  It reserves 1540 bytes per block while a block takes 1028 (32 records of 32 bytes and a
 * 4-byte header), so the buffer holds about 1.5x `capacity_blocks`: renders denser than the caller's estimate keep all
 * their records instead of recomputing tiles in the backward. */
size_t umr_raster_pair_buffer_bytes(int32_t batch_size, int32_t image_size, int32_t anti_aliasing,
                                    uint64_t capacity_blocks);

/* Forward.  face_vertices [B,F,9] f32 (x0,y0,z0,x1,...), textures [B,F,T2,3] f32.
 * Outputs (all fully written, no pre-fill needed):
 *   images      [B,4,is,is]   pooled RGBA (== soft_colors when anti_aliasing == 0); [B,5,..] with color_channels == 4
 *   soft_colors [B,4,S,S]     un-pooled RGBA, needed by backward; may be NULL when anti_aliasing==0
 *                             (images is then the un-pooled tensor) or when no backward will follow
 *   aggrs_info  [B,2,S,S]     softmax: (sum, max); hard: (depth_min, float(face_index_min))
 *   p2f_info    [B,F,2]       normalised pixel->face affinity (zeros in hard mode); may be NULL */
int umr_raster_forward(const float* face_vertices, const float* textures, float* images,
                       float* soft_colors, float* aggrs_info, float* p2f_info,
                       const UmrRasterParams* params, void* workspace, void* stream);

/* Visibility only: aggrs_info [B,2,S,S] = (depth_min, float(face_index_min)) of the hard z-buffer, bit-identical to what
 * umr_raster_forward writes with func_id_rgb = UMR_RGB_HARD, without the distance / sigmoid / alpha / colour arithmetic and
 * without image planes.  This is all the reference keeps of the hard render in MultiTextureLoss (nnutils/loss_utils.py:327-329:
 * `_, p2f_info, aggr_info = self.hard_renderer(...)`; p2f_info is zero in hard mode, kernel.cu:417-431).  Same params
 * struct and workspace as umr_raster_forward (UMR's configuration: euclidean / prod / surface).
 * visible_faces [B,F] u8 (optional): 1 where the face wins at least one pixel (a background pixel marks face F-1, as the
 * reference's negative index does) -- the set TexCycle extracts from the plane with torch.unique (loss_utils.py:161-166); hand it to umr_texcycle_forward(face_ids = NULL, visible = ...).  aggrs_info
 * may then be NULL: no plane is written at all. */
int umr_raster_visibility(const float* face_vertices, float* aggrs_info, uint8_t* visible_faces,
                          const UmrRasterParams* params, void* workspace, void* stream);

/* Backward.  grad_images [B,4,is,is] is the gradient w.r.t. `images` (the 2x2 pool backward is
 * fused).  Outputs are zero-filled by the call, then accumulated:
 *   grad_faces    [B,F,9]     may be NULL when grad_textures is given: texture-only backward for renders of DETACHED
 *                             geometry (UMR's texture branch, experiments/train_s2.py:248) -- the vertex-gradient
 *                             arithmetic is compiled out (euclidean / prod / surface configuration only)
 *   grad_textures [B,F,T2,3]  may be NULL (skips the texture gradient, e.g. silhouette renders)
 * Only the sampled texel receives texture gradient (intended semantics of kernel.cu:199-218; the
 * reference's uninitialised-variable behaviour is NOT reproduced -- SURVEY.md App. B-1). */
int umr_raster_backward(const float* face_vertices, const float* textures, const float* soft_colors,
                        const float* aggrs_info, const float* grad_images, float* grad_faces,
                        float* grad_textures, const UmrRasterParams* params, void* workspace,
                        void* stream);

/* Deterministic mode (DESIGN.md §3).  Same arguments and outputs as umr_raster_forward / umr_raster_backward, but every
 * output is bitwise identical for identical inputs on the same device type and library build, whatever the stream, host
 * thread, concurrent work or CUDA-graph replay: p2f sums are exact fixed point (integer REDs), and the backward is a
 * face-parallel gather in which every gradient element has exactly one writer.  The pair buffer and tile_mode are ignored
 * (the 16x16-tile forward always runs, and the backward recomputes every pair).  No host synchronisation; constant launch
 * count.  Every mode check_params accepts (all distance, alpha and texture modes, softmax or hard, 3 or 4 channels, shared
 * textures, any F up to UMR_RASTER_MAX_FACES, grad_faces == NULL for a texture-only backward); a raster side S above
 * 65535 * 16 returns UMR_ERR_TOO_LARGE.  A face covering most of the raster is walked by one warp (DESIGN.md §3).  The workspace must hold
 * umr_raster_workspace_bytes_deterministic() bytes: umr_raster_workspace_bytes() plus 104 bytes per (image, face) for the
 * fixed-point accumulators (rounded up to 256). */
size_t umr_raster_workspace_bytes_deterministic(int32_t batch_size, int32_t num_faces, int32_t image_size,
                                                int32_t anti_aliasing);
int umr_raster_forward_deterministic(const float* face_vertices, const float* textures, float* images,
                                     float* soft_colors, float* aggrs_info, float* p2f_info,
                                     const UmrRasterParams* params, void* workspace, void* stream);
int umr_raster_backward_deterministic(const float* face_vertices, const float* textures, const float* soft_colors,
                                      const float* aggrs_info, const float* grad_images, float* grad_faces,
                                      float* grad_textures, const UmrRasterParams* params, void* workspace,
                                      void* stream);

/* Double precision (DESIGN.md §9).  The arguments, outputs, validation and error codes of umr_raster_forward /
 * umr_raster_backward with every buffer in double: an operation-for-operation twin of the reference kernels' `scalar_t =
 * double` instantiation (every operation one IEEE binary64 rounding; the scalars of UmrRasterParams stay float, as in the
 * reference binding, and are widened on use; background_color is the float value widened).  Every mode combination with 3
 * colour channels (color_channels 0 or 3; 4 returns UMR_ERR_BAD_ARG), shared textures, any F up to UMR_RASTER_MAX_FACES,
 * grad_faces == NULL or grad_textures == NULL in the backward; pair_buffer and tile_mode are ignored.  A raster side S
 * above 65535 * 16 returns UMR_ERR_TOO_LARGE.  Every output is bitwise identical for identical inputs on the same device
 * type and library build, whatever the stream, host thread, concurrent work or CUDA-graph replay: p2f sums are exact fixed
 * point with 128 fractional bits (integer REDs), and the backward is a face-parallel gather in which every gradient element
 * has exactly one writer, so there is no separate deterministic variant.  A face covering most of the raster is walked by
 * one warp in the backward.  No host synchronisation; constant launch count.  The workspace must hold
 * umr_raster_workspace_bytes_f64() bytes (256-byte aligned): 440 bytes per (image, face), each part rounded up to 256. */
size_t umr_raster_workspace_bytes_f64(int32_t batch_size, int32_t num_faces, int32_t image_size, int32_t anti_aliasing);
int umr_raster_forward_f64(const double* face_vertices, const double* textures, double* images, double* soft_colors,
                           double* aggrs_info, double* p2f_info, const UmrRasterParams* params, void* workspace,
                           void* stream);
int umr_raster_backward_f64(const double* face_vertices, const double* textures, const double* soft_colors,
                            const double* aggrs_info, const double* grad_images, double* grad_faces,
                            double* grad_textures, const UmrRasterParams* params, void* workspace, void* stream);

/* Fused vertex pipeline (SURVEY.md §8f-1): 7-dof orthographic camera projection with z
 * (nnutils/geom_utils.py:74-91,119-165), y flip (nnutils/smr.py:36), look_at with the eye on the z axis
 * + orthogonal scale (SoftRas/functional/look_at.py:48-60, orthogonal.py:13-16), the face gather
 * (functional/face_vertices.py:16-22) and, optionally, the per-face surface light
 * (SoftRas/lighting.py:50-57, mesh.py:112-118) in ONE kernel; bit-identical to the torch-op chain. */
typedef struct UmrProjectParams {
    int32_t batch_size, num_vertices, num_faces;
    int32_t flip_y;              /* 1: y *= -1 after the projection (smr.py:36) */
    int64_t faces_batch_stride;  /* elements between consecutive batches of `faces` (F*3, or 0 if shared) */
    float offset_z;              /* smr.py:66 */
    float eye_z;                 /* look_at eye = (0, 0, eye_z) (smr.py:60: -2.732) */
    float viewing_scale;         /* orthogonal scale */
    int32_t light_enabled;       /* 0: `light` is not written */
    float light_intensity_ambient, light_intensity_directional;
    float light_color_ambient[3], light_color_directional[3], light_direction[3];
    /* > 1: every `num_hypotheses` consecutive renders (camera hypotheses, cams [B,7]) share ONE mesh: vertices are
     * [B / num_hypotheses, V, 3] (faces likewise when batched) -- the reference materialises repeat(1, 8, ...) copies
     * (loss_utils.py:260-261, 303-304); grad_vertices is [B / num_hypotheses, V, 3], summed over the hypotheses. */
    int32_t num_hypotheses;
} UmrProjectParams;

/* vertices [B,V,3] f32, cams [B,7] = [s,tx,ty,qw,qx,qy,qz], faces int32 -> face_vertices [B,F,9]
 * (raster space) and light [B,F,3] (NULL or light_enabled == 0 to skip).  A face index outside [0,V) is never
 * dereferenced: that face's vertices (and light) become NaN in the forward and it contributes nothing in the
 * backward (the reference's torch indexing raises a device-side assert, functional/face_vertices.py:22). */
int umr_project_faces_forward(const float* vertices, const float* cams, const int32_t* faces,
                              float* face_vertices, float* light, const UmrProjectParams* params,
                              void* stream);
/* grad_face_vertices [B,F,9] (+ grad_light [B,F,3] or NULL) -> grad_vertices [B,V,3] (NULL to skip),
 * grad_cams [B,7] (NULL to skip).  grad_proj [B,V,3] is scratch (zero-filled by the call). */
int umr_project_faces_backward(const float* vertices, const float* cams, const int32_t* faces,
                               const float* grad_face_vertices, const float* grad_light, float* grad_proj,
                               float* grad_vertices, float* grad_cams, const UmrProjectParams* params,
                               void* stream);

/* Bilinear sampler, align_corners=True, zeros padding (geom_utils.py:41-59, loss_utils.py:59-64).
 * image [B,C,H,W], flow [B,N,2] (x,y in [-1,1]) -> out [B,N,C] (i.e. already permuted to the
 * `B x F x T x T x C` order sample_textures returns).  Backward: gradient w.r.t. flow only
 * (grad_flow [B,N,2], fully written) -- and optionally w.r.t. image (grad_image [B,C,H,W],
 * zero-filled by the call then accumulated; NULL to skip). */
int umr_bilinear_sample_forward(const float* image, const float* flow, float* out, int32_t B,
                                int32_t C, int32_t H, int32_t W, int32_t N, void* stream);
int umr_bilinear_sample_backward(const float* image, const float* flow, const float* grad_out,
                                 float* grad_flow, float* grad_image, int32_t B, int32_t C,
                                 int32_t H, int32_t W, int32_t N, void* stream);

/* neg_iou_loss (loss_utils.py:41-48).  predict/target [B,N] -> inter[B], uni[B] (uni includes the
 * +1e-6) and loss[B] = 1 - inter/uni.  `predict` may be a strided view (e.g. the alpha plane of the
 * RGBA render): predict_bstride = elements between batch items (N when contiguous).
 * Backward: grad_predict[B,N] (contiguous) = grad_loss[b] * dloss/dp. */
int umr_iou_forward(const float* predict, int64_t predict_bstride, const float* target, float* inter,
                    float* uni, float* loss, int32_t B, int64_t N, void* stream);
int umr_iou_backward(const float* target, const float* inter, const float* uni,
                     const float* grad_loss, float* grad_predict, int32_t B, int64_t N,
                     void* stream);

/* texture_loss_masks (loss_utils.py:103-116): per image mean |pred*mask_pred - gt*mask_gt| over C*H*W.
 * pred [B,C,HW] and mask_pred [B,HW] may be strided views of the RGBA render: their batch strides (in
 * elements) are passed; gt [B,C,HW], mask_gt [B,HW] contiguous.  loss [B] (zero-filled by the call).
 * Backward: grad_pred [B,C,HW], grad_mask_pred [B,HW] (contiguous, fully written; either may be NULL). */
int umr_masked_l1_forward(const float* pred, int64_t pred_bstride, const float* mask_pred,
                          int64_t mask_pred_bstride, const float* gt, const float* mask_gt, float* loss,
                          int32_t B, int32_t C, int64_t HW, void* stream);
int umr_masked_l1_backward(const float* pred, int64_t pred_bstride, const float* mask_pred,
                           int64_t mask_pred_bstride, const float* gt, const float* mask_gt,
                           const float* grad_loss, float* grad_pred, float* grad_mask_pred, int32_t B,
                           int32_t C, int64_t HW, void* stream);

/* Fused loss head on one RGBA render: loss[0] = w_iou * mean_b neg_iou_loss(alpha, mask_gt) +
 * w_tex * mean_b texture_loss_masks(rgb, gt, mask_gt, alpha) -- loss_utils.py:41-48 and :103-116 applied to the same
 * render (the reference computes them with ~25 elementwise / reduce kernels; train_s1.py:211-215, bench step §8d).
 * rgba [B,4,HW] (the renderer's output, contiguous), gt [B,3,HW], mask_gt [B,HW].
 * stats [B,3] (written: I, U + 1e-6, sum|.|; needed by backward), per_image [B,2] = (1 - I/U, L1 mean), loss [1].
 * Backward: grad_rgba [B,4,HW] fully written from the scalar grad_loss[1]. */
int umr_loss_head_forward(const float* rgba, const float* gt, const float* mask_gt, float* stats, float* per_image,
                          float* loss, int32_t B, int64_t HW, float w_iou, float w_tex, void* stream);
int umr_loss_head_backward(const float* rgba, const float* gt, const float* mask_gt, const float* stats,
                           const float* grad_loss, float* grad_rgba, int32_t B, int64_t HW, float w_iou, float w_tex,
                           void* stream);

/* distChamfer (chamfer_python.py:43-64) for D == 2 or 3.  a [B,N,D], b [B,M,D] ->
 * dist_ab[B,N], dist_ba[B,M], idx_ab[B,N] (int32), idx_ba[B,M] (int32), using the reference's
 * expanded form |a|^2 + |b|^2 - 2 a.b and lowest-index tie-breaking.
 * Backward: grad_a[B,N,D], grad_b[B,M,D] from grad_dist_ab / grad_dist_ba (either may be NULL). */
int umr_chamfer_forward(const float* a, const float* b, float* dist_ab, float* dist_ba,
                        int32_t* idx_ab, int32_t* idx_ba, int32_t B, int32_t N, int32_t M,
                        int32_t D, void* stream);
int umr_chamfer_backward(const float* a, const float* b, const int32_t* idx_ab,
                         const int32_t* idx_ba, const float* grad_dist_ab,
                         const float* grad_dist_ba, float* grad_a, float* grad_b, int32_t B,
                         int32_t N, int32_t M, int32_t D, void* stream);

/* CorrLossChamfer (nnutils/loss_utils.py:194-248; call site experiments/train_s2.py:300-315) fused: project the NS selected
 * part vertices (`selection` [NS] int32 = head | belly | neck | back indices concatenated, `part_ends` [4] their cumulative
 * counts, loss_utils.py:211-216) with the render's camera (orthographic_proj_withz(...)[:, :, :2], geom_utils.py:74-91),
 * squared distance of every projected vertex to the nearest of its part's targets (targets[g] [B, target_counts[g], 2];
 * the `dist1` of distChamfer, chamfer_python.py:43-64, in the defined fp32 order of umr_chamfer_forward), times weights[g],
 * mean over the NS vertices (loss_utils.py:232-239).  vertices [B,V,3] with `vertices_batch_stride` elements between renders
 * (0 = one mesh shared by all renders, e.g. the mean shape).  Outputs: vert2d [B,NS,2], nearest [B,NS] int32, loss [B].
 * The four `targets` pointers / counts / ends / weights are HOST arrays of length 4.
 * Backward: grad_loss [B], optional grad_vert2d [B,NS,2] -> grad_vertices [B,V,3] (zero-filled by the call; may be NULL) and
 * grad_cams [B,7] (may be NULL).  Targets receive no gradient (they are data in the reference). */
int umr_corr_chamfer_forward(const float* vertices, int64_t vertices_batch_stride, const float* cams,
                             const int32_t* selection, const float* const* targets, const int32_t* target_counts,
                             const int32_t* part_ends, const float* weights, float* vert2d, int32_t* nearest,
                             float* loss, int32_t B, int32_t NS, void* stream);
int umr_corr_chamfer_backward(const float* vertices, int64_t vertices_batch_stride, const float* cams,
                              const int32_t* selection, const float* const* targets, const int32_t* target_counts,
                              const int32_t* part_ends, const float* weights, const float* vert2d,
                              const int32_t* nearest, const float* grad_loss, const float* grad_vert2d,
                              float* grad_vertices, float* grad_cams, int32_t B, int32_t NS, int32_t V, void* stream);

/* TexCycle (loss_utils.py:152-182).  flow [B,F,T2,2], prob [B,F,2], face_ids [B,P] (the hard
 * renderer's aggrs_info[:,1] plane as float, -1 = background which marks face F-1 visible like the
 * reference's negative index does).  visible [B,F] (uint8 scratch, written), loss[1].
 * Backward: grad_flow [B,F,T2,2] = grad_loss * dloss/dflow. */
int umr_texcycle_forward(const float* flow, const float* prob, const float* face_ids,
                         uint8_t* visible, float* loss, int32_t B, int32_t F, int32_t T2,
                         int64_t P, void* stream);
int umr_texcycle_backward(const float* flow, const float* prob, const uint8_t* visible,
                          const float* grad_loss, float* grad_flow, int32_t B, int32_t F,
                          int32_t T2, void* stream);

/* Texture atlas (SoftRas natives, SURVEY.md §8f-3).
 * umr_create_texture_image: cuda/create_texture_image_cuda_kernel.cu:10-105.  faces_uv [F,3,2] (pixel coordinates of the
 *   three corners in the atlas), textures [F,R*R,3] -> image [H,W,3] (pixels of tiles >= F are left untouched).
 * umr_load_textures: cuda/load_textures_cuda_kernel.cu:8-98.  image [H,W,3], faces_uv [F,3,2] in [0,1], is_update [F]
 *   int32 -> textures [F,R*R,3] (faces with is_update == 0 are left untouched); bilinear. */
int umr_create_texture_image(const float* faces_uv, const float* textures, float* image, int32_t num_faces,
                             int32_t texture_res_in, int32_t image_height, int32_t image_width, float eps, void* stream);
int umr_load_textures(const float* image, const float* faces_uv, const int32_t* is_update, float* textures,
                      int32_t num_faces, int32_t texture_res, int32_t image_height, int32_t image_width, void* stream);

/* Mesh regularisers (SoftRas/losses.py, SURVEY.md §8f-4).
 * Laplacian (losses.py:6-37): CSR neighbour table rowptr [V+1], col [nnz], coef [nnz] (off-diagonal entries of the
 *   row-normalised Laplacian; the diagonal is 1); x [B,V,3] -> y [B,V,3] = L x (saved for backward), loss [B] = |y|^2.
 *   Backward: tcoef [nnz] = coef of row col[e] towards the row's vertex (the transposed entries); grad_x [B,V,3].
 * Flatten (losses.py:39-114): edges [E,4] = (v0, v1, v2, v3) int32; loss [B] = sum_e (cos + 1)^2; backward zero-fills
 *   grad_vertices [B,V,3] and accumulates. */
int umr_laplacian_forward(const float* x, const int32_t* rowptr, const int32_t* col, const float* coef, float* y,
                          float* loss, int32_t B, int32_t V, void* stream);
int umr_laplacian_backward(const float* y, const int32_t* rowptr, const int32_t* col, const float* tcoef,
                           const float* grad_loss, float* grad_x, int32_t B, int32_t V, void* stream);
int umr_flatten_forward(const float* vertices, const int32_t* edges, float* loss, int32_t B, int32_t V, int32_t E,
                        float eps, void* stream);
int umr_flatten_backward(const float* vertices, const int32_t* edges, const float* grad_loss, float* grad_vertices,
                         int32_t B, int32_t V, int32_t E, float eps, void* stream);

/* Barrier distance transform of the GT masks (utils/image.py:130-141 `compute_dt_barrier`, run with scipy on the host
 * per image per step at train_s2.py:196): mask [B,H,W] (non-zero = object) -> dt [B,H,W] =
 * 1 / (1 + exp(-k * (EDT(1-mask) - EDT(mask)) / max(H,W))), exact Euclidean distances.  workspace:
 * umr_dt_barrier_workspace_bytes(B,H,W) bytes of device scratch. */
size_t umr_dt_barrier_workspace_bytes(int32_t B, int32_t H, int32_t W);
int umr_dt_barrier(const float* mask, float* dt, void* workspace, int32_t B, int32_t H, int32_t W, float k, void* stream);

/* One-shot all-reduce of the flat shared-parameter gradient over NVLink peer memory (SURVEY.md §8e; reference:
 * the implicit gradient reduce of torch.nn.DataParallel, experiments/train_s2.py:101,133,149,164).
 *   peer_buffers_dev  device array of `world` uint64: the address of every rank's SYMMETRIC buffer as mapped into this
 *                     process (rank r's own buffer at index r).  Each buffer holds n_floats fp32 gradient values and,
 *                     at flag_offset_bytes (16-byte aligned, >= 4*n_floats), umr_p2p_allreduce_flag_bytes() bytes of flag
 *                     words, zero-initialised ONCE by the caller before the first call.
 *   out               local [n_floats]: scale * sum over ranks (every rank computes the same bits).
 *   local_state       16 bytes of local device memory, zero-initialised once.
 * n_floats must be a multiple of 4.  Every rank must issue the same sequence of calls.  The call only enqueues one
 * kernel (CUDA-graph capturable); when it has completed, the symmetric buffer may be overwritten. */
size_t umr_p2p_allreduce_flag_bytes(void);
int umr_p2p_allreduce(const void* peer_buffers_dev, float* out, int64_t n_floats, int64_t flag_offset_bytes,
                      void* local_state, int32_t rank, int32_t world, float scale, void* stream);

/* Hard z-buffer renderer with neural_renderer's conventions: the `Renderer` of nnutils/nmr_pytorch.py:42-43 in UMR's
 * configuration (look_at camera with the eye on the z axis, orthographic), forward and texture gradient.  The render
 * contract is DESIGN.md §7.  The vertex / camera gradient is not built (every UMR call site renders detached geometry). */
typedef struct UmrNmrParams {
    int32_t batch_size, num_vertices, num_faces; /* B, V, F */
    int32_t texture_res;       /* T: textures [B/G, F, T, T, T, 3] (>= 2); ignored without textures */
    int32_t image_size;        /* output side `is`; raster side S = is * (anti_aliasing ? 2 : 1) */
    int32_t anti_aliasing;     /* 1: rasterise at 2*is, then 2x2 average pool */
    int32_t fill_back;         /* 1: faces F..2F-1 are faces 0..F-1 with the vertex order reversed */
    int32_t shared_textures;   /* G: G consecutive renders share one texture (camera hypotheses); 0 or 1: per render */
    float eye_z;               /* look_at eye = (0, 0, eye_z), eye_z < 0: a translation z - eye_z */
    float near_plane, far_plane;
    float light_intensity_ambient, light_intensity_directional;
    float light_color_ambient[3], light_color_directional[3], light_direction[3];
    float background_color[3];
} UmrNmrParams;

size_t umr_sizeof_nmr_params(void);
/* Bytes of 256-byte aligned device scratch umr_nmr_forward / umr_nmr_backward_textures need. */
size_t umr_nmr_workspace_bytes(int32_t batch_size, int32_t num_faces, int32_t fill_back);
/* vertices [B,V,3] f32 (what nmr_pytorch.Render hands over: orthographic_proj_withz(..., offset_z=5) with y negated),
 * faces [B,F,3] int32 (an index outside [0,V) makes that face invisible), textures [B/G,F,T,T,T,3] f32 or NULL.
 * Outputs, all fully written:
 *   face_index   [B,S,S] int32  winning face copy per raster pixel (raster row order, not flipped), -1 = background
 *   raster_depth [B,S,S] f32    its depth, far_plane where no face wins
 *   rgb          [B,3,is,is]    flipped + pooled image (NULL to skip; needs textures)
 *   alpha, depth [B,is,is]      flipped + pooled coverage / depth (NULL to skip) */
int umr_nmr_forward(const float* vertices, const int32_t* faces, const float* textures, int32_t* face_index,
                    float* raster_depth, float* rgb, float* alpha, float* depth, const UmrNmrParams* params,
                    void* workspace, void* stream);
/* Texture gradient of the rgb output: grad_rgb [B,3,is,is] -> grad_textures [B/G,F,T,T,T,3] (zero-filled by the call,
 * then accumulated).  face_index is the forward's plane; vertices / faces / params are the forward's. */
int umr_nmr_backward_textures(const float* vertices, const int32_t* faces, const int32_t* face_index,
                              const float* grad_rgb, float* grad_textures, const UmrNmrParams* params, void* workspace,
                              void* stream);

/* Mesh voxelisation: SoftRas `functional.voxelization` (functional/voxelization.py:41-58, kernels
 * cuda/voxelization_cuda_kernel.cu).  faces [B,F,3,3] (float32 or float64 as `dtype` says, contiguous; coordinates are
 * multiplied by `scale` in that type first: `size`, or 1 for normalize=True) -> voxels [B,vs,vs,vs] int32 (16-byte
 * aligned, fully written): 1 for surface voxels and every empty voxel not 6-connected through empty voxels to the grid
 * boundary, 0 elsewhere.  Bit-exact with the reference's `-fmad=false` build; NaN / inf mark nothing.  The contract is
 * DESIGN.md §8.  workspace: umr_voxelize_workspace_bytes(B, vs) bytes of 256-byte aligned device scratch.  Its first
 * uint32 is a status word, cleared at the start of every call: non-zero when the fill stopped at its sweep cap, i.e.
 * when the result is wrong (a library bug, never expected).  One memset and at most three kernels, whatever the mesh;
 * no allocation, no synchronisation (CUDA-graph capturable).  UMR_ERR_TOO_LARGE when B*vs^3 >= 2^31. */
#define UMR_DTYPE_FLOAT32 0
#define UMR_DTYPE_FLOAT64 1
size_t umr_voxelize_workspace_bytes(int32_t B, int32_t vs);
int umr_voxelize(const void* faces, int32_t dtype, int32_t* voxels, int32_t B, int32_t F, int32_t vs, double scale,
                 void* workspace, void* stream);

/* Deterministic loss kernels (DESIGN.md §2), taken by the autograd Functions of umr_b200/ops.py under
 * torch.use_deterministic_algorithms(True).  Each takes the arguments of its default symbol above, plus a caller-allocated
 * device `workspace` of the size its *_workspace_bytes_deterministic query returns (a function of the sizes only; 0 for an
 * empty size).  Outputs are the default symbol's, bitwise identical for identical inputs (values and memory layout) on
 * the same device type and library build, whatever the stream, host thread, concurrent work or CUDA-graph replay.  No
 * host synchronisation; the launch count depends on the arguments only.  No atomics reach an output:
 *   - reductions (IoU, masked L1, loss head, TexCycle, Laplacian, flatten loss): every CTA of a grid sized from the
 *     shapes stores its partial (the default kernel's in-CTA tree) into its own float slot, and a finalize kernel sums
 *     each image's slots in ascending CTA order, in float, then applies the default finalize (+1e-6, 1 - I/U, scales,
 *     loss-head weights).  The outputs the default call zero-fills or accumulates are fully written instead.
 *   - umr_chamfer_backward_deterministic: a gather with one writer per gradient element (no workspace).  grad_a[i] is
 *     its own idx_ab term plus the idx_ba terms of every j with idx_ba[j] == i; likewise grad_b.
 *   - umr_flatten_backward_deterministic: per-edge vertex terms go to the workspace [B,E,4,3], then a per-vertex gather
 *     sums them over the transposed incidence table: vert_rowptr [V+1], vert_incidence [4E] = edge * 4 + role
 *     (role 0..3 = v0..v3 of the edge row) in ascending order per vertex.
 *   - umr_corr_chamfer_backward_deterministic: per-(render, j) vertex terms go to the workspace [B,NS,3], then a
 *     per-(render, vertex) gather sums them over the transposed selection table: vert_rowptr [V+1], vert_selection [NS]
 *     = the j with selection[j] == v in ascending order per vertex.  grad_cams is the default kernel's.  The workspace
 *     and tables may be NULL when grad_vertices is. */
size_t umr_iou_workspace_bytes_deterministic(int32_t B, int64_t N);                 /* 8 * B * ceil(N / 16384) */
int umr_iou_forward_deterministic(const float* predict, int64_t predict_bstride, const float* target, float* inter,
                                  float* uni, float* loss, int32_t B, int64_t N, void* workspace, void* stream);
size_t umr_masked_l1_workspace_bytes_deterministic(int32_t B, int64_t HW);          /* 4 * B * ceil(HW / 2048) */
int umr_masked_l1_forward_deterministic(const float* pred, int64_t pred_bstride, const float* mask_pred,
                                        int64_t mask_pred_bstride, const float* gt, const float* mask_gt, float* loss,
                                        int32_t B, int32_t C, int64_t HW, void* workspace, void* stream);
size_t umr_loss_head_workspace_bytes_deterministic(int32_t B, int64_t HW);          /* 12 * B * ceil(HW / 2048) */
int umr_loss_head_forward_deterministic(const float* rgba, const float* gt, const float* mask_gt, float* stats,
                                        float* per_image, float* loss, int32_t B, int64_t HW, float w_iou, float w_tex,
                                        void* workspace, void* stream);
size_t umr_texcycle_workspace_bytes_deterministic(int32_t B, int32_t F);            /* 4 * ceil(B * F / 256) */
int umr_texcycle_forward_deterministic(const float* flow, const float* prob, const float* face_ids, uint8_t* visible,
                                       float* loss, int32_t B, int32_t F, int32_t T2, int64_t P, void* workspace,
                                       void* stream);
size_t umr_laplacian_workspace_bytes_deterministic(int32_t B, int32_t V);           /* 4 * B * ceil(V / 256) */
int umr_laplacian_forward_deterministic(const float* x, const int32_t* rowptr, const int32_t* col, const float* coef,
                                        float* y, float* loss, int32_t B, int32_t V, void* workspace, void* stream);
size_t umr_flatten_forward_workspace_bytes_deterministic(int32_t B, int32_t E);     /* 4 * B * ceil(E / 128) */
int umr_flatten_forward_deterministic(const float* vertices, const int32_t* edges, float* loss, int32_t B, int32_t V,
                                      int32_t E, float eps, void* workspace, void* stream);
size_t umr_flatten_backward_workspace_bytes_deterministic(int32_t B, int32_t E);    /* 48 * B * E */
int umr_flatten_backward_deterministic(const float* vertices, const int32_t* edges, const int32_t* vert_rowptr,
                                       const int32_t* vert_incidence, const float* grad_loss, float* grad_vertices,
                                       int32_t B, int32_t V, int32_t E, float eps, void* workspace, void* stream);
int umr_chamfer_backward_deterministic(const float* a, const float* b, const int32_t* idx_ab, const int32_t* idx_ba,
                                       const float* grad_dist_ab, const float* grad_dist_ba, float* grad_a, float* grad_b,
                                       int32_t B, int32_t N, int32_t M, int32_t D, void* stream);
size_t umr_corr_chamfer_workspace_bytes_deterministic(int32_t B, int32_t NS);       /* 12 * B * NS */
int umr_corr_chamfer_backward_deterministic(const float* vertices, int64_t vertices_batch_stride, const float* cams,
                                            const int32_t* selection, const float* const* targets,
                                            const int32_t* target_counts, const int32_t* part_ends, const float* weights,
                                            const float* vert2d, const int32_t* nearest, const float* grad_loss,
                                            const float* grad_vert2d, float* grad_vertices, float* grad_cams, int32_t B,
                                            int32_t NS, int32_t V, const int32_t* vert_rowptr,
                                            const int32_t* vert_selection, void* workspace, void* stream);

/* Deterministic backwards of the vertex pipeline, the NMR texture gradient and the sampler's image gradient (DESIGN.md §2),
 * taken by vertex.ProjectFacesFunction, neural_renderer's _NmrFunction and ops.BilinearSampleFunction under
 * torch.use_deterministic_algorithms(True).  Same guarantees as the loss kernels above: the default symbol's outputs,
 * bitwise identical for identical inputs on the same device type and library build, no atomics reaching an output, no
 * host synchronisation, a launch count that depends on the arguments only.  The transposed tables are "row -> ascending
 * positions" tables (rowptr [R+1], positions), built on the device by umr_b200.ops.device_incidence.
 *   - umr_project_faces_backward_deterministic: the arguments of umr_project_faces_backward, plus the faces' incidence
 *     table and a workspace.  Positions are face * 3 + corner of the flattened faces: rows v over V vertices when the faces
 *     are shared (faces_batch_stride == 0), rows vb * V + v over the Bv meshes otherwise, with positions vb * F * 3 +
 *     face * 3 + corner.  An out-of-range face index must have no row (the builder drops it).  The per-(render, face,
 *     corner) gradients, light term included, are stored to the workspace (zeros for a face with an out-of-range index);
 *     grad_proj[b][v] is their sum in ascending table order; grad_vertices sums the per-render vertex terms in ascending
 *     hypothesis (plain store when num_hypotheses <= 1); grad_cams keeps the default in-CTA tree, each CTA stores its
 *     partial into a slot and the slots are summed in ascending CTA order.
 *     Workspace: 4 * B * (9 * F + 3 * V + 7 * ceil(V / 256)) bytes.
 *   - umr_nmr_backward_textures_deterministic: the arguments and workspace of umr_nmr_backward_textures.  One warp per
 *     (texture group, face) gathers the face's texel gradients over the pixel boxes of its copies (DESIGN.md §3); a thin
 *     or non-finite face is walked over the whole raster.
 *   - umr_bilinear_sample_cells: one int32 cell key per sample (cells [B,N]): (y0+1) * (W+1) + (x0+1) + b * (H+1) * (W+1)
 *     of the sample's top-left corner (x0, y0) as umr_bilinear_sample_backward computes it, or the drop key
 *     B * (H+1) * (W+1) when none of its four corners is inside the image.  UMR_ERR_TOO_LARGE when B * (H+1) * (W+1)
 *     exceeds INT32_MAX.
 *   - umr_bilinear_sample_backward_deterministic: the arguments of umr_bilinear_sample_backward, plus the table of those
 *     keys over R = B * (H+1) * (W+1) rows (cell_rowptr [R+1], cell_samples: flat sample indices b * N + n), NULL when
 *     grad_image is.  grad_flow is the default kernel's; grad_image is fully written by a per-pixel gather (no zero-fill):
 *     roles 00 of cell (y,x), 10 of (y,x-1), 01 of (y-1,x), 11 of (y-1,x-1), samples in ascending order within each. */
size_t umr_project_faces_workspace_bytes_deterministic(int32_t B, int32_t V, int32_t F);
int umr_project_faces_backward_deterministic(const float* vertices, const float* cams, const int32_t* faces,
                                             const float* grad_face_vertices, const float* grad_light, float* grad_proj,
                                             float* grad_vertices, float* grad_cams, const UmrProjectParams* params,
                                             const int32_t* vert_rowptr, const int32_t* vert_incidence, void* workspace,
                                             void* stream);
int umr_nmr_backward_textures_deterministic(const float* vertices, const int32_t* faces, const int32_t* face_index,
                                            const float* grad_rgb, float* grad_textures, const UmrNmrParams* params,
                                            void* workspace, void* stream);
int umr_bilinear_sample_cells(const float* flow, int32_t* cells, int32_t B, int32_t H, int32_t W, int32_t N, void* stream);
int umr_bilinear_sample_backward_deterministic(const float* image, const float* flow, const float* grad_out,
                                               float* grad_flow, float* grad_image, int32_t B, int32_t C, int32_t H,
                                               int32_t W, int32_t N, const int32_t* cell_rowptr,
                                               const int32_t* cell_samples, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* UMR_B200_H_ */
