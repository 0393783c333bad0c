/* umr_semantic_template.h -- the SCOPS semantic template UMR builds between its training stages
 * (experiments/avg_uv.py:203-293 `compute_uv`): the dataset-wide UV part average and the per-texel, per-face and
 * per-vertex part labels of the template.  Part of the C ABI of libumr_b200.so and included by umr_b200.h, whose
 * conventions hold here (caller-allocated device buffers, work enqueued on `stream`, 0 / positive cudaError_t / negative
 * UMR_ERR_* return).  Declared apart from umr_b200.h's own list and bound by _lib.ST_EXPORTS, with its refusals tested
 * beside it.  Every buffer is float32 or int32 unless named otherwise.  No atomics (bitwise reproducible), no host
 * synchronisation.  Contract: DESIGN.md §18. */
#ifndef UMR_SEMANTIC_TEMPLATE_H_
#define UMR_SEMANTIC_TEMPLATE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UMR_ST_MAX_IMAGES 1024        /* B: images one umr_st_average_add ranks */
#define UMR_ST_MAX_CHANNELS 32        /* C: part channels, a label per warp lane */
#define UMR_ST_MAX_COUNT (1 << 30)    /* S * S, H * W, 3 F, F * T2 and V stay below this */

/* Bytes of the workspace of umr_st_average_add: B * ceil(H * W / 1024) float partial distances; 0 for B, H or W <= 0,
 * B > UMR_ST_MAX_IMAGES or H * W >= UMR_ST_MAX_COUNT. */
size_t umr_st_average_workspace_bytes(int32_t B, int32_t H, int32_t W);

/* One batch of the averaging pass.  uv_parts[b] = part_segs[b] [C,S,S] sampled at uvimage_pred[b] [2,H,W] (bilinear,
 * zeros padding, align_corners=True: the sampler's arithmetic, every operation rounded once), never materialised;
 *   dist[b] = sum over (c, y, x) of (uv_parts[b] - exemplar)^2, exemplar [C,H,W] -- per-thread serial sums over 4 pixels
 *   and every channel, a 256-wide shared-memory tree per 1024-pixel tile, then the tiles in order;
 *   selected [k] = the k images first in ascending (dist, image index) order, a NaN distance after every number;
 *   acc [C,H,W] += (((uv_parts[sel0] + uv_parts[sel1]) + ...) + uv_parts[sel(k-1)]).
 * Two launches.  Refused before any device work: a NULL or not 4-byte aligned buffer, B, C, S, H, W or k <= 0, k > B ->
 * UMR_ERR_BAD_ARG; B > UMR_ST_MAX_IMAGES, C > UMR_ST_MAX_CHANNELS, S * S or H * W >= UMR_ST_MAX_COUNT ->
 * UMR_ERR_TOO_LARGE. */
int umr_st_average_add(const float* part_segs, const float* uvimage_pred, const float* exemplar, int32_t B, int32_t C,
                       int32_t S, int32_t H, int32_t W, int32_t k, void* workspace, float* dist, int32_t* selected,
                       float* acc, void* stream);

/* avg_prob [H,W,C] = acc [C,H,W] / (float)count, one IEEE division per element.  One launch.  Refused: a NULL or not
 * 4-byte aligned buffer, C, H, W or count <= 0 -> UMR_ERR_BAD_ARG; C > UMR_ST_MAX_CHANNELS or H * W >= UMR_ST_MAX_COUNT
 * -> UMR_ERR_TOO_LARGE. */
int umr_st_average_mean(const float* acc, int32_t C, int32_t H, int32_t W, int64_t count, float* avg_prob, void* stream);

/* The labelling pass over avg_prob [H,W,C].  argmax below is over the C channels, the first NaN if any, else the first
 * largest value; a mode is the most frequent label, ties to the smallest.
 *   label_image [H,W] uint8 = argmax avg_prob[y, x];
 *   texel_labels [F,T2] = argmax of avg_prob sampled (as umr_st_average_add samples) at uv_sampler [F_src,T2,2] of face
 *   f, or of face f - num_sym_faces for f >= F_src, F = F_src + num_sym_faces;
 *   face_labels [F] = the mode of the face's T2 texel labels;
 *   vertex_labels [V] = the mode of the labels of the faces with a corner at the vertex, each face once, -1 for none.
 * vertex_rowptr [V+1] and vertex_corners are the vertex -> face-corner table of faces [F,3] (corner f * 3 + j, ascending
 * in each row), as ops.device_incidence builds it.  Three launches.  Refused before any device work: a NULL buffer, one
 * not aligned to its element (uv_sampler: 8 bytes), H, W, C, F_src, T2 or V <= 0, num_sym_faces outside [0, F_src] ->
 * UMR_ERR_BAD_ARG; C > UMR_ST_MAX_CHANNELS, H * W, 3 F, F * T2 or V >= UMR_ST_MAX_COUNT -> UMR_ERR_TOO_LARGE. */
int umr_st_labels(const float* avg_prob, int32_t H, int32_t W, int32_t C, const float* uv_sampler, int32_t F_src, int32_t T2,
                  int32_t num_sym_faces, const int32_t* vertex_rowptr, const int32_t* vertex_corners, int32_t V,
                  uint8_t* label_image, int32_t* texel_labels, int32_t* face_labels, int32_t* vertex_labels, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* UMR_SEMANTIC_TEMPLATE_H_ */
