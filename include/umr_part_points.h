/* umr_part_points.h -- SCOPS part centres and part points of CorrLossChamfer's targets (utils/image.py:143-206, called per
 * image in data/base.py:155-166), for a whole batch per call.  Part of the C ABI of libumr_b200.so and included by
 * umr_b200.h, whose conventions hold here (caller-allocated device buffers, work enqueued on `stream`, 0 / positive
 * cudaError_t / negative UMR_ERR_* return).  Declared apart from umr_b200.h's own list and bound by _lib.PP_EXPORTS, with
 * its refusals tested beside it.  Contract: DESIGN.md §17. */
#ifndef UMR_PART_POINTS_H_
#define UMR_PART_POINTS_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UMR_PART_POINTS_MAX_CHANNELS 8   /* channels (K) one call samples */
#define UMR_PART_POINTS_MAX_DRAWS 1024   /* m = floor(1.5 n) pixels drawn per (image, channel) */
#define UMR_PART_POINTS_MAX_SIDE 4096    /* S: S * S pixel indices stay below 2^24 */

/* status values, one int32 per (image, channel) */
#define UMR_PART_POINTS_OK 0
#define UMR_PART_POINTS_BAD_VALUES 1     /* a NaN, infinite or negative q, or sum(q) zero or not finite */
#define UMR_PART_POINTS_TOO_FEW 2        /* fewer than m pixels with q > 0 */

/* For each image b < B and requested channel k < K (channel ch = channels[k] of part_prob, n = num_samples[k],
 * m = floor(1.5 n)): q = part_prob[b, :, :, ch] * mask[b] on the S x S map, pdf = q / sum(q);
 *   centers[b, k] = (sum pdf * x_map, sum pdf * y_map), x_map[i, j] = j / S * 2 - 1, y_map[i, j] = i / S * 2 - 1;
 *   the m pixels of largest key log(u) / q (u = uniforms[b, k, pixel], in [0, 1); pixels with q = 0 never), ties to the
 *   lower pixel index -- Efraimidis-Spirakis, the sequential without-replacement law of torch.multinomial(pdf, m);
 *   points[k][b] [n,2] = the n of them nearest the centre (squared distance, ascending, ties to the lower pixel index),
 *   pixel k = y * S + x at ((x / 256) * 2 - 1, (y / 256) * 2 - 1) -- the reference's hard-coded 256, right at S = 256;
 *   drawn[k][b] [m] (optional: drawn or drawn[k] may be NULL) = the m drawn pixel indices in ascending order;
 *   status[b, k] = UMR_PART_POINTS_* -- on a non-zero status that channel's centre and points are NaN and its drawn
 *   indices -1.
 * centers_in [B,K,2] (optional, NULL: the computed centres) replaces the centre of the nearest-n selection.
 * dtype UMR_DTYPE_FLOAT32 or UMR_DTYPE_FLOAT64 types part_prob [B,S,S,C], mask [B,S,S], uniforms [B,K,S*S], centers,
 * centers_in and points; each is computed in its own precision.  Two kernel launches, no atomics (bitwise reproducible
 * given the uniforms), no host synchronisation.  channels, num_samples, points and drawn are host arrays of K entries.
 * Refused before any device work: a NULL part_prob, mask, uniforms, channels, num_samples, centers, points, points[k] or
 * status, B, S, C or K <= 0, K > UMR_PART_POINTS_MAX_CHANNELS, a channel outside [0, C), num_samples[k] <= 0, another
 * dtype, a buffer not aligned to its element size (centers, centers_in and points: twice it) -> UMR_ERR_BAD_ARG;
 * floor(1.5 num_samples[k]) > UMR_PART_POINTS_MAX_DRAWS, S > UMR_PART_POINTS_MAX_SIDE or B * K >= 2^31 ->
 * UMR_ERR_TOO_LARGE. */
int umr_part_points(const void* part_prob, const void* mask, const void* uniforms, int32_t B, int32_t S, int32_t C, int32_t K,
                    const int32_t* channels, const int32_t* num_samples, int32_t dtype, const void* centers_in, void* centers,
                    void* const* points, int32_t* const* drawn, int32_t* status, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* UMR_PART_POINTS_H_ */
