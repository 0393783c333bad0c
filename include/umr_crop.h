/* umr_crop.h -- the pixel half of the training loader's `forward_img` (data/base.py:88-186: crop, cv2.resize, mirror)
 * and `set_input`'s two normalisations (experiments/train_s2.py:166-192), for a whole batch per call.  Part of the C ABI
 * of libumr_b200.so and included by umr_b200.h, whose conventions hold here (caller-allocated device buffers, work
 * enqueued on `stream`, 0 / positive cudaError_t / negative UMR_ERR_* return).  Declared apart from umr_b200.h's own
 * list and bound by _lib.CROP_EXPORTS, with its refusals tested beside it.  No atomics (bitwise reproducible), no host
 * synchronisation.  Contract: DESIGN.md §19. */
#ifndef UMR_CROP_H_
#define UMR_CROP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UMR_CROP_MAX_SIDE 4096        /* S: output side */
#define UMR_CROP_MAX_FRAME 65536      /* L: crop frame side */
#define UMR_CROP_MAX_CHANNELS 8       /* C: part channels */

/* The per-image table, UMR_CROP_TABLE_COLS int32 per image, in this column order */
#define UMR_CROP_OFFSET 0    /* byte offset of the window in the pack */
#define UMR_CROP_H 1         /* window height */
#define UMR_CROP_W 2         /* window width */
#define UMR_CROP_CH 3        /* window channels: 1 (grey, replicated to RGB) or 3 */
#define UMR_CROP_X0 4        /* window position inside the crop frame */
#define UMR_CROP_Y0 5
#define UMR_CROP_L 6         /* crop frame side */
#define UMR_CROP_FLIP 7      /* 1: mirror the outputs */
#define UMR_CROP_TABLE_COLS 8

/* For each image b < B, its table row (offset, h, w, ch, x0, y0, L, flip) places a uint8 window in an L x L crop frame:
 * the pack holds at `offset` the image window [h,w,ch] then the mask window [h,w], both row-major.  The frame pixel is
 * u8 / 255.0 (image, grey replicated) or the raw mask value, in double, inside the window, and 1.0 (image) / 0.0 (mask)
 * outside it.  Each frame is resized L -> S as cv2.resize INTER_LINEAR does float64 (scale = 1 / (S / L); per output
 * index d: fx = (float)((d + 0.5) * scale - 0.5), sx = floor(fx), fx -= sx, clamped to (0, 0) below 0 and (L - 1, 0) from
 * L - 1; float weights (1 - fx, fx); a horizontal then a vertical pass in double), rounded once to float32 and, with
 * flip, mirrored x -> S - 1 - x:
 *   imgs [B,3,S,S], masks [B,S,S];
 *   input_imgs [B,3,S,S] = (imgs - mean) / std, float32, ImageNet's mean / std as float32 (torchvision's Normalize).
 * With part_prob [B,S,S,C] (float32, optional: NULL skips the part maps and part_prob_out / part_segs may be NULL):
 *   part_prob_out [B,S,S,C] = part_prob mirrored as the image is;
 *   part_segs [B,C,S,S] = q / max(q) per (image, channel), q = part_prob_out * masks in float32, max propagating NaN.
 * Two launches with part maps, one without.  table_dev is the device copy of table_host [B,8]; the table is validated
 * from the host copy.  Refused before any device work: a NULL pack, table, imgs, input_imgs or masks, a NULL
 * part_prob_out or part_segs with part_prob, a float buffer not 4-byte aligned, B or S <= 0, C outside [1,
 * UMR_CROP_MAX_CHANNELS] with part_prob, and per image: h, w or L <= 0, x0 or y0 < 0, x0 + w or y0 + h > L, ch not 1 or 3,
 * offset < 0 or the window past pack_bytes, flip not 0 or 1 -> UMR_ERR_BAD_ARG; S > UMR_CROP_MAX_SIDE, L >
 * UMR_CROP_MAX_FRAME or B * S >= 2^31 -> UMR_ERR_TOO_LARGE. */
int umr_crop_batch(const uint8_t* pack, int64_t pack_bytes, const int32_t* table_dev, const int32_t* table_host, int32_t B,
                   int32_t S, const float* part_prob, int32_t C, float* imgs, float* input_imgs, float* masks,
                   float* part_prob_out, float* part_segs, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* UMR_CROP_H_ */
