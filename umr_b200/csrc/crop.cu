// crop.cu -- the pixel half of the training loader (data/base.py:88-186 `forward_img`: crop with background padding,
// cv2.resize INTER_LINEAR in float64, mirror) and of `set_input` (experiments/train_s2.py:166-192: ResNet Normalize, the
// SCOPS maps' mask product and per-channel max normalisation), for a whole batch per call.  Compiled with -fmad=false: the
// resize is a twin of cv2's float64 arithmetic, restated bit for bit by tests/crop_oracle.py.  Contract: DESIGN.md §19.
//
//   k_crop_resize  one CTA per (image, output row): the two source rows and the row weight, then per output pixel the two
//                  source columns and weights of its (mirrored) column, the frame samples from the uint8 window (1.0 /
//                  0.0 outside it), the horizontal then vertical pass in double, one rounding to float32; writes imgs,
//                  input_imgs and masks, and the row of the mirrored part maps.
//   k_part_segs    one CTA per (image, part channel): the NaN-propagating max of q = part * mask over the map by a
//                  fixed shared-memory tree, then q / max.  No atomics on any output.
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "umr_b200.h"

namespace umr {

constexpr int CROP_THREADS = 256;
constexpr int SEGS_THREADS = 512;

// One output index's source pair and weights along an axis of a frame of side L (cv2 resize.cpp, INTER_LINEAR)
struct Tap {
    int i0, i1;
    float w0, w1;
};

__device__ __forceinline__ Tap linear_tap(int d, double scale, int L) {
    float f = __double2float_rn((d + 0.5) * scale - 0.5);
    int s = (int)floorf(f);
    f -= (float)s;
    if (s < 0) s = 0, f = 0.f;
    if (s >= L - 1) s = L - 1, f = 0.f;
    return {s, min(s + 1, L - 1), 1.f - f, f};
}

struct Window {
    const uint8_t* img;   // [h,w,ch]
    const uint8_t* mask;  // [h,w]
    int h, w, ch, x0, y0;
};

// The crop frame's image sample of channel c at frame pixel (x, y): u8 / 255 inside the window, 1 outside
__device__ __forceinline__ double frame_img(const Window& win, int x, int y, int c) {
    const int wx = x - win.x0, wy = y - win.y0;
    if ((unsigned)wx >= (unsigned)win.w || (unsigned)wy >= (unsigned)win.h) return 1.0;
    const size_t k = ((size_t)wy * win.w + wx) * win.ch + (win.ch == 3 ? c : 0);
    return (double)__ldg(win.img + k) / 255.0;
}

// The crop frame's mask sample: the raw value inside the window, 0 outside
__device__ __forceinline__ double frame_mask(const Window& win, int x, int y) {
    const int wx = x - win.x0, wy = y - win.y0;
    if ((unsigned)wx >= (unsigned)win.w || (unsigned)wy >= (unsigned)win.h) return 0.0;
    return (double)__ldg(win.mask + (size_t)wy * win.w + wx);
}

// horizontal pass over frame rows y0 and y1, then the vertical pass, in double; one rounding to float32
template <typename F>
__device__ __forceinline__ float bilinear(F sample, const Tap& tx, const Tap& ty) {
    const double a0 = tx.w0, a1 = tx.w1, b0 = ty.w0, b1 = ty.w1;
    const double r0 = sample(tx.i0, ty.i0) * a0 + sample(tx.i1, ty.i0) * a1;
    const double r1 = sample(tx.i0, ty.i1) * a0 + sample(tx.i1, ty.i1) * a1;
    return __double2float_rn(r0 * b0 + r1 * b1);
}

__global__ void __launch_bounds__(CROP_THREADS) k_crop_resize(const uint8_t* __restrict__ pack, const int32_t* __restrict__ table,
                                                              int S, const float* __restrict__ part_in, int C,
                                                              float* __restrict__ imgs, float* __restrict__ input_imgs,
                                                              float* __restrict__ masks, float* __restrict__ part_out) {
    const int b = blockIdx.x / S, y = blockIdx.x - b * S;
    const int32_t* row = table + (size_t)b * UMR_CROP_TABLE_COLS;
    const int64_t off = __ldg(row + UMR_CROP_OFFSET);
    Window win;
    win.h = __ldg(row + UMR_CROP_H);
    win.w = __ldg(row + UMR_CROP_W);
    win.ch = __ldg(row + UMR_CROP_CH);
    win.x0 = __ldg(row + UMR_CROP_X0);
    win.y0 = __ldg(row + UMR_CROP_Y0);
    win.img = pack + off;
    win.mask = pack + off + (int64_t)win.h * win.w * win.ch;
    const int L = __ldg(row + UMR_CROP_L);
    const bool flip = __ldg(row + UMR_CROP_FLIP) != 0;
    // cv2: inv_scale = dsize / ssize, scale = 1 / inv_scale, both in double
    const double scale = 1.0 / ((double)S / (double)L);
    const Tap ty = linear_tap(y, scale, L);
    // torchvision Normalize's ImageNet constants, each the float32 nearest the Python double
    const float mean[3] = {(float)0.485, (float)0.456, (float)0.406};
    const float stdv[3] = {(float)0.229, (float)0.224, (float)0.225};
    const size_t plane = (size_t)S * S, pix = (size_t)y * S;
    for (int x = threadIdx.x; x < S; x += CROP_THREADS) {
        const Tap tx = linear_tap(flip ? S - 1 - x : x, scale, L);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float v = bilinear([&](int fx, int fy) { return frame_img(win, fx, fy, c); }, tx, ty);
            const size_t o = ((size_t)b * 3 + c) * plane + pix + x;
            imgs[o] = v;
            input_imgs[o] = __fdiv_rn(__fsub_rn(v, mean[c]), stdv[c]);
        }
        masks[(size_t)b * plane + pix + x] = bilinear([&](int fx, int fy) { return frame_mask(win, fx, fy); }, tx, ty);
    }
    if (part_in) {
        const size_t base = ((size_t)b * plane + pix) * C;
        for (int j = threadIdx.x; j < S * C; j += CROP_THREADS) {
            const int x = j / C, c = j - x * C;
            part_out[base + j] = __ldg(part_in + base + (flip ? (size_t)(S - 1 - x) * C + c : (size_t)j));
        }
    }
}

// torch.max's order: a NaN wins, else the larger
__device__ __forceinline__ float nan_max(float a, float b) {
    if (isnan(a)) return a;
    if (isnan(b)) return b;
    return b > a ? b : a;
}

__global__ void __launch_bounds__(SEGS_THREADS) k_part_segs(const float* __restrict__ part, const float* __restrict__ masks,
                                                            int S, int C, float* __restrict__ part_segs) {
    __shared__ float red[SEGS_THREADS];
    const int b = blockIdx.x / C, c = blockIdx.x - b * C;
    const int N = S * S;
    const float* p = part + (size_t)b * N * C + c;
    const float* mk = masks + (size_t)b * N;
    float m = -INFINITY;
    for (int i = threadIdx.x; i < N; i += SEGS_THREADS) m = nan_max(m, __fmul_rn(__ldg(p + (size_t)i * C), __ldg(mk + i)));
    red[threadIdx.x] = m;
#pragma unroll
    for (int o = SEGS_THREADS / 2; o > 0; o >>= 1) {
        __syncthreads();
        if (threadIdx.x < o) red[threadIdx.x] = nan_max(red[threadIdx.x], red[threadIdx.x + o]);
    }
    __syncthreads();
    const float k = red[0];
    float* out = part_segs + ((size_t)b * C + c) * N;
    for (int i = threadIdx.x; i < N; i += SEGS_THREADS)
        out[i] = __fdiv_rn(__fmul_rn(__ldg(p + (size_t)i * C), __ldg(mk + i)), k);
}

static inline bool misaligned4(const void* p) { return ((uintptr_t)p & 3u) != 0; }

}  // namespace umr

using namespace umr;

extern "C" int umr_crop_batch(const uint8_t* pack, int64_t pack_bytes, const int32_t* table_dev, const int32_t* table_host,
                              int32_t B, int32_t S, const float* part_prob, int32_t C, float* imgs, float* input_imgs,
                              float* masks, float* part_prob_out, float* part_segs, void* stream_) {
    if (!pack || !table_dev || !table_host || !imgs || !input_imgs || !masks || B <= 0 || S <= 0 || pack_bytes <= 0)
        return UMR_ERR_BAD_ARG;
    if (misaligned4(table_dev) || misaligned4(imgs) || misaligned4(input_imgs) || misaligned4(masks)) return UMR_ERR_BAD_ARG;
    if (part_prob && (!part_prob_out || !part_segs || C < 1 || C > UMR_CROP_MAX_CHANNELS || misaligned4(part_prob) ||
                      misaligned4(part_prob_out) || misaligned4(part_segs)))
        return UMR_ERR_BAD_ARG;
    bool too_large = S > UMR_CROP_MAX_SIDE || (int64_t)B * S > INT32_MAX;
    for (int b = 0; b < B; ++b) {
        const int32_t* r = table_host + (size_t)b * UMR_CROP_TABLE_COLS;
        const int64_t off = r[UMR_CROP_OFFSET], h = r[UMR_CROP_H], w = r[UMR_CROP_W], ch = r[UMR_CROP_CH];
        const int64_t x0 = r[UMR_CROP_X0], y0 = r[UMR_CROP_Y0], L = r[UMR_CROP_L], flip = r[UMR_CROP_FLIP];
        if (h <= 0 || w <= 0 || L <= 0 || x0 < 0 || y0 < 0 || x0 + w > L || y0 + h > L || (ch != 1 && ch != 3) || off < 0 ||
            (flip != 0 && flip != 1))
            return UMR_ERR_BAD_ARG;
        if (L > UMR_CROP_MAX_FRAME) {
            too_large = true;   // refused below; h * w may not fit the byte count
            continue;
        }
        if (off + h * w * (ch + 1) > pack_bytes) return UMR_ERR_BAD_ARG;
    }
    if (too_large) return UMR_ERR_TOO_LARGE;
    const cudaStream_t stream = (cudaStream_t)stream_;
    launch(k_crop_resize, (unsigned)(B * S), CROP_THREADS, 0, stream, pack, table_dev, S, part_prob, C, imgs, input_imgs, masks,
           part_prob_out);
    if (part_prob) launch(k_part_segs, (unsigned)(B * C), SEGS_THREADS, 0, stream, part_prob_out, masks, S, C, part_segs);
    return (int)cudaGetLastError();
}
