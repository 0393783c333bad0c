// kp_transfer.cu -- keypoint transfer between image pairs, the two modes of UMR's keypoint evaluation
// (experiments/test_kp.py:125-193, utils/kp_utils.py:13-69), for P pairs in one launch.  Compiled with -fmad=false: the
// heat-map and grid samples are the sampler's torch-1.1 arithmetic (losses.cuh `bilinear_tap` / `bilinear_value`) with
// every product and sum rounded once, as tests/kp_transfer_oracle.py restates it.  Float32, no atomics, no host
// synchronisation.  Contract and deviations: DESIGN.md §16.
//
//   k_kp_flow  one warp per (pair, keypoint): the keypoint's Gaussian heat map (never materialised: a lookup in the
//              shared table `gauss` inside its window) sampled at every face's T^2 source-flow points, the T^2 mean per
//              face, the first face of largest mean, then the identity grid sampled at that face's target flow
//   k_kp_cam   one warp per (pair, keypoint): the nearest projected source vertex to the keypoint, then the nearest
//              foreground pixel (mask != 0) of the target to that vertex's target projection, in k_chamfer_nn's
//              distance and tie order
#include <cuda_runtime.h>
#include <stdint.h>

#include <climits>

#include "common.cuh"
#include "losses.cuh"
#include "umr_b200.h"

namespace umr {

constexpr int KP_WARPS = 8;                 // (pair, keypoint) items per CTA
constexpr float KP_HEATMAP_SCALE = 256.f;   // test_kp.py:146: (kp + 1) / 2 * 256 whatever the image size
constexpr int KP_MAX_SIGMA = 18;            // (6 sigma + 1)^2 floats of table within 48 KB of shared memory
constexpr int64_t KP_MAX_COUNT = 1LL << 30;  // P * K, F * T^2, V and S^2: int indices with room for the lane stride

__global__ void __launch_bounds__(KP_WARPS * 32) k_kp_flow(const float2* __restrict__ kps, const float2* __restrict__ flow_src,
                                                          const float2* __restrict__ flow_tgt, const float* __restrict__ gauss,
                                                          const float* __restrict__ grid, float2* __restrict__ out, int P,
                                                          int K, int F, int T2, int S, int sigma) {
    extern __shared__ float s_gauss[];
    const int n = 6 * sigma + 1;
    for (int i = threadIdx.x; i < n * n; i += blockDim.x) s_gauss[i] = __ldg(gauss + i);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * KP_WARPS + (threadIdx.x >> 5);
    if (item >= P * K) return;
    const int p = item / K;

    // draw_labelmap (kp_utils.py:42-69): window corners ul = int(pt - 3 sigma), br = int(pt + 3 sigma + 1), truncated
    // toward zero; an all-zero map when ul >= S or br < 0 on either axis, i.e. when a >= S or b <= -1 before the
    // truncation (also for a NaN keypoint, which the reference cannot convert to int).  Heat-map pixel (x, y) is
    // gauss[(y - ul1) * n + (x - ul0)] on [max(0, ul), min(br, S, ul + n)) per axis, 0 elsewhere.  br - ul is n = 6 sigma
    // + 1 in exact arithmetic, but pt + 3 sigma can round up across an integer in float32 and make it n + 1 (e.g.
    // sigma = 3, kp = -0.06250006: pt = 119.99999, ul = 110, br = 130); the reference's slice assignment then fails on
    // the shape mismatch.  The window is clamped to the table, so that extra column / row is 0 and nothing is read past
    // the table.
    const float2 kp = __ldg(kps + item);
    const float pt[2] = {((kp.x + 1.f) / 2.f) * KP_HEATMAP_SCALE, ((kp.y + 1.f) / 2.f) * KP_HEATMAP_SCALE};
    int ul[2] = {0, 0}, lo[2] = {0, 0}, hi[2] = {0, 0};
    bool drawn = true;
#pragma unroll
    for (int d = 0; d < 2; ++d) {
        const float a = pt[d] - (float)(3 * sigma), b = (pt[d] + (float)(3 * sigma)) + 1.f;
        drawn = drawn && a < (float)S && b > -1.f;
    }
    if (drawn) {
#pragma unroll
        for (int d = 0; d < 2; ++d) {
            ul[d] = (int)(pt[d] - (float)(3 * sigma));
            const int br = (int)((pt[d] + (float)(3 * sigma)) + 1.f);
            lo[d] = max(0, ul[d]);
            hi[d] = min(min(br, S), ul[d] + n);
        }
    }
    auto heat = [&](int x, int y) -> float {
        return (x >= lo[0] && x < hi[0] && y >= lo[1] && y < hi[1]) ? s_gauss[(y - ul[1]) * n + (x - ul[0])] : 0.f;
    };

    // k2face: the T^2 mean of the heat map sampled at each face's source flow; the first face of largest mean
    // (torch.max's choice, NaN included: ph_beats)
    float best = -INFINITY;
    int bf = INT_MAX;
    const float2* fs = flow_src + (size_t)p * F * T2;
    for (int f = lane; f < F; f += 32) {
        float sum = 0.f;
        for (int t = 0; t < T2; ++t) sum += bilinear_value(bilinear_tap<float>(__ldg(fs + (size_t)f * T2 + t), S, S), heat);
        const float mean = sum / (float)T2;
        if (ph_beats(mean, f, best, bf)) { best = mean; bf = f; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bf, o);
        if (ph_beats(ob, oi, best, bf)) { best = ob; bf = oi; }
    }
    if (lane != 0) return;

    // p2face of the chosen face: the identity grid (channel 0 = grid[x], channel 1 = grid[y]) sampled at its target
    // flow, T^2 mean
    const float2* ft = flow_tgt + ((size_t)p * F + bf) * T2;
    float sx = 0.f, sy = 0.f;
    for (int t = 0; t < T2; ++t) {
        const BilinearTap<float> tap = bilinear_tap<float>(__ldg(ft + t), S, S);
        sx += bilinear_value(tap, [&](int x, int) { return __ldg(grid + x); });
        sy += bilinear_value(tap, [&](int, int y) { return __ldg(grid + y); });
    }
    out[item] = make_float2(sx / (float)T2, sy / (float)T2);
}

__global__ void __launch_bounds__(KP_WARPS * 32) k_kp_cam(const float2* __restrict__ kps, const float2* __restrict__ proj_src,
                                                         const float2* __restrict__ proj_tgt, const float* __restrict__ mask,
                                                         const float* __restrict__ grid, float2* __restrict__ out, int P, int K,
                                                         int V, int S) {
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * KP_WARPS + (threadIdx.x >> 5);
    if (item >= P * K) return;
    const int p = item / K;
    // the keypoint's nearest projected source vertex (test_kp.py:188)
    const float2 kp = __ldg(kps + item);
    const float qv[2] = {kp.x, kp.y};
    const float qq = chamfer_sqnorm(qv);
    float best = INFINITY;
    int bi = INT_MAX;
    const float2* ps = proj_src + (size_t)p * V;
    for (int j = lane; j < V; j += 32) {
        const float2 v = __ldg(ps + j);
        const float kv[2] = {v.x, v.y};
        const float d = chamfer_dist(qv, qq, kv);
        if (d < best) { best = d; bi = j; }
    }
    warp_argmin(best, bi);
    // that vertex's target projection against every foreground pixel (test_kp.py:177-180): the pixel's index in
    // `nonzero` order is its flat index, so the lowest flat index wins ties
    int bp = INT_MAX;
    if (bi != INT_MAX) {
        const float2 v = __ldg(proj_tgt + (size_t)p * V + bi);
        const float tv[2] = {v.x, v.y};
        const float tt = chamfer_sqnorm(tv);
        const float* m = mask + (size_t)p * S * S;
        best = INFINITY;
        for (int i = lane; i < S * S; i += 32) {
            if (__ldg(m + i) == 0.f) continue;
            const int y = i / S, x = i - y * S;
            const float kv[2] = {__ldg(grid + x), __ldg(grid + y)};
            const float d = chamfer_dist(tv, tt, kv);
            if (d < best) { best = d; bp = i; }
        }
        warp_argmin(best, bp);
    }
    if (lane != 0) return;
    // no finite vertex distance or no foreground pixel (an empty mask): NaN, where the reference fails
    out[item] = bp == INT_MAX ? make_float2(NAN, NAN) : make_float2(__ldg(grid + bp % S), __ldg(grid + bp / S));
}

static inline bool f2_misaligned(const void* p) { return ((uintptr_t)p & 7) != 0; }
static inline bool f_misaligned(const void* p) { return ((uintptr_t)p & 3) != 0; }

}  // namespace umr

using namespace umr;

extern "C" int umr_kp_transfer_flow(const float* kps, const float* flow_src, const float* flow_tgt, const float* gauss,
                                    const float* grid, float* out, int32_t P, int32_t K, int32_t F, int32_t T2, int32_t S,
                                    int32_t sigma, void* stream_) {
    if (!kps || !flow_src || !flow_tgt || !gauss || !grid || !out || P <= 0 || K <= 0 || F <= 0 || T2 <= 0 || S <= 0 ||
        sigma <= 0 || f2_misaligned(kps) || f2_misaligned(flow_src) || f2_misaligned(flow_tgt) || f2_misaligned(out) ||
        f_misaligned(gauss) || f_misaligned(grid))
        return UMR_ERR_BAD_ARG;
    if (sigma > KP_MAX_SIGMA || (int64_t)P * K >= KP_MAX_COUNT || (int64_t)F * T2 >= KP_MAX_COUNT) return UMR_ERR_TOO_LARGE;
    const int n = 6 * sigma + 1;
    const int items = P * K;
    launch(k_kp_flow, (unsigned)((items + KP_WARPS - 1) / KP_WARPS), KP_WARPS * 32, (size_t)n * n * sizeof(float),
           (cudaStream_t)stream_, reinterpret_cast<const float2*>(kps), reinterpret_cast<const float2*>(flow_src),
           reinterpret_cast<const float2*>(flow_tgt), gauss, grid, reinterpret_cast<float2*>(out), P, K, F, T2, S, sigma);
    return (int)cudaGetLastError();
}

extern "C" int umr_kp_transfer_cam(const float* kps, const float* proj_src, const float* proj_tgt, const float* mask_tgt,
                                   const float* grid, float* out, int32_t P, int32_t K, int32_t V, int32_t S, void* stream_) {
    if (!kps || !proj_src || !proj_tgt || !mask_tgt || !grid || !out || P <= 0 || K <= 0 || V <= 0 || S <= 0 ||
        f2_misaligned(kps) || f2_misaligned(proj_src) || f2_misaligned(proj_tgt) || f2_misaligned(out) ||
        f_misaligned(mask_tgt) || f_misaligned(grid))
        return UMR_ERR_BAD_ARG;
    if ((int64_t)P * K >= KP_MAX_COUNT || V >= KP_MAX_COUNT || (int64_t)S * S >= KP_MAX_COUNT) return UMR_ERR_TOO_LARGE;
    const int items = P * K;
    launch(k_kp_cam, (unsigned)((items + KP_WARPS - 1) / KP_WARPS), KP_WARPS * 32, 0, (cudaStream_t)stream_,
           reinterpret_cast<const float2*>(kps), reinterpret_cast<const float2*>(proj_src),
           reinterpret_cast<const float2*>(proj_tgt), mask_tgt, grid, reinterpret_cast<float2*>(out), P, K, V, S);
    return (int)cudaGetLastError();
}
