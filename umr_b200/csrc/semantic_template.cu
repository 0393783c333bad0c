// semantic_template.cu -- the SCOPS semantic template UMR builds between its two training stages
// (experiments/avg_uv.py:203-293 `compute_uv`): the dataset-wide average of the k SCOPS part maps nearest the exemplar in
// UV space, and the per-texel, per-face and per-vertex part labels of the template mesh.  Compiled with -fmad=false: the
// UV samples are the sampler's torch-1.1 arithmetic (losses.cuh `bilinear_tap` / `bilinear_value`) with every product and
// sum rounded once, as tests/semantic_template_oracle.py restates it.  Float32, no atomics, no host synchronisation.
// Contract, tie rules and deviations: DESIGN.md §18.
//
//   k_st_dist        grid (pixel tiles, image): each thread sums (sample - exemplar)^2 over its ST_PIX pixels and every
//                    channel, a fixed shared-memory tree adds the CTA's partials; one partial per (image, tile)
//   k_st_accumulate  one pixel per thread: every CTA finishes the B distances (serially over tiles) and ranks them by
//                    (distance, image index), NaN last; then at its pixels sums the k selected images' samples in
//                    selection order and adds the sum to the accumulator.  CTA 0 also writes the distances and selection.
//   k_st_mean        one pixel per thread: avg_prob[y, x, c] = acc[c, y, x] / count
//   k_st_label_image one pixel per thread: the argmax over channels of avg_prob
//   k_st_face_labels one warp per face: avg_prob sampled at the face's T^2 points, the argmax per texel, the mode per face
//   k_st_vertex_labels one warp per vertex: the mode of its incident faces' labels over the vertex -> face-corner table
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "losses.cuh"
#include "umr_b200.h"

namespace umr {

constexpr int ST_THREADS = 256;
constexpr int ST_PIX = 4;                        // pixels per thread of k_st_dist
constexpr int ST_TILE = ST_THREADS * ST_PIX;     // pixels per k_st_dist CTA
constexpr int ST_WARPS = ST_THREADS / 32;        // faces / vertices per labelling CTA

__device__ __forceinline__ float2 uv_at(const float* __restrict__ uv, int b, int N, int p) {
    const float* u = uv + (size_t)b * 2 * N;
    return make_float2(__ldg(u + p), __ldg(u + N + p));
}

// Image b's channel c sampled at its UV pixel p: part_segs [B,C,S,S] at uvimage_pred[b, :, p]
__device__ __forceinline__ float sample_part(const float* __restrict__ segs, const BilinearTap<float>& tap, int b, int c,
                                             int C, int S) {
    const float* img = segs + ((size_t)b * C + c) * S * S;
    return bilinear_value(tap, [&](int x, int y) { return __ldg(img + (size_t)y * S + x); });
}

__global__ void __launch_bounds__(ST_THREADS) k_st_dist(const float* __restrict__ segs, const float* __restrict__ uv,
                                                       const float* __restrict__ exemplar, int C, int S, int N,
                                                       float* __restrict__ partials) {
    __shared__ float red[ST_THREADS];
    const int t = threadIdx.x, tile = blockIdx.x, b = blockIdx.y;
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < ST_PIX; ++i) {
        const int p = tile * ST_TILE + i * ST_THREADS + t;
        if (p >= N) break;
        const BilinearTap<float> tap = bilinear_tap<float>(uv_at(uv, b, N, p), S, S);
        for (int c = 0; c < C; ++c) {
            const float d = sample_part(segs, tap, b, c, C, S) - __ldg(exemplar + (size_t)c * N + p);
            acc += d * d;
        }
    }
    red[t] = acc;
#pragma unroll
    for (int off = ST_THREADS / 2; off > 0; off >>= 1) {
        __syncthreads();
        if (t < off) red[t] += red[t + off];
    }
    if (t == 0) partials[(size_t)b * gridDim.x + tile] = red[0];
}

// (d_j, j) before (d_i, i): ascending distance, a NaN after every number, ties and NaNs by image index
__device__ __forceinline__ bool before(float dj, int j, float di, int i) {
    const bool nj = isnan(dj), ni = isnan(di);
    if (nj != ni) return ni;
    if (nj || dj == di) return j < i;
    return dj < di;
}

__global__ void __launch_bounds__(ST_THREADS) k_st_accumulate(const float* __restrict__ segs, const float* __restrict__ uv,
                                                             const float* __restrict__ partials, int B, int C, int S, int N,
                                                             int tiles, int k, float* __restrict__ dist,
                                                             int32_t* __restrict__ selected, float* __restrict__ acc) {
    __shared__ float sd[UMR_ST_MAX_IMAGES];
    __shared__ int sel[UMR_ST_MAX_IMAGES];
    const int t = threadIdx.x;
    for (int b = t; b < B; b += ST_THREADS) {
        const float* pb = partials + (size_t)b * tiles;
        float s = 0.f;
        for (int j = 0; j < tiles; ++j) s += __ldg(pb + j);
        sd[b] = s;
    }
    __syncthreads();
    for (int b = t; b < B; b += ST_THREADS) {
        const float d = sd[b];
        int r = 0;
        for (int j = 0; j < B; ++j) r += before(sd[j], j, d, b);
        if (r < k) sel[r] = b;
        if (blockIdx.x == 0) {
            dist[b] = d;
            if (r < k) selected[r] = b;
        }
    }
    __syncthreads();
    const int p = blockIdx.x * ST_THREADS + t;
    if (p >= N) return;
    for (int c = 0; c < C; ++c) {
        float s = 0.f;
        for (int r = 0; r < k; ++r) {
            const int b = sel[r];
            s += sample_part(segs, bilinear_tap<float>(uv_at(uv, b, N, p), S, S), b, c, C, S);
        }
        float* a = acc + (size_t)c * N + p;
        *a = *a + s;
    }
}

__global__ void __launch_bounds__(ST_THREADS) k_st_mean(const float* __restrict__ acc, int C, int N, float count,
                                                       float* __restrict__ avg) {
    const int p = blockIdx.x * ST_THREADS + threadIdx.x;
    if (p >= N) return;
    for (int c = 0; c < C; ++c) avg[(size_t)p * C + c] = __ldg(acc + (size_t)c * N + p) / count;
}

// Argmax over C values v(0..C-1): the first NaN if there is one, else the first largest value (torch.argmax's rule)
template <typename Value>
__device__ __forceinline__ int argmax_channels(int C, Value v) {
    float best = v(0);
    if (isnan(best)) return 0;
    int bi = 0;
    for (int c = 1; c < C; ++c) {
        const float x = v(c);
        if (isnan(x)) return c;
        if (x > best) {
            best = x;
            bi = c;
        }
    }
    return bi;
}

__global__ void __launch_bounds__(ST_THREADS) k_st_label_image(const float* __restrict__ avg, int C, int N,
                                                              uint8_t* __restrict__ label_image) {
    const int p = blockIdx.x * ST_THREADS + threadIdx.x;
    if (p >= N) return;
    const float* a = avg + (size_t)p * C;
    label_image[p] = (uint8_t)argmax_channels(C, [&](int c) { return __ldg(a + c); });
}

// Warp-wide label counts: lane c < C adds how many lanes hold label c (label < 0: none)
__device__ __forceinline__ int count_labels(int label, int C, int lane, int count) {
    for (int c = 0; c < C; ++c) {
        const unsigned m = __ballot_sync(0xffffffffu, label == c);
        if (lane == c) count += __popc(m);
    }
    return count;
}

// The mode of the counted labels, ties to the smallest label; -1 when nothing was counted.  Every lane gets it.
__device__ __forceinline__ int warp_mode(int count, int lane) {
    unsigned long long key = ((unsigned long long)count << 5) | (unsigned)(31 - lane);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const unsigned long long o = __shfl_xor_sync(0xffffffffu, key, off);
        key = o > key ? o : key;
    }
    return (key >> 5) == 0 ? -1 : 31 - (int)(key & 31u);
}

__global__ void __launch_bounds__(ST_THREADS) k_st_face_labels(const float* __restrict__ avg, int H, int W, int C,
                                                              const float2* __restrict__ uv_sampler, int F_src, int T2,
                                                              int num_sym, int32_t* __restrict__ texel_labels,
                                                              int32_t* __restrict__ face_labels) {
    const int lane = threadIdx.x & 31;
    const int f = blockIdx.x * ST_WARPS + (threadIdx.x >> 5);
    if (f >= F_src + num_sym) return;
    const int src = f < F_src ? f : f - num_sym;     // the copies of the last num_sym faces (avg_uv.py:260-261)
    int count = 0;
    for (int base = 0; base < T2; base += 32) {
        const int t = base + lane;
        int label = -1;
        if (t < T2) {
            const BilinearTap<float> tap = bilinear_tap<float>(__ldg(uv_sampler + (size_t)src * T2 + t), H, W);
            label = argmax_channels(C, [&](int c) {
                return bilinear_value(tap, [&](int x, int y) { return __ldg(avg + ((size_t)y * W + x) * C + c); });
            });
            texel_labels[(size_t)f * T2 + t] = label;
        }
        count = count_labels(label, C, lane, count);
    }
    const int mode = warp_mode(count, lane);
    if (lane == 0) face_labels[f] = mode;
}

__global__ void __launch_bounds__(ST_THREADS) k_st_vertex_labels(const int32_t* __restrict__ rowptr,
                                                                const int32_t* __restrict__ corners,
                                                                const int32_t* __restrict__ face_labels, int V, int C,
                                                                int32_t* __restrict__ vertex_labels) {
    const int lane = threadIdx.x & 31;
    const int v = blockIdx.x * ST_WARPS + (threadIdx.x >> 5);
    if (v >= V) return;
    const int begin = __ldg(rowptr + v), end = __ldg(rowptr + v + 1);
    int count = 0;
    for (int base = begin; base < end; base += 32) {
        const int i = base + lane;
        int label = -1;
        if (i < end) {
            // corners of one face are adjacent in the row (ascending positions): a face that repeats the vertex counts once
            const int f = __ldg(corners + i) / 3;
            if (i == begin || __ldg(corners + i - 1) / 3 != f) label = __ldg(face_labels + f);
        }
        count = count_labels(label, C, lane, count);
    }
    const int mode = warp_mode(count, lane);
    if (lane == 0) vertex_labels[v] = mode;
}

static inline bool misaligned(const void* p, size_t a) { return ((uintptr_t)p % a) != 0; }
static inline unsigned blocks(int64_t n, int per) { return (unsigned)((n + per - 1) / per); }
static inline int dist_tiles(int64_t N) { return (int)((N + ST_TILE - 1) / ST_TILE); }

}  // namespace umr

using namespace umr;

extern "C" size_t umr_st_average_workspace_bytes(int32_t B, int32_t H, int32_t W) {
    if (B <= 0 || H <= 0 || W <= 0 || B > UMR_ST_MAX_IMAGES || (int64_t)H * W >= UMR_ST_MAX_COUNT) return 0;
    return (size_t)B * dist_tiles((int64_t)H * W) * sizeof(float);
}

extern "C" int umr_st_average_add(const float* part_segs, const float* uvimage_pred, const float* exemplar, int32_t B,
                                  int32_t C, int32_t S, int32_t H, int32_t W, int32_t k, void* workspace, float* dist,
                                  int32_t* selected, float* acc, void* stream_) {
    if (!part_segs || !uvimage_pred || !exemplar || !workspace || !dist || !selected || !acc || B <= 0 || C <= 0 ||
        S <= 0 || H <= 0 || W <= 0 || k <= 0 || k > B)
        return UMR_ERR_BAD_ARG;
    if (misaligned(part_segs, 4) || misaligned(uvimage_pred, 4) || misaligned(exemplar, 4) || misaligned(workspace, 4) ||
        misaligned(dist, 4) || misaligned(selected, 4) || misaligned(acc, 4))
        return UMR_ERR_BAD_ARG;
    const int64_t N = (int64_t)H * W;
    if (B > UMR_ST_MAX_IMAGES || C > UMR_ST_MAX_CHANNELS || (int64_t)S * S >= UMR_ST_MAX_COUNT || N >= UMR_ST_MAX_COUNT)
        return UMR_ERR_TOO_LARGE;
    const cudaStream_t stream = (cudaStream_t)stream_;
    const int tiles = dist_tiles(N);
    float* partials = static_cast<float*>(workspace);
    launch(k_st_dist, dim3(tiles, B), ST_THREADS, 0, stream, part_segs, uvimage_pred, exemplar, (int)C, (int)S, (int)N,
           partials);
    launch(k_st_accumulate, blocks(N, ST_THREADS), ST_THREADS, 0, stream, part_segs, uvimage_pred,
           static_cast<const float*>(partials), (int)B, (int)C, (int)S, (int)N, tiles, (int)k, dist, selected, acc);
    return (int)cudaGetLastError();
}

extern "C" int umr_st_average_mean(const float* acc, int32_t C, int32_t H, int32_t W, int64_t count, float* avg_prob,
                                   void* stream_) {
    if (!acc || !avg_prob || C <= 0 || H <= 0 || W <= 0 || count <= 0 || misaligned(acc, 4) || misaligned(avg_prob, 4))
        return UMR_ERR_BAD_ARG;
    const int64_t N = (int64_t)H * W;
    if (C > UMR_ST_MAX_CHANNELS || N >= UMR_ST_MAX_COUNT) return UMR_ERR_TOO_LARGE;
    launch(k_st_mean, blocks(N, ST_THREADS), ST_THREADS, 0, (cudaStream_t)stream_, acc, (int)C, (int)N, (float)count,
           avg_prob);
    return (int)cudaGetLastError();
}

extern "C" int umr_st_labels(const float* avg_prob, int32_t H, int32_t W, int32_t C, const float* uv_sampler,
                             int32_t F_src, int32_t T2, int32_t num_sym_faces, const int32_t* vertex_rowptr,
                             const int32_t* vertex_corners, int32_t V, uint8_t* label_image, int32_t* texel_labels,
                             int32_t* face_labels, int32_t* vertex_labels, void* stream_) {
    if (!avg_prob || !uv_sampler || !vertex_rowptr || !vertex_corners || !label_image || !texel_labels || !face_labels ||
        !vertex_labels || H <= 0 || W <= 0 || C <= 0 || F_src <= 0 || T2 <= 0 || V <= 0 || num_sym_faces < 0 ||
        num_sym_faces > F_src)
        return UMR_ERR_BAD_ARG;
    if (misaligned(avg_prob, 4) || misaligned(uv_sampler, 8) || misaligned(vertex_rowptr, 4) ||
        misaligned(vertex_corners, 4) || misaligned(texel_labels, 4) || misaligned(face_labels, 4) ||
        misaligned(vertex_labels, 4))
        return UMR_ERR_BAD_ARG;
    const int64_t N = (int64_t)H * W, F = (int64_t)F_src + num_sym_faces;
    if (C > UMR_ST_MAX_CHANNELS || N >= UMR_ST_MAX_COUNT || 3 * F >= UMR_ST_MAX_COUNT || F * T2 >= UMR_ST_MAX_COUNT ||
        V >= UMR_ST_MAX_COUNT)
        return UMR_ERR_TOO_LARGE;
    const cudaStream_t stream = (cudaStream_t)stream_;
    launch(k_st_label_image, blocks(N, ST_THREADS), ST_THREADS, 0, stream, avg_prob, (int)C, (int)N, label_image);
    launch(k_st_face_labels, blocks(F, ST_WARPS), ST_THREADS, 0, stream, avg_prob, (int)H, (int)W, (int)C,
           reinterpret_cast<const float2*>(uv_sampler), (int)F_src, (int)T2, (int)num_sym_faces, texel_labels,
           face_labels);
    launch(k_st_vertex_labels, blocks(V, ST_WARPS), ST_THREADS, 0, stream, vertex_rowptr, vertex_corners,
           static_cast<const int32_t*>(face_labels), (int)V, (int)C, vertex_labels);
    return (int)cudaGetLastError();
}
