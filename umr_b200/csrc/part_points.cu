// part_points.cu -- SCOPS part centres and part points, the targets of CorrLossChamfer, for a whole batch per call
// (utils/image.py:143-206 `prob2center` / `sample_prob`, called four times per image in data/base.py:155-166).  Compiled
// with -fmad=false: the per-pixel keys, coordinates and distances are single IEEE operations, restated bit for bit by
// tests/part_points_oracle.py.  float and double, each in its own precision.  Contract: DESIGN.md §17.
//
//   k_pp_centre  one CTA per (image, channel): q = p * mask; sum(q), the count of q > 0 and the NaN / inf / negative test,
//                then the centre sum(q / sum(q) * coordinate); per-thread strided sums and a fixed shared-memory tree, so
//                the centres are bitwise reproducible.  Writes the centre and the status.
//   k_pp_draw    one CTA per (image, channel): the m = floor(1.5 n) largest keys log(u) / q (Efraimidis-Spirakis) by an
//                8-bit radix select over the recomputed keys (shared-memory histograms of integer counts), the drawn
//                pixels compacted in ascending index order, then each drawn pixel's rank by (squared distance to the
//                centre, pixel index); ranks below n are written.  No atomics on any output.
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "umr_b200.h"

namespace umr {

constexpr int PP_CENTRE_THREADS = 256;
constexpr int PP_DRAW_THREADS = 512;
constexpr int PP_WARPS = PP_DRAW_THREADS / 32;

struct PartPointsArgs {
    int32_t channel[UMR_PART_POINTS_MAX_CHANNELS];
    int32_t n[UMR_PART_POINTS_MAX_CHANNELS];
    void* points[UMR_PART_POINTS_MAX_CHANNELS];
    int32_t* drawn[UMR_PART_POINTS_MAX_CHANNELS];
};

// A key's order-preserving unsigned image: larger key, larger image.  0 is below every key's image (-inf's included), so
// it marks a pixel with q = 0, which is never drawn.
__device__ __forceinline__ uint32_t ordered_bits(float f) {
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ uint64_t ordered_bits(double f) {
    const uint64_t b = (uint64_t)__double_as_longlong(f);
    return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
template <typename T> struct KeyBits;
template <> struct KeyBits<float> { using type = uint32_t; };
template <> struct KeyBits<double> { using type = uint64_t; };

// log(u) / q with log taken in double and, for float, rounded once to float: the same value as numpy's
// np.log(u.astype(float64)).astype(float32), whatever the two libraries' last-place log errors.  log(u) / q orders the
// pixels as log(u) / pdf does, pdf = q / sum(q) with sum(q) > 0, so the draw does not depend on how sum(q) rounds.
template <typename T>
__device__ __forceinline__ typename KeyBits<T>::type draw_key(T p, T mk, T u) {
    const T q = p * mk;
    if (!(q > (T)0)) return 0;
    const T l = (T)log((double)u);
    return ordered_bits(l / q);
}

// The reference's pixel coordinate (utils/image.py:199-201): c / 256 * 2 - 1, the 256 hard-coded whatever S is
template <typename T>
__device__ __forceinline__ T ref_coord(int c) { return ((T)c / (T)256) * (T)2 - (T)1; }

// Fixed-order block sum over PP_CENTRE_THREADS values; every thread gets the total
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* red) {
    const int t = threadIdx.x;
    red[t] = v;
#pragma unroll
    for (int off = PP_CENTRE_THREADS / 2; off > 0; off >>= 1) {
        __syncthreads();
        if (t < off) red[t] += red[t + off];
    }
    __syncthreads();
    const T s = red[0];
    __syncthreads();
    return s;
}

template <typename T>
__global__ void __launch_bounds__(PP_CENTRE_THREADS) k_pp_centre(const T* __restrict__ prob, const T* __restrict__ mask, int S,
                                                                 int C, int K, PartPointsArgs a, vec2_t<T>* __restrict__ centers,
                                                                 int32_t* __restrict__ status) {
    __shared__ T red[PP_CENTRE_THREADS];
    __shared__ int ired[PP_CENTRE_THREADS];
    const int item = blockIdx.x, b = item / K, k = item - b * K;
    const int N = S * S;
    const T* p = prob + (size_t)b * N * C + a.channel[k];
    const T* mk = mask + (size_t)b * N;
    T s = 0;
    int pos = 0, bad = 0;
    for (int i = threadIdx.x; i < N; i += PP_CENTRE_THREADS) {
        const T q = __ldg(p + (size_t)i * C) * __ldg(mk + i);
        s += q;
        pos += q > (T)0;
        bad |= !(q >= (T)0) || isinf(q);
    }
    bad = __syncthreads_or(bad);
    const T total = block_sum(s, red);
    const int positive = block_sum(pos, ired);
    int st = UMR_PART_POINTS_OK;
    if (bad || !(total > (T)0) || isinf(total)) st = UMR_PART_POINTS_BAD_VALUES;
    else if (positive < a.n[k] * 3 / 2) st = UMR_PART_POINTS_TOO_FEW;
    if (st != UMR_PART_POINTS_OK) {
        if (threadIdx.x == 0) {
            centers[item] = make_vec2((T)NAN, (T)NAN);
            status[item] = st;
        }
        return;
    }
    T cx = 0, cy = 0;
    for (int i = threadIdx.x; i < N; i += PP_CENTRE_THREADS) {
        const T pdf = (__ldg(p + (size_t)i * C) * __ldg(mk + i)) / total;
        const int y = i / S, x = i - y * S;
        // get_coordinate_tensors (utils/image.py:143-150): numpy float64 maps, then the tensor's dtype
        cx += pdf * (T)((double)x / (double)S * 2.0 - 1.0);
        cy += pdf * (T)((double)y / (double)S * 2.0 - 1.0);
    }
    cx = block_sum(cx, red);
    cy = block_sum(cy, red);
    if (threadIdx.x == 0) {
        centers[item] = make_vec2(cx, cy);
        status[item] = UMR_PART_POINTS_OK;
    }
}

// (distance, index) order of the nearest-n selection; a NaN distance sorts last, as torch.topk ranks NaN largest
template <typename T>
__device__ __forceinline__ bool nearer(T dl, int l, T dj, int j) {
    const bool nl = isnan(dl), nj = isnan(dj);
    if (nl != nj) return nj;
    if (nl || dl == dj) return l < j;
    return dl < dj;
}

template <typename T>
__global__ void __launch_bounds__(PP_DRAW_THREADS) k_pp_draw(const T* __restrict__ prob, const T* __restrict__ mask,
                                                             const T* __restrict__ uniforms, int S, int C, int K,
                                                             PartPointsArgs a, const vec2_t<T>* __restrict__ centers_in,
                                                             const vec2_t<T>* __restrict__ centers,
                                                             const int32_t* __restrict__ status) {
    using U = typename KeyBits<T>::type;
    __shared__ unsigned hist[256];
    __shared__ U s_prefix;
    __shared__ int s_need;
    __shared__ int s_eq[PP_WARPS], s_take[PP_WARPS];
    __shared__ int sel[UMR_PART_POINTS_MAX_DRAWS];
    __shared__ T sd[UMR_PART_POINTS_MAX_DRAWS];
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const int item = blockIdx.x, b = item / K, k = item - b * K;
    const int n = a.n[k], m = n * 3 / 2;
    const int N = S * S;
    T* out = reinterpret_cast<T*>(a.points[k]) + (size_t)b * n * 2;
    int32_t* dr = a.drawn[k] ? a.drawn[k] + (size_t)b * m : nullptr;
    if (__ldg(status + item) != UMR_PART_POINTS_OK) {
        for (int i = t; i < 2 * n; i += PP_DRAW_THREADS) out[i] = (T)NAN;
        if (dr)
            for (int i = t; i < m; i += PP_DRAW_THREADS) dr[i] = -1;
        return;
    }
    const T* p = prob + (size_t)b * N * C + a.channel[k];
    const T* mk = mask + (size_t)b * N;
    const T* u = uniforms + (size_t)item * N;

    // radix select of the m-th largest key image, 8 bits per pass from the top: `prefix` holds the decided digits and
    // `need` how many keys equal to the final threshold are still to be taken
    U prefix = 0, decided = 0;
    int need = m;
    for (int shift = (int)sizeof(U) * 8 - 8; shift >= 0; shift -= 8) {
        for (int i = t; i < 256; i += PP_DRAW_THREADS) hist[i] = 0;
        __syncthreads();
        for (int i = t; i < N; i += PP_DRAW_THREADS) {
            const U key = draw_key(__ldg(p + (size_t)i * C), __ldg(mk + i), __ldg(u + i));
            if ((key & decided) == prefix) atomicAdd(&hist[(unsigned)(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (t == 0) {
            int above = 0, d = 255;
            for (; d > 0; --d) {
                if (above + (int)hist[d] >= need) break;
                above += (int)hist[d];
            }
            s_prefix = prefix | ((U)d << shift);
            s_need = need - above;
        }
        __syncthreads();
        prefix = s_prefix;
        need = s_need;
        decided |= (U)255 << shift;
    }

    // the drawn pixels in ascending index order: every key above the threshold, and the `need` lowest-indexed keys equal
    // to it
    const unsigned lt_mask = (1u << lane) - 1u;
    int eq_seen = 0, taken = 0;
    for (int base = 0; base < N; base += PP_DRAW_THREADS) {
        const int i = base + t;
        const U key = i < N ? draw_key(__ldg(p + (size_t)i * C), __ldg(mk + i), __ldg(u + i)) : (U)0;
        const bool gt = key > prefix, eq = key == prefix;
        const unsigned beq = __ballot_sync(0xffffffffu, eq);
        if (lane == 0) s_eq[w] = __popc(beq);
        __syncthreads();
        int eq_rank = eq_seen + __popc(beq & lt_mask), eq_tile = 0;
        for (int v = 0; v < PP_WARPS; ++v) {
            eq_rank += v < w ? s_eq[v] : 0;
            eq_tile += s_eq[v];
        }
        const bool take = gt || (eq && eq_rank < need);
        const unsigned btake = __ballot_sync(0xffffffffu, take);
        if (lane == 0) s_take[w] = __popc(btake);
        __syncthreads();
        int at = taken + __popc(btake & lt_mask), take_tile = 0;
        for (int v = 0; v < PP_WARPS; ++v) {
            at += v < w ? s_take[v] : 0;
            take_tile += s_take[v];
        }
        if (take) sel[at] = i;
        eq_seen += eq_tile;
        taken += take_tile;
        __syncthreads();
    }

    // the n nearest of the m drawn pixels, ascending (squared distance, pixel index); sel is in index order
    const vec2_t<T> c = centers_in ? centers_in[item] : centers[item];
    for (int j = t; j < m; j += PP_DRAW_THREADS) {
        const int idx = sel[j], y = idx / S, x = idx - y * S;
        const T dx = ref_coord<T>(x) - c.x, dy = ref_coord<T>(y) - c.y;
        sd[j] = dx * dx + dy * dy;
        if (dr) dr[j] = idx;
    }
    __syncthreads();
    for (int j = t; j < m; j += PP_DRAW_THREADS) {
        const T dj = sd[j];
        int r = 0;
        for (int l = 0; l < m; ++l) r += nearer(sd[l], l, dj, j);
        if (r < n) {
            const int idx = sel[j], y = idx / S, x = idx - y * S;
            out[2 * r] = ref_coord<T>(x);
            out[2 * r + 1] = ref_coord<T>(y);
        }
    }
}

static inline bool misaligned(const void* p, size_t a) { return ((uintptr_t)p % a) != 0; }

template <typename T>
static int part_points(const void* prob, const void* mask, const void* uniforms, int B, int S, int C, int K,
                       const PartPointsArgs& a, const void* centers_in, void* centers, int32_t* status, cudaStream_t stream) {
    const unsigned items = (unsigned)B * (unsigned)K;
    launch(k_pp_centre<T>, items, PP_CENTRE_THREADS, 0, stream, static_cast<const T*>(prob), static_cast<const T*>(mask), S,
           C, K, a, static_cast<vec2_t<T>*>(centers), status);
    launch(k_pp_draw<T>, items, PP_DRAW_THREADS, 0, stream, static_cast<const T*>(prob), static_cast<const T*>(mask),
           static_cast<const T*>(uniforms), S, C, K, a, static_cast<const vec2_t<T>*>(centers_in),
           static_cast<const vec2_t<T>*>(centers), static_cast<const int32_t*>(status));
    return (int)cudaGetLastError();
}

}  // namespace umr

using namespace umr;

extern "C" int umr_part_points(const void* part_prob, const void* mask, const void* uniforms, int32_t B, int32_t S, int32_t C,
                               int32_t K, const int32_t* channels, const int32_t* num_samples, int32_t dtype,
                               const void* centers_in, void* centers, void* const* points, int32_t* const* drawn,
                               int32_t* status, void* stream_) {
    if (!part_prob || !mask || !uniforms || !channels || !num_samples || !centers || !points || !status || B <= 0 || S <= 0 ||
        C <= 0 || K <= 0 || K > UMR_PART_POINTS_MAX_CHANNELS || (dtype != UMR_DTYPE_FLOAT32 && dtype != UMR_DTYPE_FLOAT64))
        return UMR_ERR_BAD_ARG;
    const size_t e = dtype == UMR_DTYPE_FLOAT64 ? sizeof(double) : sizeof(float);
    if (misaligned(part_prob, e) || misaligned(mask, e) || misaligned(uniforms, e) || misaligned(centers, 2 * e) ||
        misaligned(centers_in, 2 * e) || misaligned(status, sizeof(int32_t)))
        return UMR_ERR_BAD_ARG;
    PartPointsArgs a = {};
    bool too_many = false;
    for (int k = 0; k < K; ++k) {
        if (channels[k] < 0 || channels[k] >= C || num_samples[k] <= 0 || !points[k] || misaligned(points[k], 2 * e) ||
            (drawn && misaligned(drawn[k], sizeof(int32_t))))
            return UMR_ERR_BAD_ARG;
        too_many |= (int64_t)num_samples[k] * 3 / 2 > UMR_PART_POINTS_MAX_DRAWS;
        a.channel[k] = channels[k];
        a.n[k] = num_samples[k];
        a.points[k] = points[k];
        a.drawn[k] = drawn ? drawn[k] : nullptr;
    }
    if (too_many || S > UMR_PART_POINTS_MAX_SIDE || (int64_t)B * K > INT32_MAX) return UMR_ERR_TOO_LARGE;
    const cudaStream_t stream = (cudaStream_t)stream_;
    return dtype == UMR_DTYPE_FLOAT64
               ? part_points<double>(part_prob, mask, uniforms, B, S, C, K, a, centers_in, centers, status, stream)
               : part_points<float>(part_prob, mask, uniforms, B, S, C, K, a, centers_in, centers, status, stream);
}
