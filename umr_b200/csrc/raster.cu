// raster.cu -- tile-binned soft rasteriser (forward + backward) for sm_90a.
//
// Replaces the reference kernels external/SoftRas/soft_renderer/cuda/soft_rasterize_cuda_kernel.cu
// :222-282 (prep), :285-476 (forward), :479-656 (backward), which run one thread per pixel over ALL
// faces.  Design (DESIGN.md §3):
//   k_prep            one thread per face -> a 128-byte face record (vertices, barycentric inverse, Gram
//                     matrix, cull box expanded by the sigmoid cut-off radius, obtuse/front flags), a
//                     compact float4 cull box for binning, and the image's UNION cull box (tiles outside
//                     it skip the face scan).
//   tile list         one CTA per 16x16-pixel tile: the image's cull boxes are contiguous, so they are
//                     staged into shared memory with ONE TMA bulk copy (cp.async.bulk + mbarrier) per
//                     <= 2048 faces; the scan ballot-compacts the faces touching the tile into an ORDER-
//                     PRESERVING index list (ascending face index is required: p2f prefix-max weights,
//                     hard z-buffer tie-break).  The scattered 128-byte records of the list are gathered
//                     with 16-byte cp.async copies, double buffered (32 records per stage).
//   k_raster_fwd      thread = pixel (a warp = an 8x4 block): walks the staged records in face order;
//                     fuses the background fill, the p2f accumulation (warp-shuffle reduce, totals owned
//                     by lane j, one global RED per (warp, face)) and the 2x2 average pool (shuffles).
//   k_raster_bwd_pairs  the backward has no ordering constraint, so the tile's work is flattened to
//                     (pixel, face) PAIRS: each face's cull box selects a rectangle of tile pixels, the
//                     rectangle sizes are prefix-summed and every warp owns an equal contiguous run of
//                     pairs, walked face by face; the 9 vertex gradients are accumulated privately and
//                     combined once per (warp, face) (shuffle reduce + 9 global REDs) instead of the
//                     reference's 9 global atomics per (pixel, face); the pool backward is fused.
//   k_raster_bwd      per-pixel backward.
//   k_raster_fwd / k_raster_bwd serve the generic modes only: they read the distance / alpha / texture mode
//                     ids at run time (hard / barycentric distance, hard / sum alpha, vertex textures).
//
// PARITY: this translation unit is compiled with -fmad=false.  The per-(pixel, face) arithmetic is an
// operation-for-operation twin of the reference's float instantiation (same expression order, same
// float/double promotions -- SURVEY.md App. B-6), because the reference's output is numerically
// chaotic on sliver faces (App. B-15) and only an identical IEEE op sequence reproduces its discrete
// decisions.  Only expf() may differ from a CPU libm by ulps.  Shortcuts are taken only where the result
// is provably bit-identical (double-rounding-innocuous divisions, x*0 / 0/x cases).
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "raster_generic.cuh"
#include "umr_b200.h"

namespace umr {

constexpr int CHUNK = 32;         // face records per TMA stage
constexpr int NSTAGE = 2;
// float records (layout in raster_generic.cuh) also carry, after the flags:
constexpr int R_IZ2 = 29;  // 3 : 1 / (z_k * z_k)  (backward z-gradient factor)

// Face indices.  Meshes of up to NARROW_MAX_FACES faces keep them in 16 bits (coarse-bin lists, tile lists, pair-block
// headers); larger meshes take the wide instantiations (IdxT = uint32_t) of the same kernels.  The hard render's
// face-index plane stores face ids as float, exact below 2^24, which bounds F (UMR_RASTER_MAX_FACES).
constexpr int NARROW_MAX_FACES = 65535;
// Pair-block header: face | count << HDR_SHIFT (count <= 32).  16 face bits (narrow) or 24 (wide).
template <typename IdxT>
__host__ __device__ constexpr int hdr_shift() { return sizeof(IdxT) == 2 ? 16 : 24; }
// Generic kernels and the recompute backward hold a tile list of window-relative u16 offsets in shared memory: faces are
// listed and consumed in ascending windows of at most FACE_WINDOW faces (one window when F <= 65535).
constexpr int FACE_WINDOW = 65536;

struct WorkspaceLayout {
    size_t rec_off, box_off, p2f_off, ubox_off, ccount_off, clist_off, total;
    size_t clist_cap;  // wide layout: entries of the shared coarse-list pool
};
__host__ __device__ inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
constexpr int COARSE_BIN = 64;  // == CB in raster_stream.cuh
// Wide coarse lists: one pool for all bins, WIDE_BIN_ENTRIES entries (32 bytes) per face; a bin whose list does not fit
// is marked and its consumers walk every face instead (same result, box tests filter them).
constexpr size_t WIDE_BIN_ENTRIES = 8;
constexpr uint32_t BIN_ALL_FACES = 0xffffffffu;
// S = raster side (0: no coarse-bin lists, e.g. the generic-mode kernels)
inline WorkspaceLayout ws_layout(int B, int F, int S) {
    WorkspaceLayout L;
    const size_t n = (size_t)B * F;
    const size_t ncb = (size_t)(S + COARSE_BIN - 1) / COARSE_BIN;
    const size_t nbin = (size_t)B * ncb * ncb;
    L.rec_off = 0;
    L.box_off = align256(n * REC_LEN * sizeof(float));
    L.p2f_off = L.box_off + align256(n * sizeof(float4));
    L.ubox_off = L.p2f_off + align256(n * 4 * sizeof(float));
    L.ccount_off = L.ubox_off + align256((size_t)B * 4 * sizeof(uint32_t));
    if (F <= NARROW_MAX_FACES) {  // ccount int[nbin], clist u16[nbin][F]
        L.clist_cap = 0;
        L.clist_off = L.ccount_off + align256(nbin * sizeof(int));
        L.total = L.clist_off + align256(nbin * F * sizeof(uint16_t));
    } else {  // ccount {count, pool offset}[nbin] + the pool cursor (u64), clist u32[clist_cap]
        L.clist_cap = n * WIDE_BIN_ENTRIES;
        if (L.clist_cap > 0xfffffff0u) L.clist_cap = 0xfffffff0u;
        L.clist_off = L.ccount_off + align256(nbin * 2 * sizeof(uint32_t) + sizeof(unsigned long long));
        L.total = L.clist_off + align256(L.clist_cap * sizeof(uint32_t));
    }
    return L;
}

// ---------------------------------------------------------------------------------------------
// prep: kernel.cu:222-282 + the per-face parts of :32-44
// ---------------------------------------------------------------------------------------------
// Monotone key of a cull-box bound for atomicMax on a zero-initialised word: positive floats order like
// their bit patterns; non-positive values map to 0 (the union box then merely contains the screen
// centre, which stays conservative); NaN poisons the union so nothing is ever skipped.
__device__ __forceinline__ uint32_t ubox_key(float v) {
    if (v != v) return 0xffffffffu;
    return v > 0.f ? __float_as_uint(v) : 0u;
}

// grid (ceil(F/256), B): every block belongs to one image.  Also accumulates the image's UNION cull box
// ubox[b] = {max xhi, max -xlo, max yhi, max -ylo} (keys) so tiles outside it skip the face scan.
__global__ void __launch_bounds__(256) k_prep(const float* __restrict__ fv, float* __restrict__ rec,
                                              float4* __restrict__ box, uint32_t* __restrict__ ubox, int F, float r,
                                              const uint32_t* __restrict__ only_if_nonzero = nullptr) {
    // texture-only backward with a pair buffer: the records are only needed by the recompute fallback -- skip when no tile
    // needs it
    if (only_if_nonzero != nullptr && __ldg(only_if_nonzero) == 0u) return;
    const int fidx = blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = fidx < F;
    const int i = blockIdx.y * F + (valid ? fidx : F - 1);  // clamp: the tail threads redo the last face
    const float* f = fv + (size_t)i * 9;
    float v[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) v[k] = __ldg(f + k);
    const float x0 = v[0], y0 = v[1], x1 = v[3], y1 = v[4], x2 = v[6], y2 = v[7];
    float star[9] = {y1 - y2, x2 - x1, x1 * y2 - x2 * y1,  //
                     y2 - y0, x0 - x2, x2 * y0 - x0 * y2,  //
                     y0 - y1, x1 - x0, x0 * y1 - x1 * y0};
    float det = x2 * (y0 - y1) + x0 * (y1 - y2) + x1 * (y2 - y0);
    // max(det, 1e-10) / min(det, -1e-10) are evaluated in double by the reference and stored as
    // float; a float select against the rounded constant is bit-identical (DESIGN.md §4).
    det = det > 0 ? fmaxf(det, 1e-10f) : fminf(det, -1e-10f);
    float out[REC_LEN];
#pragma unroll
    for (int k = 0; k < 9; ++k) out[R_V + k] = v[k];
#pragma unroll
    for (int k = 0; k < 9; ++k) out[R_INV + k] = star[k] / det;
    out[R_SYM + 0] = x0 * x0 + y0 * y0 + 1.f;
    out[R_SYM + 1] = x0 * x1 + y0 * y1 + 1.f;
    out[R_SYM + 2] = x0 * x2 + y0 * y2 + 1.f;
    out[R_SYM + 3] = x1 * x1 + y1 * y1 + 1.f;
    out[R_SYM + 4] = x1 * x2 + y1 * y2 + 1.f;
    out[R_SYM + 5] = x2 * x2 + y2 * y2 + 1.f;
    const float xlo = fminf(fminf(x0, x1), x2) - r, xhi = fmaxf(fmaxf(x0, x1), x2) + r;
    const float ylo = fminf(fminf(y0, y1), y2) - r, yhi = fmaxf(fmaxf(y0, y1), y2) + r;
    out[R_BOX + 0] = xlo;
    out[R_BOX + 1] = xhi;
    out[R_BOX + 2] = ylo;
    out[R_BOX + 3] = yhi;
    uint32_t flags = 0;
    if ((x1 - x0) * (x2 - x0) + (y1 - y0) * (y2 - y0) < 0) flags = 1;
    else if ((x2 - x1) * (x0 - x1) + (y2 - y1) * (y0 - y1) < 0) flags = 2;
    else if ((x0 - x2) * (x1 - x2) + (y0 - y2) * (y1 - y2) < 0) flags = 4;
    if ((y2 - y0) * (x1 - x0) < (y1 - y0) * (x2 - x0)) flags |= 8;  // kernel.cu:42-44
    {
        // bit 4: thin / degenerate triangle (sine of its smallest angle below ~1e-3): its barycentric inverse is not
        // trustworthy, so "inside" may be claimed far from the triangle (SURVEY.md App. B-15).  Only k_visible_faces reads
        // it -- such faces are scanned over their whole cull box there instead of the tight bounding box.
        const float l01 = (x1 - x0) * (x1 - x0) + (y1 - y0) * (y1 - y0);
        const float l02 = (x2 - x0) * (x2 - x0) + (y2 - y0) * (y2 - y0);
        const float l12 = (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1);
        const float lmin = fminf(fminf(l01, l02), l12);
        const float prod2 = (l01 * l02 * l12) / fmaxf(lmin, 1e-30f);   // product of the two longest squared edges
        const float draw = x2 * (y0 - y1) + x0 * (y1 - y2) + x1 * (y2 - y0);
        if (!(draw * draw >= 1e-6f * prod2)) flags |= 16u;               // also NaN / zero area
    }
    out[R_FLG] = __uint_as_float(flags);
    out[R_IZ2 + 0] = 1.f / (v[2] * v[2]);
    out[R_IZ2 + 1] = 1.f / (v[5] * v[5]);
    out[R_IZ2 + 2] = 1.f / (v[8] * v[8]);
    if (valid) {
        float4* dst = reinterpret_cast<float4*>(rec + (size_t)i * REC_LEN);
#pragma unroll
        for (int k = 0; k < REC_LEN / 4; ++k)
            dst[k] = make_float4(out[4 * k], out[4 * k + 1], out[4 * k + 2], out[4 * k + 3]);
        box[i] = make_float4(xlo, xhi, ylo, yhi);
    }
    // union box: warp max of the 4 keys, then one atomicMax per warp and bound
    uint32_t k0 = ubox_key(xhi), k1 = ubox_key(-xlo), k2 = ubox_key(yhi), k3 = ubox_key(-ylo);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        k0 = max(k0, __shfl_xor_sync(0xffffffffu, k0, o));
        k1 = max(k1, __shfl_xor_sync(0xffffffffu, k1, o));
        k2 = max(k2, __shfl_xor_sync(0xffffffffu, k2, o));
        k3 = max(k3, __shfl_xor_sync(0xffffffffu, k3, o));
    }
    if ((threadIdx.x & 31) == 0) {
        uint32_t* u = ubox + (size_t)blockIdx.y * 4;
        atomicMax(u + 0, k0); atomicMax(u + 1, k1); atomicMax(u + 2, k2); atomicMax(u + 3, k3);
    }
}

// true when the tile (pixel-centre extents in s_ext) lies completely outside the image's union cull box
__device__ __forceinline__ bool tile_outside_union(const uint32_t* __restrict__ ubox, int b, const float* s_ext) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(ubox) + b);
    if (u.x == 0xffffffffu || u.y == 0xffffffffu || u.z == 0xffffffffu || u.w == 0xffffffffu) return false;  // NaN seen
    const float xhi = __uint_as_float(u.x), xlo = -__uint_as_float(u.y);
    const float yhi = __uint_as_float(u.z), ylo = -__uint_as_float(u.w);
    return s_ext[0] > xhi || s_ext[1] < xlo || s_ext[2] > yhi || s_ext[3] < ylo;
}

// ---------------------------------------------------------------------------------------------
// Deterministic mode (umr_raster_*_deterministic, DESIGN.md §3): the forward adds its per-(warp, face) p2f partials as
// exact fixed point.  A partial v (|v| <= 32: a warp sum of 32 pixel terms of magnitude <= 1) becomes the integer
// round(|v| * 2^P2F_FRAC_BITS) < 2^102, split into P2F_LIMBS limbs of P2F_LIMB_BITS bits, each added into its own int64
// word with an integer RED.  Integer addition is associative, so the words do not depend on the order of the REDs, and a
// limb word holds at most (8x4 pixel blocks of the raster) * 2^26 < 2^63 for every raster the kernels can launch.
// ---------------------------------------------------------------------------------------------
constexpr int P2F_LIMBS = 4;
constexpr int P2F_LIMB_BITS = 26;
constexpr int P2F_FRAC_BITS = 96;
constexpr int P2F_DET_WORDS = 3 * P2F_LIMBS + 1;  // x, y, w limbs, then a word set when a partial was not finite

__device__ __forceinline__ void red_add_u64(unsigned long long* addr, unsigned long long v) {
    asm volatile("red.global.add.u64 [%0], %1;" ::"l"(addr), "l"(v) : "memory");
}

__device__ __forceinline__ void red_fixed(unsigned long long* limbs, unsigned long long* bad, float v) {
    const uint32_t u = __float_as_uint(v);
    const int e = (int)((u >> 23) & 0xffu);
    const int s = (e ? e : 1) - (150 - P2F_FRAC_BITS);  // |v| * 2^96 = m * 2^s
    if (e == 0xff || s > P2F_LIMBS * P2F_LIMB_BITS - 24) {  // NaN / inf (|v| <= 32 otherwise)
        atomicOr(bad, 1ull);
        return;
    }
    const uint32_t m = (u & 0x7fffffu) | (e ? 0x800000u : 0u);
    unsigned __int128 q;
    if (s >= 0) q = (unsigned __int128)m << s;
    else if (s > -32) q = ((unsigned long long)m + (1ull << (-s - 1))) >> (-s);  // round half away from zero
    else return;
    const bool neg = (u >> 31) != 0;
#pragma unroll
    for (int k = 0; k < P2F_LIMBS; ++k) {
        const unsigned long long l = (unsigned long long)(q >> (k * P2F_LIMB_BITS)) & ((1ull << P2F_LIMB_BITS) - 1ull);
        if (l != 0ull) red_add_u64(limbs + k, neg ? 0ull - l : l);
    }
}

// one (warp, face) p2f partial into the face's P2F_DET_WORDS accumulator words
__device__ __forceinline__ void red_p2f_fixed(unsigned long long* acc, float x, float y, float w) {
    red_fixed(acc, acc + 3 * P2F_LIMBS, x);
    red_fixed(acc + P2F_LIMBS, acc + 3 * P2F_LIMBS, y);
    red_fixed(acc + 2 * P2F_LIMBS, acc + 3 * P2F_LIMBS, w);
}

// ---------------------------------------------------------------------------------------------
// tile machinery shared by forward and backward
// ---------------------------------------------------------------------------------------------
constexpr int PT = 16;          // pixel-tile side of the pair-parallel backward kernel
static_assert(PT * PT == CTA, "k_raster_bwd_det stages one per-pixel slot per thread; bwd_pair_acc reads them with stride PT * PT");
constexpr int BOX_PIECE = 2048;  // cull boxes staged per TMA bulk copy (32 KB)

// dynamic shared memory: [ records NSTAGE*CHUNK*128 B | cull boxes min(F,BOX_PIECE)*16 B | list u16[F] ]
__host__ __device__ inline size_t smem_box_off() { return (size_t)NSTAGE * CHUNK * REC_LEN * 4; }
__host__ __device__ inline size_t smem_list_off(int F) {
    return smem_box_off() + (size_t)(F < BOX_PIECE ? F : BOX_PIECE) * 16;
}

// Ordered compaction of the faces whose cull box touches the tile.  The image's cull boxes are
// contiguous in HBM/L2, so each piece (<= 2048 faces, 32 KB) is staged with ONE TMA bulk copy signalled
// on an mbarrier; the scan then runs out of shared memory.  Each warp owns a contiguous run of the
// piece (ascending face order = warp-major, round, lane), keeps its ballots in registers, and one
// barrier per piece turns the per-warp counts into list offsets.  Returns the list length (uniform).
// `list` == nullptr: count only.
template <typename IdxT = uint16_t>
__device__ __forceinline__ int build_tile_list(const float4* __restrict__ box, int F, float tx_first,
                                               float tx_last, float ty_bot, float ty_top, float4* s_box,
                                               IdxT* list, int* s_warp_cnt, uint64_t* bar, uint32_t& phase) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int total = 0;
    for (int base = 0; base < F; base += BOX_PIECE) {
        const int P = min(BOX_PIECE, F - base);
        if (tid == 0) {
            mbar_arrive_expect_tx(bar, (uint32_t)P * 16u);
            tma_bulk_g2s(s_box, box + base, (uint32_t)P * 16u, bar);
        }
        mbar_wait(bar, phase);
        phase ^= 1u;
        const int per = ((P + NWARP * 32 - 1) / (NWARP * 32)) * 32;  // faces per warp, multiple of 32, <= 256
        uint32_t masks[BOX_PIECE / (NWARP * 32)];
        int cnt = 0;
#pragma unroll
        for (int r = 0; r < BOX_PIECE / (NWARP * 32); ++r) {
            const int f = warp * per + r * 32 + lane;
            bool hit = false;
            if (r * 32 < per && f < P) {
                const float4 bb = s_box[f];
                hit = !(tx_first > bb.y || tx_last < bb.x || ty_bot > bb.w || ty_top < bb.z);
            }
            masks[r] = __ballot_sync(0xffffffffu, hit);
            cnt += __popc(masks[r]);
        }
        if (lane == 0) s_warp_cnt[warp] = cnt;
        __syncthreads();
        int off = total;
#pragma unroll
        for (int w = 0; w < NWARP; ++w) {
            const int c = s_warp_cnt[w];
            if (w < warp) off += c;
            total += c;
        }
        const uint32_t lt = (1u << lane) - 1u;
        if (sizeof(IdxT) == 2 || list != nullptr) {
#pragma unroll
            for (int r = 0; r < BOX_PIECE / (NWARP * 32); ++r) {
                if ((masks[r] >> lane) & 1u) list[off + __popc(masks[r] & lt)] = (IdxT)(base + warp * per + r * 32 + lane);
                off += __popc(masks[r]);
            }
        }
        __syncthreads();  // list visible; s_box / s_warp_cnt reusable
    }
    return total;
}

// Gather chunk c of the tile list (32 records x 128 B, scattered in L2) into stage c % NSTAGE with one
// 16-byte cp.async per thread (8 consecutive threads fetch one 128-byte record = one cache line).
// Always commits a group so every thread's group count stays uniform.
__device__ __forceinline__ void issue_chunk(const float* __restrict__ rec_img, const uint16_t* list, int n,
                                            int c, float* s_rec) {
    const int j = threadIdx.x >> 3, q = threadIdx.x & 7;
    const int idx = c * CHUNK + j;
    if (idx < n) {
        const int f = list[idx];
        cp_async16(s_rec + ((size_t)(c % NSTAGE) * CHUNK + j) * REC_LEN + q * 4, rec_img + (size_t)f * REC_LEN + q * 4);
    }
    cp_async_commit();
}


// =============================================================================================
// thread <-> pixel mapping: a warp covers an 8x4 pixel block (better lane utilisation against the
// ~23x23-pixel cull boxes than a 16x2 strip), a CTA a 16x16 tile = 2x4 warp blocks.
// The 2x2 anti-aliasing quad of the (even x, even y) lane is lanes ^1, ^8, ^9.
// =============================================================================================
struct PixelMap {
    int px, py;
    bool live;
    float xp, yp;
};
__device__ __forceinline__ PixelMap map_pixel(int S) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    PixelMap m;
    m.px = blockIdx.x * TILE + (warp & 1) * 8 + (lane & 7);
    m.py = blockIdx.y * TILE + (warp >> 1) * 4 + (lane >> 3);  // image row (0 = top)
    m.live = m.px < S && m.py < S;
    m.xp = pixel_coord(m.px, S);
    m.yp = pixel_coord(S - 1 - m.py, S);
    return m;
}

// tile extents in pixel-centre coordinates (monotone in the index, so the cull test is conservative);
// four threads compute one division each and broadcast through shared memory
__device__ __forceinline__ void tile_extents_at(int S, float* s_ext, int tile, int bx, int by) {
    const int t = threadIdx.x;
    if (t < 4) {
        const int x_last_i = min(bx * tile + tile - 1, S - 1);
        const int y_last_i = min(by * tile + tile - 1, S - 1);
        const int i = t == 0 ? bx * tile : t == 1 ? x_last_i : t == 2 ? S - 1 - y_last_i : S - 1 - by * tile;
        s_ext[t] = pixel_coord(i, S);  // 0: x first, 1: x last, 2: y bottom, 3: y top
    }
}
__device__ __forceinline__ void tile_extents(int S, float* s_ext, int tile = TILE) {
    tile_extents_at(S, s_ext, tile, (int)blockIdx.x, (int)blockIdx.y);
}

// =============================================================================================
// forward
// =============================================================================================
// RGB: 1 softmax, 0 hard; dist/alpha/texture modes read at run time.  DET: fixed-point p2f (red_p2f_fixed).
template <int RGB, bool DET = false>
__global__ void __launch_bounds__(CTA, 3) k_raster_fwd(const float* __restrict__ rec_all,
                                                       const float4* __restrict__ box_all,
                                                       const float* __restrict__ textures,
                                                       float* __restrict__ images, float* __restrict__ colors_hi,
                                                       float* __restrict__ aggrs, float* __restrict__ p2f_acc,
                                                       const uint32_t* __restrict__ ubox, Consts<float> K, float eps,
                                                       float bg0, float bg1, float bg2) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_rec = reinterpret_cast<float*>(smem_raw);
    float4* s_box = reinterpret_cast<float4*>(smem_raw + smem_box_off());
    uint16_t* s_list = reinterpret_cast<uint16_t*>(smem_raw + smem_list_off(K.F));
    __shared__ uint64_t s_bar;
    __shared__ int s_warp_cnt[NWARP];
    __shared__ float s_ext[4];

    const int tid = threadIdx.x, lane = tid & 31;
    const int b = blockIdx.z;
    const int S = K.S, F = K.F;
    const PixelMap pm = map_pixel(S);
    const int px = pm.px, py = pm.py;
    const bool live = pm.live;
    const float xp = pm.xp, yp = pm.yp;

    if (tid == 0) {
        mbar_init(&s_bar, 1);
        fence_mbar_init();
    }
    tile_extents(S, s_ext);
    __syncthreads();

    const float4* box = box_all + (size_t)b * F;
    uint32_t bar_phase = 0;
    const bool outside = tile_outside_union(ubox, b, s_ext);
    bool any = false;  // some window listed a face (uniform)

    // pixel state (kernel.cu:335-348)
    float acc_a = K.alpha == UMR_ALPHA_PROD ? 1.f : 0.f;  // alpha accumulator (kernel.cu:335-336)
    float ssum = expf(eps / K.gamma);
    float smax = eps;
    float c0, c1, c2;
    if (RGB == 1) { c0 = bg0 * ssum; c1 = bg1 * ssum; c2 = bg2 * ssum; }
    else { c0 = bg0; c1 = bg1; c2 = bg2; }
    float zmin = 10000000.f;
    int fid = -1;

    const float* tex_img = textures + (size_t)(b / K.tex_div) * K.tex_bs;
    // torch-1.1 affine_grid (align_corners=True) coordinates of this pixel: linspace(-1, 1, S)
    // S = 1: torch 1.1's affine_grid takes linspace(-1, 1, 1) = [-1] (DESIGN.md §2), where 2 / 0 would give -1 + inf * 0 = NaN
    const float gstep = S > 1 ? 2.f / (float)(S - 1) : 0.f;
    const float gx = (px * 2 < S) ? (-1.f + gstep * px) : (1.f - gstep * (S - 1 - px));
    const float gy = (py * 2 < S) ? (-1.f + gstep * py) : (1.f - gstep * (S - 1 - py));

    for (int wb = 0; wb < F && !outside; wb += FACE_WINDOW) {
    const int n = build_tile_list(box + wb, min(F - wb, FACE_WINDOW), s_ext[0], s_ext[1], s_ext[2], s_ext[3], s_box, s_list,
                                  s_warp_cnt, &s_bar, bar_phase);
    // (build_tile_list ends with __syncthreads: the list is visible)
    any = any || n > 0;
    const float* rec_img = rec_all + ((size_t)b * F + wb) * REC_LEN;
    const int nchunk = (n + CHUNK - 1) / CHUNK;
    if (nchunk > 0) {
        issue_chunk(rec_img, s_list, n, 0, s_rec);
        issue_chunk(rec_img, s_list, n, 1, s_rec);
    }
    for (int c = 0; c < nchunk; ++c) {
        const int st = c % NSTAGE;
        const int cnt = min(CHUNK, n - c * CHUNK);
        cp_async_wait<1>();  // chunk c has landed (c+1 may still be in flight)
        __syncthreads();     // ... for every thread
        const float* chunk = s_rec + (size_t)st * CHUNK * REC_LEN;
        // p2f partial sums of this warp: lane j owns chunk face j (registers, no shared traffic)
        float own_x = 0.f, own_y = 0.f, own_w = 0.f;
        float4 bb = *reinterpret_cast<const float4*>(chunk + R_BOX);
        for (int j = 0; j < cnt; ++j) {
            const float* rc = chunk + j * REC_LEN;
            // prefetch the next cull box while this face is evaluated
            const float4 bbn = *reinterpret_cast<const float4*>(chunk + (j + 1 < cnt ? j + 1 : j) * REC_LEN + R_BOX);
            float a_x = 0.f, a_y = 0.f, a_w = 0.f;
            bool contrib = false;
            if (live && !(xp > bb.y || xp < bb.x || yp > bb.w || yp < bb.z)) {
                Frag<float> fr;
                if (fragment_any(rc, xp, yp, K, fr)) {
                    if (K.alpha == UMR_ALPHA_PROD) {
                        acc_a = (float)((double)acc_a * (1. - (double)fr.D));  // kernel.cu:396
                    } else if (K.alpha == UMR_ALPHA_SUM) {
                        acc_a += fr.D;                                         // :394
                    } else if (fr.D > 0.5f) {
                        acc_a = 1.f;                                           // :392 hard
                    }
                    float k0 = fr.w0, k1 = fr.w1, k2 = fr.w2;
                    clip_bary(k0, k1, k2);
                    const float zp = depth_of(rc, k0, k1, k2);
                    if (!(zp < K.near_ || zp > K.far_)) {
                        const uint32_t flg = __float_as_uint(rc[R_FLG]);
                        const bool front = (flg & 8u) != 0;
                        const int f = wb + s_list[c * CHUNK + j];
                        if (RGB == 0) {
                            const bool inside = fr.w0 <= 1 && fr.w0 >= 0 && fr.w1 <= 1 && fr.w1 >= 0 &&
                                                fr.w2 <= 1 && fr.w2 >= 0;
                            if (zp < zmin && inside && (K.double_side || front)) {
                                zmin = zp;
                                fid = f;
                                sample_texture(tex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, c0, c1, c2);
                            }
                        } else if (front || K.double_side) {
                            const float zn = (K.far_ - zp) / (K.far_ - K.near_);
                            float ed = 1.f;
                            if (zn > smax) { ed = expf((smax - zn) / K.gamma); smax = zn; }
                            const float ez = expf((zn - smax) / K.gamma);
                            ssum = ed * ssum + ez * fr.D;
                            const float a = ez * fr.D;
                            // a == 0 with no max update (occluded face whose weight underflowed): the colour
                            // update is c = 1*c + 0*texel = c and the p2f terms are 0 -- skip the texel fetch
                            if (a != 0.f || ed != 1.f) {
                                a_x = a * gx; a_y = a * gy; a_w = a;
                                contrib = a != 0.f;
                                float t0, t1, t2;
                                sample_texture(tex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, t0, t1, t2);
                                c0 = ed * c0 + a * t0;
                                c1 = ed * c1 + a * t1;
                                c2 = ed * c2 + a * t2;
                            }
                        }
                    }
                }
            }
            if (RGB == 1 && p2f_acc != nullptr) {
                // p2f: warp-shuffle reduction (replaces the 4 global atomics per (pixel, face) of
                // kernel.cu:427-430); the totals stay in the registers of lane j
                if (__any_sync(0xffffffffu, contrib)) {
                    a_x = warp_sum(a_x); a_y = warp_sum(a_y); a_w = warp_sum(a_w);
                    if (lane == j) { own_x += a_x; own_y += a_y; own_w += a_w; }
                }
            }
            bb = bbn;
        }
        if (RGB == 1 && p2f_acc != nullptr && own_w != 0.f) {  // one global RED per (warp, face, component)
            if constexpr (DET) {
                red_p2f_fixed(reinterpret_cast<unsigned long long*>(p2f_acc) + ((size_t)b * F + wb + s_list[c * CHUNK + lane]) * P2F_DET_WORDS,
                              own_x, own_y, own_w);
            } else {
            float* dst = p2f_acc + ((size_t)b * F + wb + s_list[c * CHUNK + lane]) * 4;
            red_add_global(dst + 0, own_x);
            red_add_global(dst + 1, own_y);
            red_add_global(dst + 2, own_w);
            }
        }
        __syncthreads();  // everyone is done with stage st
        issue_chunk(rec_img, s_list, n, c + NSTAGE, s_rec);  // commits an empty group past the end
    }
    }

    // finalise (kernel.cu:443-475)
    float alpha;
    if (K.alpha == UMR_ALPHA_PROD) alpha = (float)(1. - (double)acc_a);  // kernel.cu:449-451
    else if (K.alpha == UMR_ALPHA_SUM) alpha = acc_a / K.F;              // :447
    else alpha = acc_a;                                                  // :445
    float o0, o1, o2, g0, g1;
    if (RGB == 0) {
        o0 = c0; o1 = c1; o2 = c2;  // background kept when no face won (c* still bg)
        g0 = zmin; g1 = (float)fid;
    } else {
        // 0 / ssum == 0 exactly: skip the IEEE division for black-background / untouched pixels
        o0 = c0 == 0.f ? c0 : c0 / ssum;
        o1 = c1 == 0.f ? c1 : c1 / ssum;
        o2 = c2 == 0.f ? c2 : c2 / ssum;
        g0 = ssum; g1 = smax;
    }
    const size_t np = (size_t)S * S;
    // pooled values: avg_pool2d(2,2) = ((a00 + a01) + a10) + a11, then /4 (rasterizer.py:52-53)
    float v[4] = {o0, o1, o2, alpha};
    if (K.aa) {
        if (any) {  // uniform
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float a01 = __shfl_xor_sync(0xffffffffu, v[k], 1);
                const float a10 = __shfl_xor_sync(0xffffffffu, v[k], 8);
                const float a11 = __shfl_xor_sync(0xffffffffu, v[k], 9);
                v[k] = (((v[k] + a01) + a10) + a11) * 0.25f;  // meaningful on the (even x, even y) lane
            }
        } else {  // untouched tile: the quad holds four identical values; same arithmetic, no shuffles
#pragma unroll
            for (int k = 0; k < 4; ++k) v[k] = (((v[k] + v[k]) + v[k]) + v[k]) * 0.25f;
        }
    }
    const int tx0 = blockIdx.x * TILE, ty0 = blockIdx.y * TILE;
    if (K.aa && K.vec_store && tx0 + TILE <= S && ty0 + TILE <= S) {  // uniform: full tile, aligned buffers
        // Coalesced 128-bit stores: the tile's 6 raster-resolution planes (RGBA + 2 aggregation planes) and its
        // 4 pooled planes are transposed through shared memory (the record stages are free now) so every
        // thread issues float4 stores of 64-byte row segments instead of scattered 4-byte stores.
        cp_async_wait<0>();
        __syncthreads();
        float* st = s_rec;  // 6 * 256 + 4 * 64 = 1792 floats <= NSTAGE * CHUNK * REC_LEN = 2048
        const int o = (py - ty0) * TILE + (px - tx0);
        st[0 * 256 + o] = o0; st[1 * 256 + o] = o1; st[2 * 256 + o] = o2; st[3 * 256 + o] = alpha;
        st[4 * 256 + o] = g0; st[5 * 256 + o] = g1;
        if ((lane & 1) == 0 && (lane & 8) == 0) {
            const int po = ((py - ty0) >> 1) * (TILE / 2) + ((px - tx0) >> 1);
#pragma unroll
            for (int k = 0; k < 4; ++k) st[6 * 256 + k * 64 + po] = v[k];
        }
        __syncthreads();
        for (int i = tid; i < 6 * 64; i += CTA) {
            const int plane = i >> 6, rem = i & 63, row = rem >> 2, q = rem & 3;
            const float4 val = *reinterpret_cast<const float4*>(st + plane * 256 + row * TILE + q * 4);
            const size_t off = (size_t)(ty0 + row) * S + tx0 + q * 4;
            if (plane < 4) {
                if (colors_hi != nullptr)
                    *reinterpret_cast<float4*>(colors_hi + ((size_t)b * 4 + plane) * np + off) = val;
            } else {
                *reinterpret_cast<float4*>(aggrs + ((size_t)b * 2 + (plane - 4)) * np + off) = val;
            }
        }
        if (tid < 64) {
            const int k = tid >> 4, rem = tid & 15, row = rem >> 1, q = rem & 1;
            const float4 val = *reinterpret_cast<const float4*>(st + 6 * 256 + k * 64 + row * (TILE / 2) + q * 4);
            const int IS = K.IS;
            const size_t nq = (size_t)IS * IS;
            *reinterpret_cast<float4*>(images + ((size_t)b * 4 + k) * nq + (size_t)((ty0 >> 1) + row) * IS + (tx0 >> 1) + q * 4) = val;
        }
        return;
    }
    if (live) {
        const size_t p = (size_t)py * S + px;
        aggrs[((size_t)b * 2 + 0) * np + p] = g0;
        aggrs[((size_t)b * 2 + 1) * np + p] = g1;
        if (colors_hi != nullptr) {
            colors_hi[((size_t)b * 4 + 0) * np + p] = o0;
            colors_hi[((size_t)b * 4 + 1) * np + p] = o1;
            colors_hi[((size_t)b * 4 + 2) * np + p] = o2;
            colors_hi[((size_t)b * 4 + 3) * np + p] = alpha;
        }
    }
    if (K.aa) {
        if (live && (lane & 1) == 0 && (lane & 8) == 0) {
            const int IS = K.IS;
            const size_t q = (size_t)(py >> 1) * IS + (px >> 1);
            const size_t nq = (size_t)IS * IS;
#pragma unroll
            for (int k = 0; k < 4; ++k) images[((size_t)b * 4 + k) * nq + q] = v[k];
        }
    } else if (live && images != colors_hi) {
        const size_t p = (size_t)py * S + px;
        images[((size_t)b * 4 + 0) * np + p] = o0;
        images[((size_t)b * 4 + 1) * np + p] = o1;
        images[((size_t)b * 4 + 2) * np + p] = o2;
        images[((size_t)b * 4 + 3) * np + p] = alpha;
    }
}

__global__ void k_p2f_finalize(const float* __restrict__ acc, float* __restrict__ p2f, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 a = reinterpret_cast<const float4*>(acc)[i];
    const float d = fmaxf(a.z, 1e-12f);  // soft_rasterize.py:73 clamp_min(1e-12)
    reinterpret_cast<float2*>(p2f)[i] = make_float2(a.x / d, a.y / d);
}

// =============================================================================================
// backward
// =============================================================================================
template <int RGB, bool TEXGRAD>
__global__ void __launch_bounds__(CTA, 3) k_raster_bwd(const float* __restrict__ rec_all,
                                                       const float4* __restrict__ box_all,
                                                       const float* __restrict__ textures,
                                                       const float* __restrict__ colors_hi,
                                                       const float* __restrict__ aggrs,
                                                       const float* __restrict__ grad_images,
                                                       float* __restrict__ grad_faces, float* __restrict__ grad_tex,
                                                       const uint32_t* __restrict__ ubox, Consts<float> K) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_rec = reinterpret_cast<float*>(smem_raw);
    float4* s_box = reinterpret_cast<float4*>(smem_raw + smem_box_off());
    uint16_t* s_list = reinterpret_cast<uint16_t*>(smem_raw + smem_list_off(K.F));
    __shared__ uint64_t s_bar;
    __shared__ int s_warp_cnt[NWARP];
    __shared__ float s_ext[4];
    __shared__ float s_g[CHUNK][9];  // per-(tile, chunk face) vertex-gradient partial sums

    const int tid = threadIdx.x, lane = tid & 31;
    const int b = blockIdx.z;
    const int S = K.S, F = K.F;
    const PixelMap pm = map_pixel(S);
    const int px = pm.px, py = pm.py;
    const bool live = pm.live;
    const float xp = pm.xp, yp = pm.yp;

    if (tid == 0) {
        mbar_init(&s_bar, 1);
        fence_mbar_init();
    }
    tile_extents(S, s_ext);
    for (int i = tid; i < CHUNK * 9; i += CTA) (&s_g[0][0])[i] = 0.f;
    __syncthreads();
    const float4* box = box_all + (size_t)b * F;
    if (tile_outside_union(ubox, b, s_ext)) return;  // uniform
    uint32_t bar_phase = 0;
    float g0 = 0, g1 = 0, g2 = 0, g3 = 0, C0 = 0, C1 = 0, C2 = 0, C3 = 0, ssum = 1, smax = 0;
    bool loaded = false;  // per-pixel inputs, read once the first window lists a face
    const float* tex_img = textures + (size_t)(b / K.tex_div) * K.tex_bs;
    float* gtex_img = TEXGRAD ? grad_tex + (size_t)(b / K.tex_div) * K.tex_bs : nullptr;
    for (int wb = 0; wb < F; wb += FACE_WINDOW) {
    const int n = build_tile_list(box + wb, min(F - wb, FACE_WINDOW), s_ext[0], s_ext[1], s_ext[2], s_ext[3], s_box, s_list,
                                  s_warp_cnt, &s_bar, bar_phase);
    if (n == 0) continue;  // uniform
    const float* rec_img = rec_all + ((size_t)b * F + wb) * REC_LEN;

    const int nchunk = (n + CHUNK - 1) / CHUNK;
    issue_chunk(rec_img, s_list, n, 0, s_rec);
    issue_chunk(rec_img, s_list, n, 1, s_rec);

    // per-pixel inputs
    const size_t np = (size_t)S * S;
    if (live && !loaded) {
        const size_t p = (size_t)py * S + px;
        if (K.aa) {  // avg_pool2d backward: g / 4
            const size_t nq = (size_t)K.IS * K.IS;
            const size_t q = (size_t)(py >> 1) * K.IS + (px >> 1);
            g0 = __ldg(grad_images + ((size_t)b * 4 + 0) * nq + q) * 0.25f;
            g1 = __ldg(grad_images + ((size_t)b * 4 + 1) * nq + q) * 0.25f;
            g2 = __ldg(grad_images + ((size_t)b * 4 + 2) * nq + q) * 0.25f;
            g3 = __ldg(grad_images + ((size_t)b * 4 + 3) * nq + q) * 0.25f;
        } else {
            g0 = __ldg(grad_images + ((size_t)b * 4 + 0) * np + p);
            g1 = __ldg(grad_images + ((size_t)b * 4 + 1) * np + p);
            g2 = __ldg(grad_images + ((size_t)b * 4 + 2) * np + p);
            g3 = __ldg(grad_images + ((size_t)b * 4 + 3) * np + p);
        }
        C0 = __ldg(colors_hi + ((size_t)b * 4 + 0) * np + p);
        C1 = __ldg(colors_hi + ((size_t)b * 4 + 1) * np + p);
        C2 = __ldg(colors_hi + ((size_t)b * 4 + 2) * np + p);
        C3 = __ldg(colors_hi + ((size_t)b * 4 + 3) * np + p);
        ssum = __ldg(aggrs + ((size_t)b * 2 + 0) * np + p);
        smax = __ldg(aggrs + ((size_t)b * 2 + 1) * np + p);
    }
    loaded = true;

    for (int c = 0; c < nchunk; ++c) {
        const int st = c % NSTAGE;
        const int cnt = min(CHUNK, n - c * CHUNK);
        cp_async_wait<1>();
        __syncthreads();  // chunk c visible to all; s_g is zero again
        const float* chunk = s_rec + (size_t)st * CHUNK * REC_LEN;
        float own[9];  // vertex-gradient partial sums of this warp: lane j owns chunk face j
#pragma unroll
        for (int k = 0; k < 9; ++k) own[k] = 0.f;
        bool own_any = false;
        float4 bb = *reinterpret_cast<const float4*>(chunk + R_BOX);
        for (int j = 0; j < cnt; ++j) {
            const float* rc = chunk + j * REC_LEN;
            const float4 bbn = *reinterpret_cast<const float4*>(chunk + (j + 1 < cnt ? j + 1 : j) * REC_LEN + R_BOX);
            float gv[9];
#pragma unroll
            for (int k = 0; k < 9; ++k) gv[k] = 0.f;
            bool contrib = false;
            if (live && !(xp > bb.y || xp < bb.x || yp > bb.w || yp < bb.z)) {
                Frag<float> fr;
                if (fragment_any(rc, xp, yp, K, fr)) {
                    // alpha: kernel.cu:577-585 (hard alpha passes the raw gradient through, as the reference does)
                    const float one_m_a = 1 - C3;
                    float Cxy;
                    if (K.alpha == UMR_ALPHA_PROD) {
                        Cxy = (one_m_a == 0.f || g3 == 0.f)
                                  ? g3 * one_m_a
                                  : (float)((double)g3 * ((double)one_m_a / fmax((double)(1 - fr.D), 1e-6)));
                    } else if (K.alpha == UMR_ALPHA_SUM) {
                        Cxy = g3 / K.F;
                    } else {
                        Cxy = g3;
                    }
                    float k0 = fr.w0, k1 = fr.w1, k2 = fr.w2;
                    clip_bary(k0, k1, k2);
                    const float zp = depth_of(rc, k0, k1, k2);
                    if (!(zp < K.near_ || zp > K.far_)) {  // :592 drops the alpha gradient as well
                        contrib = true;
                        const uint32_t flg = __float_as_uint(rc[R_FLG]);
                        const bool front = (flg & 8u) != 0;
                        const int f = wb + s_list[c * CHUNK + j];
                        float gz0 = 0.f, gz1 = 0.f, gz2 = 0.f;
                        if (RGB == 0) {
                            if ((float)f == smax) {  // aggrs[1] = winning face id (:596)
                                if (TEXGRAD)
                                    add_texture_grad(gtex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, 1.f, g0, g1, g2, false, TexRedSink());
                            }
                        } else if ((front || K.double_side) && (g0 != 0.f || g1 != 0.f || g2 != 0.f)) {
                            const float zn = (K.far_ - zp) / (K.far_ - K.near_);
                            const float s = fr.D * expf((zn - smax) / K.gamma) / ssum;  // :608
                            if (s != 0.f) {
                                if (TEXGRAD)
                                    add_texture_grad(gtex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, s, g0, g1, g2, true, TexRedSink());
                                float t0, t1, t2;
                                sample_texture(tex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, t0, t1, t2);
                                float Crgb = 0.f;
                                Crgb += g0 * (t0 - C0);
                                Crgb += g1 * (t1 - C1);
                                Crgb += g2 * (t2 - C2);
                                Crgb *= s;
                                if (Crgb != 0.f) {
                                    Cxy += Crgb / fr.D;
                                    const float Cz = Crgb / K.gamma / (K.near_ - K.far_) * zp * zp;  // :624
                                    gz0 = Cz * k0 / rc[2] / rc[2];
                                    gz1 = Cz * k1 / rc[5] / rc[5];
                                    gz2 = Cz * k2 / rc[8] / rc[8];
                                }
                            }
                        }
                        Cxy *= fr.D * (1 - fr.D) / K.sigma;  // :632
                        gv[2] = gz0; gv[5] = gz1; gv[8] = gz2;
                        if (K.dist == UMR_DIST_EUCLIDEAN) {
                            const float q = 2 * fr.sign * Cxy;  // :640
                            gv[0] = q * (fr.t0 + fr.w0) * fr.dx;
                            gv[1] = q * (fr.t0 + fr.w0) * fr.dy;
                            gv[3] = q * (fr.t1 + fr.w1) * fr.dx;
                            gv[4] = q * (fr.t1 + fr.w1) * fr.dy;
                            gv[6] = q * (fr.t2 + fr.w2) * fr.dx;
                            gv[7] = q * (fr.t2 + fr.w2) * fr.dy;
                        } else if (K.dist == UMR_DIST_BARYCENTRIC) {  // kernel.cu:162-176
                            const float w0 = fr.t0, w1 = fr.t1, w2 = fr.t2;  // unclipped barycentrics
                            const int pidx = w0 > w1 ? (w1 > w2 ? 2 : 1) : (w0 > w2 ? 2 : 0);
                            const double scale = fr.dis > 0 ? (2. * (double)sqrtf(fr.dis)) : (2. * (double)sqrtf(-fr.dis));
#pragma unroll
                            for (int l = 0; l < 2; ++l) {
                                const float ip = rc[R_INV + 3 * pidx + l];
#pragma unroll
                                for (int k = 0; k < 3; ++k) {
                                    float gkl = 0.f;
                                    gkl += -ip * rc[R_INV + 3 * k + 0] * xp;
                                    gkl += -ip * rc[R_INV + 3 * k + 1] * yp;
                                    gkl += -ip * rc[R_INV + 3 * k + 2] * 1.f;
                                    gv[3 * k + l] = (float)((double)(gkl * Cxy) * scale);
                                }
                            }
                        }
                    }
                }
            }
            // 9 vertex gradients: warp-shuffle reduction instead of the reference's 9 global atomics per
            // (pixel, face) (kernel.cu:645-654); totals stay in the registers of lane j
            if (__any_sync(0xffffffffu, contrib)) {
#pragma unroll
                for (int k = 0; k < 9; ++k) gv[k] = warp_sum(gv[k]);
                if (lane == j) {
#pragma unroll
                    for (int k = 0; k < 9; ++k) own[k] += gv[k];
                    own_any = true;
                }
            }
            bb = bbn;
        }
        if (own_any) {  // one shared atomic per (warp, face, component)
#pragma unroll
            for (int k = 0; k < 9; ++k) red_add_shared(&s_g[lane][k], own[k]);
        }
        __syncthreads();  // everyone is done with stage st; s_g is complete
        for (int i = tid; i < cnt * 9; i += CTA) {  // one global atomic per (tile, face, component)
            const float v = (&s_g[0][0])[i];
            if (v != 0.f) {
                const int j = i / 9, k = i - j * 9;
                red_add_global(grad_faces + ((size_t)b * F + wb + s_list[c * CHUNK + j]) * 9 + k, v);
                (&s_g[0][0])[i] = 0.f;
            }
        }
        issue_chunk(rec_img, s_list, n, c + NSTAGE, s_rec);
    }
    }
}


// =============================================================================================
// backward, pair-parallel formulation
//
// The backward of a (pixel, face) pair depends only on per-pixel constants (incoming gradient, final
// colour/alpha, softmax sum/max) and the face record: there is NO ordering constraint.  So instead of
// binding a thread to a pixel and walking the face list (lanes idle whenever the face's cull box misses
// their pixel: 46 % lane utilisation, and warps of a tile finish at very different times), the tile's
// work is flattened to the list of candidate pairs: for every chunk face the cull box selects a
// RECTANGLE of tile pixels (pixel-centre coordinates are monotone), the rectangle sizes are prefix-summed
// and thread t evaluates pairs t, t+256, ...  All lanes work (until the distance cull), all warps of the
// CTA carry the same load, and the 9 vertex gradients are combined by a segmented warp reduction (lanes
// are sorted by face) followed by one shared atomic per (warp, face, component).
// =============================================================================================
// Register-lean variant used by the pair-parallel kernel: the 10 per-pixel inputs stay in shared memory
// (sp = &s_pix[0][pix], plane stride PT*PT) and are fetched where they are consumed, and the 9 gradients are
// added straight into the caller's accumulators -- this keeps the kernel at <= 64 registers (4 CTAs/SM).
// SPLIT (the split backward, softmax only): the vertex gradients keep only the terms driven by the alpha adjoint g3; the texel
// gradients are formed from the colour adjoints as always.  Skipping the colour terms leaves every other expression as it is,
// so the vertex gradients equal, bit for bit, those of the same pairs with zero colour adjoints.
// RGB_SIL (the silhouette backward): the alpha terms alone, from the staged g_alpha and alpha planes (PixPlanes).
// (Declared with its default arguments in raster_generic.cuh, for the deterministic gather.)
template <int RGB, bool TEXGRAD, int NC, class Sink, bool SPLIT>
__device__ __forceinline__ bool bwd_pair_acc(const float* __restrict__ rc, float xp, float yp, const Consts<float>& K,
                                             const float* __restrict__ sp, int f, const float* __restrict__ tex_img,
                                             float* __restrict__ gtex_img, float* acc, Sink sink) {
    Frag<float> fr;
    if (!fragment(rc, xp, yp, K.thr, K.sigma, fr)) return false;
    using PP = PixPlanes<RGB, NC>;
    constexpr int NP = PT * PT, NPL = PP::NPL, NV = PP::NV;  // planes: g[NC], g_alpha, C[NC], alpha, ssum, smax
    const float g3 = sp[PP::GA * NP];
    const float one_m_a = 1 - sp[PP::AL * NP];
    float Cxy = (one_m_a == 0.f || g3 == 0.f)
                    ? g3 * one_m_a
                    : (float)((double)g3 * ((double)one_m_a / fmax((double)(1 - fr.D), 1e-6)));
    float k0 = fr.w0, k1 = fr.w1, k2 = fr.w2;
    clip_bary(k0, k1, k2);
    const float zp = depth_of(rc, k0, k1, k2);
    if (zp < K.near_ || zp > K.far_) return false;
    const uint32_t flg = __float_as_uint(rc[R_FLG]);
    const bool front = (flg & 8u) != 0;
    if (RGB == 0) {
        if ((float)f == sp[(NV - 1) * NP]) {
            if (TEXGRAD) {
                float* gt = gtex_img + ((size_t)f * K.T2 + texel_index(k0, k1, K.R)) * NC;
                if (NC == 3) {
                    sink.add3(gt, sp[0], sp[NP], sp[2 * NP]);
                } else {
#pragma unroll
                    for (int c = 0; c < NC; ++c) red_add_global(gt + c, sp[c * NP]);
                }
            }
        }
    } else if (RGB == 1 && (front || K.double_side)) {
        float g[NC];
        bool any = false;
#pragma unroll
        for (int c = 0; c < NC; ++c) { g[c] = sp[c * NP]; any = any || g[c] != 0.f; }
        if (any) {
            const float zn = (K.far_ - zp) / (K.far_ - K.near_);
            const float s = fr.D * expf((zn - sp[(NV - 1) * NP]) / K.gamma) / sp[(NV - 2) * NP];
            if (s != 0.f) {
                const size_t to = ((size_t)f * K.T2 + texel_index(k0, k1, K.R)) * NC;
                if (TEXGRAD) {
                    if (NC == 3) {
                        sink.add3(gtex_img + to, s * g[0], s * g[1], s * g[2]);
                    } else {
#pragma unroll
                        for (int c = 0; c < NC; ++c) red_add_global(gtex_img + to + c, s * g[c]);
                    }
                }
                if (!SPLIT) {
                    float Crgb = 0.f;
#pragma unroll
                    for (int c = 0; c < NC; ++c) Crgb += g[c] * (__ldg(tex_img + to + c) - sp[(NPL + c) * NP]);
                    Crgb *= s;
                    if (Crgb != 0.f) {
                        Cxy += Crgb / fr.D;
                        const float Cz = Crgb / K.gamma / (K.near_ - K.far_) * zp * zp;
                        acc[2] += Cz * k0 / rc[2] / rc[2];
                        acc[5] += Cz * k1 / rc[5] / rc[5];
                        acc[8] += Cz * k2 / rc[8] / rc[8];
                    }
                }
            }
        }
    }
    Cxy *= fr.D * (1 - fr.D) / K.sigma;
    const float q = 2 * fr.sign * Cxy;
    acc[0] += q * (fr.t0 + fr.w0) * fr.dx;
    acc[1] += q * (fr.t0 + fr.w0) * fr.dy;
    acc[3] += q * (fr.t1 + fr.w1) * fr.dx;
    acc[4] += q * (fr.t1 + fr.w1) * fr.dy;
    acc[6] += q * (fr.t2 + fr.w2) * fr.dx;
    acc[7] += q * (fr.t2 + fr.w2) * fr.dy;
    return true;
}

// One PT x PT tile of the recompute backward (bx, by, b = tile column / row / image).  Every early exit is CTA-uniform.
// `bar_phase` carries the mbarrier parity across the tiles a CTA processes (list-driven launch).  SPLIT: see bwd_pair_acc.
template <int RGB, bool TEXGRAD, int NC = 3, bool SPLIT = false>
__device__ __forceinline__ void bwd_pairs_tile(const float* __restrict__ rec_all, const float4* __restrict__ box_all,
                                               const float* __restrict__ textures, const float* __restrict__ colors_hi,
                                               const float* __restrict__ aggrs, const float* __restrict__ grad_images,
                                               float* __restrict__ grad_faces, float* __restrict__ grad_tex,
                                               const uint32_t* __restrict__ ubox, const Consts<float>& K, int bx, int by, int b,
                                               uint64_t* s_bar_p, uint32_t& bar_phase) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_rec = reinterpret_cast<float*>(smem_raw);
    float4* s_box = reinterpret_cast<float4*>(smem_raw + smem_box_off());
    uint16_t* s_list = reinterpret_cast<uint16_t*>(smem_raw + smem_list_off(K.F));
    __shared__ int s_warp_cnt[NWARP];
    __shared__ float s_ext[4];
    // PT x PT pixel tile.
    using PP = PixPlanes<RGB, NC>;
    constexpr int NPL = PP::NPL, NV = PP::NV;
    __shared__ float s_pix[NV][PT * PT];   // g[NC], g_alpha, C[NC], alpha, ssum, smax of the tile's pixels (row-major; PixPlanes)
    __shared__ float s_xp[PT], s_yp[PT];
    __shared__ unsigned int s_cm[CHUNK], s_rm[CHUNK];  // column / row pass masks of the chunk faces
    __shared__ int s_off[CHUNK + 1];                  // prefix sums of the rectangle sizes
    __shared__ uint32_t s_geo[CHUNK];                 // cx0 | w<<8 | ry0<<16 | rcp(w)<<... (see below)
    __shared__ uint32_t s_rcpw[CHUNK];
    uint64_t& s_bar = *s_bar_p;

    const int tid = threadIdx.x, lane = tid & 31;
    const int S = K.S, F = K.F;
    const int x0 = bx * PT, y0 = by * PT;

    tile_extents_at(S, s_ext, PT, bx, by);
    if (tid < PT) s_xp[tid] = pixel_coord(x0 + tid, S);
    else if (tid < 2 * PT) s_yp[tid - PT] = pixel_coord(S - 1 - (y0 + tid - PT), S);
    __syncthreads();
    if (tile_outside_union(ubox, b, s_ext)) return;  // uniform
    const float4* box = box_all + (size_t)b * F;
    const float* tex_img = textures + (size_t)(b / K.tex_div) * K.tex_bs;
    float* gtex_img = TEXGRAD ? grad_tex + (size_t)(b / K.tex_div) * K.tex_bs : nullptr;
    for (int wb = 0; wb < F; wb += FACE_WINDOW) {
    const int n = build_tile_list(box + wb, min(F - wb, FACE_WINDOW), s_ext[0], s_ext[1], s_ext[2], s_ext[3], s_box, s_list,
                                  s_warp_cnt, &s_bar, bar_phase);
    if (n == 0) continue;  // uniform
    const float* rec_img = rec_all + ((size_t)b * F + wb) * REC_LEN;

    const int nchunk = (n + CHUNK - 1) / CHUNK;
    issue_chunk(rec_img, s_list, n, 0, s_rec);
    issue_chunk(rec_img, s_list, n, 1, s_rec);

    // per-pixel inputs -> shared (row-major, PT*PT/CTA pixels per thread, coalesced rows); rewritten per window (the
    // chunk loop's barriers order it against the previous window's readers)
    for (int pi = tid; pi < PT * PT; pi += CTA) {
        const int px = x0 + (pi % PT), py = y0 + (pi / PT);
        const size_t np = (size_t)S * S;
        float v[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) v[k] = (!PP::SIL && k == NV - 2) ? 1.f : 0.f;
        if (px < S && py < S) {
            const size_t p = (size_t)py * S + px;
            if (K.aa) {  // avg_pool2d backward: g / 4
                const size_t nq = (size_t)K.IS * K.IS;
                const size_t q = (size_t)(py >> 1) * K.IS + (px >> 1);
#pragma unroll
                for (int k = 0; k < NPL; ++k) v[k] = __ldg(grad_images + ((size_t)b * NPL + k) * nq + q) * 0.25f;
            } else {
#pragma unroll
                for (int k = 0; k < NPL; ++k) v[k] = __ldg(grad_images + ((size_t)b * NPL + k) * np + p);
            }
#pragma unroll
            for (int k = 0; k < NPL; ++k) v[NPL + k] = __ldg(colors_hi + ((size_t)b * NPL + k) * np + p);
            if (!PP::SIL) {
                v[NV - 2] = __ldg(aggrs + ((size_t)b * 2 + 0) * np + p);
                v[NV - 1] = __ldg(aggrs + ((size_t)b * 2 + 1) * np + p);
            }
        }
#pragma unroll
        for (int k = 0; k < NV; ++k) s_pix[k][pi] = v[k];
    }
    const int ncol = min(PT, S - x0), nrow = min(PT, S - y0);  // live extent of the tile

    for (int c = 0; c < nchunk; ++c) {
        const int st = c % NSTAGE;
        const int cnt = min(CHUNK, n - c * CHUNK);
        if (tid < CHUNK) { s_cm[tid] = 0u; s_rm[tid] = 0u; }
        cp_async_wait<1>();
        __syncthreads();  // chunk c (and s_pix on the first pass) visible; masks zeroed; s_g zero
        const float* chunk = s_rec + (size_t)st * CHUNK * REC_LEN;
        // ---- rectangles: thread (j = tid & 31, part = tid >> 5) tests 4 columns or 4 rows of face j
        {
            const int j = tid & 31, part = tid >> 5;
            if (j < cnt) {
                const float4 bb = *reinterpret_cast<const float4*>(chunk + j * REC_LEN + R_BOX);
                unsigned m = 0;
                constexpr int PER = PT / 4;  // columns (or rows) tested per thread
                if (part < 4) {
#pragma unroll
                    for (int i = 0; i < PER; ++i) {
                        const int cidx = part * PER + i;
                        const float x = s_xp[cidx];
                        if (cidx < ncol && !(x > bb.y || x < bb.x)) m |= 1u << cidx;
                    }
                    if (m) atomicOr(&s_cm[j], m);
                } else {
#pragma unroll
                    for (int i = 0; i < PER; ++i) {
                        const int ridx = (part - 4) * PER + i;
                        const float y = s_yp[ridx];
                        if (ridx < nrow && !(y > bb.w || y < bb.z)) m |= 1u << ridx;
                    }
                    if (m) atomicOr(&s_rm[j], m);
                }
            }
        }
        __syncthreads();
        if (tid < 32) {  // warp 0: rectangle sizes -> exclusive prefix sums
            const unsigned cm = tid < cnt ? s_cm[tid] : 0u, rm = tid < cnt ? s_rm[tid] : 0u;
            const int w = __popc(cm), h = __popc(rm);
            const int size = w * h;
            int incl = size;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int o = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += o;
            }
            s_off[tid + 1] = incl;
            if (tid == 0) s_off[0] = 0;
            // masks are contiguous intervals (pixel-centre coordinates are monotone)
            const int cx0 = cm ? __ffs(cm) - 1 : 0, ry0 = rm ? __ffs(rm) - 1 : 0;
            s_geo[tid] = (uint32_t)cx0 | ((uint32_t)(w ? w : 1) << 8) | ((uint32_t)ry0 << 16);
            s_rcpw[tid] = (65536u + (uint32_t)(w ? w : 1) - 1u) / (uint32_t)(w ? w : 1);  // exact floor(l/w), l < 1024, w <= 32
        }
        __syncthreads();
        const int T = s_off[cnt];
        // Each warp owns a contiguous run [wbeg, wend) of the chunk's pairs and walks it face by face, so
        // inside the inner loop all lanes work on the same face: the 9 vertex gradients are accumulated
        // privately and combined ONCE per (warp, face) with a shuffle reduction + 9 global REDs (shared
        // float atomics are CAS loops on this architecture and are avoided in the hot path).
        {
            const int warp = tid >> 5;
            const int per_warp = ((T + NWARP * 32 - 1) / (NWARP * 32)) * 32;
            const int wbeg = min(T, warp * per_warp), wend = min(T, (warp + 1) * per_warp);
            int j = 0;
            if (wbeg < wend) {
#pragma unroll
                for (int sft = 16; sft > 0; sft >>= 1) {
                    const int t = j + sft;
                    if (t < cnt && s_off[t] <= wbeg) j = t;
                }
            }
            for (; j < cnt && s_off[j] < wend; ++j) {
                const int fbeg = s_off[j], fend = s_off[j + 1];
                const int lo = max(wbeg, fbeg), hi = min(wend, fend);
                if (lo >= hi) continue;  // empty rectangle
                const uint32_t geo = s_geo[j];
                const int cx0 = (int)(geo & 0xff), w = (int)((geo >> 8) & 0xff), ry0 = (int)(geo >> 16);
                const uint32_t rcpw = s_rcpw[j];
                const float* rc = chunk + j * REC_LEN;
                const int f = wb + (int)s_list[c * CHUNK + j];
                float acc[9];
#pragma unroll
                for (int k = 0; k < 9; ++k) acc[k] = 0.f;
                bool acc_any = false;
                for (int p = lo + lane; p < hi; p += 32) {
                    const int local = p - fbeg;
                    const int lr = (int)(((uint32_t)local * rcpw) >> 16);
                    const int col = cx0 + (local - lr * w);
                    const int row = ry0 + lr;
                    const int pix = row * PT + col;
                    if (bwd_pair_acc<RGB, TEXGRAD, NC, TexRedSink, SPLIT>(rc, s_xp[col], s_yp[row], K, &s_pix[0][pix], f, tex_img,
                                                                          gtex_img, acc))
                        acc_any = true;
                }
                if (__any_sync(0xffffffffu, acc_any)) {
#pragma unroll
                    for (int k = 0; k < 9; ++k) acc[k] = warp_sum(acc[k]);
                    if (lane < 9) {
                        float v = acc[0];
#pragma unroll
                        for (int k = 1; k < 9; ++k) v = (lane == k) ? acc[k] : v;
                        if (v != 0.f && grad_faces != nullptr) red_add_global(grad_faces + ((size_t)b * F + f) * 9 + lane, v);
                    }
                }
            }
        }
        __syncthreads();  // everyone is done with stage st
        issue_chunk(rec_img, s_list, n, c + NSTAGE, s_rec);
    }
    }
    cp_async_wait<0>();
    __syncthreads();  // shared memory reusable by the next tile of this CTA (list-driven launch)
}


// full grid: one CTA per tile (no pair buffer: every tile is recomputed)
template <int RGB, bool TEXGRAD, int NC = 3, bool SPLIT = false>
__global__ void __launch_bounds__(CTA, 3) k_raster_bwd_pairs(const float* __restrict__ rec_all, const float4* __restrict__ box_all,
                                                             const float* __restrict__ textures, const float* __restrict__ colors_hi,
                                                             const float* __restrict__ aggrs, const float* __restrict__ grad_images,
                                                             float* __restrict__ grad_faces, float* __restrict__ grad_tex,
                                                             const uint32_t* __restrict__ ubox, Consts<float> K) {
    __shared__ uint64_t s_bar;
    if (threadIdx.x == 0) {
        mbar_init(&s_bar, 1);
        fence_mbar_init();
    }
    uint32_t phase = 0;  // (bwd_pairs_tile synchronises the CTA before the barrier is first used)
    bwd_pairs_tile<RGB, TEXGRAD, NC, SPLIT>(rec_all, box_all, textures, colors_hi, aggrs, grad_images, grad_faces, grad_tex, ubox,
                                        K, (int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z, &s_bar, phase);
}

// list-driven: with a pair buffer, only the tiles the forward could NOT save are recomputed.  The forward appended
// their ids to `ulist` (count in *ucount); a small persistent grid walks the list, so a render whose tiles were all
// saved pays one near-empty launch instead of one CTA per tile (35 us at C2 with the full grid).
template <int RGB, bool TEXGRAD, int NC = 3, bool SPLIT = false>
__global__ void __launch_bounds__(CTA, 3) k_raster_bwd_pairs_list(const float* __restrict__ rec_all, const float4* __restrict__ box_all,
                                                                  const float* __restrict__ textures, const float* __restrict__ colors_hi,
                                                                  const float* __restrict__ aggrs, const float* __restrict__ grad_images,
                                                                  float* __restrict__ grad_faces, float* __restrict__ grad_tex,
                                                                  const uint32_t* __restrict__ ubox, Consts<float> K,
                                                                  const uint32_t* __restrict__ ucount, const int32_t* __restrict__ ulist,
                                                                  int tiles_x, int tiles_y) {
    const uint32_t nu = __ldg(ucount);
    if (blockIdx.x >= nu) return;
    __shared__ uint64_t s_bar;
    if (threadIdx.x == 0) {
        mbar_init(&s_bar, 1);
        fence_mbar_init();
    }
    uint32_t phase = 0;
    for (uint32_t i = blockIdx.x; i < nu; i += gridDim.x) {
        const int t = __ldg(ulist + i);
        const int bx = t % tiles_x, by = (t / tiles_x) % tiles_y, b = t / (tiles_x * tiles_y);
        bwd_pairs_tile<RGB, TEXGRAD, NC, SPLIT>(rec_all, box_all, textures, colors_hi, aggrs, grad_images, grad_faces, grad_tex,
                                            ubox, K, bx, by, b, &s_bar, phase);
    }
}

// =============================================================================================
// deterministic mode (DESIGN.md §3)
// =============================================================================================
__device__ __forceinline__ double fixed_value(const unsigned long long* l) {
    double v = 0.0;
#pragma unroll
    for (int k = P2F_LIMBS - 1; k >= 0; --k) v += ldexp((double)(long long)l[k], k * P2F_LIMB_BITS - P2F_FRAC_BITS);
    return v;
}

// k_p2f_finalize over the fixed-point accumulators: the same clamp and divisions
__global__ void k_p2f_finalize_det(const unsigned long long* __restrict__ acc, float* __restrict__ p2f, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long* a = acc + i * P2F_DET_WORDS;
    if (a[3 * P2F_LIMBS] != 0ull) {
        reinterpret_cast<float2*>(p2f)[i] = make_float2(__int_as_float(0x7fffffff), __int_as_float(0x7fffffff));
        return;
    }
    const float x = (float)fixed_value(a), y = (float)fixed_value(a + P2F_LIMBS), w = (float)fixed_value(a + 2 * P2F_LIMBS);
    const float d = fmaxf(w, 1e-12f);  // soft_rasterize.py:73 clamp_min(1e-12)
    reinterpret_cast<float2*>(p2f)[i] = make_float2(x / d, y / d);
}

}  // namespace umr

#include "raster_stream.cuh"
#include "raster_fwd3.cuh"
#include "raster_fwd4.cuh"

#include "raster_host.cuh"

// =============================================================================================
// C ABI
// =============================================================================================
using namespace umr;

// Which forward serves the UMR configuration: 4 = k_raster_fwd4 (32x32 tiles, dynamic 8x4 pixel blocks; tile list in
// shared memory sized by F, longer coarse lists take a windowed slow path), 3 = k_raster_fwd3 (16x16 tiles, windowed
// list: any F).  Forward and backward must agree (the pair records' pixel index is relative to the forward's tile).
// Unless tile_mode = 32 asks for it, the 16x16-tile kernel: at C2 (16 x 512^2) only ~1600 of the 32x32-tile kernel's
// 4096 tiles carry work, a few waves of heavy CTAs at 4 per SM.  The 32x32 kernel stays available (tested at every
// shape), but does not earn a heuristic.
static int forward_impl(int tile_mode) { return tile_mode == 32 ? 4 : 3; }

extern "C" size_t umr_raster_workspace_bytes(int32_t B, int32_t F, int32_t image_size, int32_t anti_aliasing) {
    if (B <= 0 || F <= 0 || image_size <= 0) return 0;
    return ws_layout(B, F, image_size * (anti_aliasing ? 2 : 1)).total;
}

// Reserves PAIR_BLOCK_RESERVE bytes per block where a block takes BLK_F4 * 16 + 4 = 1028: callers size the buffer from
// an estimate of the blocks a render wants, and the extra capacity keeps renders denser than the estimate off the
// recompute path without growing the buffer.
constexpr size_t PAIR_BLOCK_RESERVE = 1540;
extern "C" size_t umr_raster_pair_buffer_bytes(int32_t B, int32_t image_size, int32_t anti_aliasing,
                                               uint64_t capacity_blocks) {
    if (B <= 0 || image_size <= 0) return 0;
    const size_t blk = (size_t)BLK_F4 * sizeof(float4) + sizeof(uint32_t);
    return pair_layout(B, image_size * (anti_aliasing ? 2 : 1), (size_t)capacity_blocks).total +
           (size_t)capacity_blocks * (PAIR_BLOCK_RESERVE - blk) + 1024;
}

// Texel-index bits of a pair record's meta word: pixel index below, front flag in bit 31.  16x16 tiles (k_raster_fwd3,
// also the 4-channel render) keep 8 pixel bits, 32x32 tiles (k_raster_fwd4) 10.
static int pair_texel_bits(const UmrRasterParams* p) {
    return (p->color_channels != 4 && forward_impl(p->tile_mode) == 4) ? 21 : 23;
}

// device pointers into the caller's pair buffer (cap == 0: no saving; also when T2 does not fit the record's texel field,
// so the backward recomputes every tile)
static PairBuf make_pairbuf(const UmrRasterParams* p, int S) {
    PairBuf pb{};
    if (!p->pair_buffer || p->pair_buffer_bytes == 0 || ((uintptr_t)p->pair_buffer & 255) != 0) return pb;
    if (p->texture_size > (1 << pair_texel_bits(p))) return pb;
    size_t cap = pair_capacity(p->batch_size, S, (size_t)p->pair_buffer_bytes);
    if (cap > 0x7fff0000u) cap = 0x7fff0000u;
    if (cap < 4) return pb;
    const PairBufLayout L = pair_layout(p->batch_size, S, cap);
    char* base = (char*)p->pair_buffer;
    pb.ctrl = (uint32_t*)(base + L.ctrl_off);
    pb.tile_head = (int32_t*)(base + L.head_off);
    pb.ulist = (int32_t*)(base + L.ulist_off);
    pb.blk_hdr = (uint32_t*)(base + L.hdr_off);
    pb.recs = (float4*)(base + L.rec_off);
    pb.cap = (uint32_t)cap;
    return pb;
}

// raster pixels per texel of the mesh, S^2 / (F * T2), from which the warp-level texel pre-reduction of k_raster_bwd2 is on.
// It only pays for very large faces; every UMR shape is far below the thresholds (6 at C2, 23 at C5, 91 at C3), where the
// plain vector REDs are faster.
constexpr double TEXGRAD_PRE_RATIO_FULL = 160.0, TEXGRAD_PRE_RATIO_TEXONLY = 120.0;

// Opt every raster kernel into the full dynamic shared-memory range ONCE per device (not per call:
// the call may be inside a CUDA-graph capture).  A 65536-face window needs 8 KB + 32 KB + 128 KB.  Every kernel
// launched with raster_dyn_smem (launch_pairs_backward's recompute kernels for each RGBM, TG, NC and SP it is called
// with, the generic forward and backward) must be listed: without the opt-in, static plus dynamic shared memory is
// capped at 48 KB, which the 4-channel recompute kernels pass from 1544 faces.
static int ensure_smem_attrs() {
    static bool done[64] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    if (dev < 0 || dev >= 64 || done[dev]) return 0;
    int optin = 0;
    e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (e != cudaSuccess) return (int)e;
    const void* const kernels[] = {
        (const void*)k_raster_fwd<0>, (const void*)k_raster_fwd<1>, (const void*)k_raster_fwd<1, true>,
        (const void*)k_raster_fwd4<0>, (const void*)k_raster_fwd4<1>,
        (const void*)k_raster_fwd4<0, uint32_t>, (const void*)k_raster_fwd4<1, uint32_t>,
        (const void*)k_raster_bwd<0, false>, (const void*)k_raster_bwd<0, true>,
        (const void*)k_raster_bwd<1, false>, (const void*)k_raster_bwd<1, true>,
        (const void*)k_raster_bwd_pairs<0, false>, (const void*)k_raster_bwd_pairs<0, true>,
        (const void*)k_raster_bwd_pairs<1, false>, (const void*)k_raster_bwd_pairs<1, true>,
        (const void*)k_raster_bwd_pairs_list<0, false>, (const void*)k_raster_bwd_pairs_list<0, true>,
        (const void*)k_raster_bwd_pairs_list<1, false>, (const void*)k_raster_bwd_pairs_list<1, true>,
        (const void*)k_raster_bwd_pairs<1, true, 3, true>, (const void*)k_raster_bwd_pairs_list<1, true, 3, true>,
        (const void*)k_raster_bwd_pairs<1, false, 4>, (const void*)k_raster_bwd_pairs_list<1, false, 4>,
        (const void*)k_raster_fwd4<RGB_SIL>, (const void*)k_raster_fwd4<RGB_SIL, uint32_t>,
        (const void*)k_raster_bwd_pairs<RGB_SIL, false>, (const void*)k_raster_bwd_pairs_list<RGB_SIL, false>,
    };
    for (const void* k : kernels) {
        cudaFuncAttributes fa;
        e = cudaFuncGetAttributes(&fa, k);
        if (e != cudaSuccess) return (int)e;
        e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
        if (e != cudaSuccess) return (int)e;
    }
    done[dev] = true;
    return 0;
}

// SM count of the current device, queried once per device
static int sm_count(int* sms) {
    static int cache[64] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    if (dev >= 0 && dev < 64 && cache[dev] > 0) {
        *sms = cache[dev];
        return 0;
    }
    e = cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return (int)e;
    if (dev >= 0 && dev < 64) cache[dev] = *sms;
    return 0;
}

static size_t raster_dyn_smem(int F) {
    const int W = F < FACE_WINDOW ? F : FACE_WINDOW;
    return smem_list_off(F) + (((size_t)W * 2 + 15) & ~(size_t)15);
}

// Deterministic-mode workspace: the default layout, then the fixed-point p2f accumulators (P2F_DET_WORDS int64 per face).
static size_t det_acc_bytes(int B, int F) { return align256((size_t)B * F * P2F_DET_WORDS * sizeof(unsigned long long)); }

extern "C" size_t umr_raster_workspace_bytes_deterministic(int32_t B, int32_t F, int32_t image_size, int32_t anti_aliasing) {
    if (B <= 0 || F <= 0 || image_size <= 0) return 0;
    return umr_raster_workspace_bytes(B, F, image_size, anti_aliasing) + det_acc_bytes(B, F);
}

// What a float32 call derives from its parameters and workspace.  The pair backward's tiles are the forward's 16x16 ones.
static_assert(PT == TILE, "grid16 serves the 16x16-tile forward and the pair backward");
struct RasterCall {
    const UmrRasterParams* p;
    cudaStream_t stream;
    int B, F, S;
    bool wide;     // F > NARROW_MAX_FACES: the 32-bit face-index instantiations
    bool gen;      // a generic mode (is_generic)
    bool softmax;  // softmax colours (else hard)
    bool nc4;      // the 4-channel part-map render
    Consts<float> K;
    WorkspaceLayout L;
    float* rec;
    float4* box;
    uint32_t* ubox;
    int* ccount;
    void* clist;
    PairBuf pb;          // cap == 0: no pair records saved or read
    dim3 grid16, grid32;  // 16x16 and 32x32 tiles of the raster
    int ncb;             // coarse bins per raster side
};

// pairs: the call may use the caller's pair buffer (the default mode in UMR's configuration)
static RasterCall raster_call(const UmrRasterParams* p, void* workspace, void* stream, bool pairs) {
    RasterCall c;
    c.p = p;
    c.stream = (cudaStream_t)stream;
    c.K = make_consts<float>(p);
    c.B = p->batch_size;
    c.F = p->num_faces;
    c.S = c.K.S;
    c.wide = c.F > NARROW_MAX_FACES;
    c.gen = is_generic(p);
    c.softmax = p->func_id_rgb == UMR_RGB_SOFTMAX;
    c.nc4 = p->color_channels == 4;
    c.L = ws_layout(c.B, c.F, c.S);
    char* ws = (char*)workspace;
    c.rec = (float*)(ws + c.L.rec_off);
    c.box = (float4*)(ws + c.L.box_off);
    c.ubox = (uint32_t*)(ws + c.L.ubox_off);
    c.ccount = (int*)(ws + c.L.ccount_off);
    c.clist = ws + c.L.clist_off;
    c.pb = pairs ? make_pairbuf(p, c.S) : PairBuf{};
    c.grid16 = dim3((c.S + TILE - 1) / TILE, (c.S + TILE - 1) / TILE, c.B);
    c.grid32 = dim3((c.S + T4 - 1) / T4, (c.S + T4 - 1) / T4, c.B);
    c.ncb = (c.S + CB - 1) / CB;
    return c;
}

// The face records and the images' union cull boxes (zeroed first).  only_if_nonzero: k_prep returns at once when the
// word it points to is 0 (records that only the recompute fallback reads, and no tile left for it).
static int prep(const RasterCall& c, const float* face_vertices, const uint32_t* only_if_nonzero) {
    cudaError_t e = cudaMemsetAsync(c.ubox, 0, (size_t)c.B * 4 * sizeof(uint32_t), c.stream);
    if (e != cudaSuccess) return (int)e;
    launch(k_prep, dim3((c.F + 255) / 256, c.B), 256, 0, c.stream, face_vertices, c.rec, c.box, c.ubox, c.F,
           sqrtf(c.K.thr), only_if_nonzero);  // r: kernel.cu:355 sqrt(threshold) in float
    return 0;
}

// Coarse binning for the UMR-configuration kernels, after the pair buffer's counters are reset: u16 lists of F entries per
// bin, or (F > 65535) the wide pool, whose cursor is reset first.
static int bin_coarse(const RasterCall& c) {
    cudaError_t e = c.pb.cap > 0 ? cudaMemsetAsync(c.pb.ctrl, 0, 16, c.stream) : cudaSuccess;
    if (e != cudaSuccess) return (int)e;
    const dim3 grid(c.ncb, c.ncb, c.B);
    const size_t smem = (size_t)(c.F < BOX_PIECE ? c.F : BOX_PIECE) * 16;
    if (!c.wide) {
        launch(k_bin_coarse<uint16_t>, grid, CTA, smem, c.stream, c.box, c.ubox, (uint16_t*)c.clist, c.ccount, c.F, c.S,
               (size_t)0);
        return 0;
    }
    e = cudaMemsetAsync(c.ccount + 2 * (size_t)c.B * c.ncb * c.ncb, 0, sizeof(unsigned long long), c.stream);
    if (e != cudaSuccess) return (int)e;
    launch(k_bin_coarse<uint32_t>, grid, CTA, smem, c.stream, c.box, c.ubox, (uint32_t*)c.clist, c.ccount, c.F, c.S,
           c.L.clist_cap);
    return 0;
}

// f(IdxT{}) with the face-index type of the UMR-configuration kernels
template <class Fn>
static void with_index(bool wide, Fn&& f) {
    if (wide) f(uint32_t{});
    else f(uint16_t{});
}

// grid of the recompute backward's list-driven launch: 3 resident CTAs per SM walk the unsaved-tile list
static int list_grid(const RasterCall& c, unsigned* grid) {
    int sms = 0;
    int rc = sm_count(&sms);
    if (rc) return rc;
    const size_t ntiles = (size_t)c.grid16.x * c.grid16.y * c.B, list_max = (size_t)3 * sms;
    *grid = (unsigned)(ntiles < list_max ? ntiles : list_max);
    return 0;
}

// zero the gradients the backward accumulates into (NULL: not computed, or written whole)
static int zero_grads(const RasterCall& c, float* grad_faces, float* grad_textures) {
    const size_t n = (size_t)c.B * c.F;
    cudaError_t e = grad_faces ? cudaMemsetAsync(grad_faces, 0, n * 9 * sizeof(float), c.stream) : cudaSuccess;
    if (e == cudaSuccess && grad_textures)
        e = cudaMemsetAsync(grad_textures, 0, (n / c.K.tex_div) * c.p->texture_size * 3 * sizeof(float), c.stream);
    return (int)e;
}

// the buffers of a float backward kernel (a silhouette's: its alpha plane and alpha gradient only)
struct BwdArgs {
    const float *textures, *colors_hi, *aggrs, *grad_images;
    float *grad_faces, *grad_tex;
};

// k_raster_bwd2 for the call: texture-only (grad_faces == NULL) and warp-level texel pre-reduction variants exist for the
// texture-gradient kernels only, the pre-reduction for softmax colours only; SP: the split backward (softmax, both gradients)
template <int RGBM, bool TG, int NC, bool SP, int TS, typename IdxT>
static void launch_bwd2(const RasterCall& c, dim3 grid, bool pre, const BwdArgs& a) {
    auto go = [&](auto geom, auto prev) {
        launch(k_raster_bwd2<RGBM, TG, TS, NC, decltype(geom)::value, decltype(prev)::value, IdxT, SP>, grid, BWD2_THREADS, 0,
               c.stream, c.rec, a.textures, a.colors_hi, a.aggrs, a.grad_images, a.grad_faces, a.grad_tex, c.K, c.pb);
    };
    using Y = std::true_type;
    using N = std::false_type;
    const bool geom = a.grad_faces != nullptr;
    if constexpr (SP) {
        if (pre) go(Y{}, Y{}); else go(Y{}, N{});
    } else if constexpr (TG && RGBM == 1) {
        if (pre) { if (geom) go(Y{}, Y{}); else go(N{}, Y{}); }
        else { if (geom) go(Y{}, N{}); else go(N{}, N{}); }
    } else if constexpr (TG) {
        if (geom) go(Y{}, N{}); else go(N{}, N{});
    } else {
        go(Y{}, N{});
    }
}

// The backward of UMR's configuration.  With a pair buffer: the streamed backward over the pairs the forward saved, on the
// forward's tiles (the 4-channel render's are always 16x16), then the recompute backward for the tiles it could not save;
// without one, the recompute backward for every tile.
template <int RGBM, bool TG, int NC, bool SP>
static void launch_pairs_backward(const RasterCall& c, unsigned list_grid, bool pre, const BwdArgs& a) {
    const size_t smem = raster_dyn_smem(c.F);
    if (c.pb.cap == 0) {
        launch(k_raster_bwd_pairs<RGBM, TG, NC, SP>, c.grid16, CTA, smem, c.stream, c.rec, c.box, a.textures, a.colors_hi,
               a.aggrs, a.grad_images, a.grad_faces, a.grad_tex, c.ubox, c.K);
        return;
    }
    with_index(c.wide, [&](auto idx) {
        using IDX = decltype(idx);
        if constexpr (NC == 3) {
            if (forward_impl(c.p->tile_mode) == 4) {
                launch_bwd2<RGBM, TG, NC, SP, 32, IDX>(c, c.grid32, pre, a);
                return;
            }
        }
        launch_bwd2<RGBM, TG, NC, SP, 16, IDX>(c, c.grid16, pre, a);
    });
    launch(k_raster_bwd_pairs_list<RGBM, TG, NC, SP>, list_grid, CTA, smem, c.stream, c.rec, c.box, a.textures, a.colors_hi,
           a.aggrs, a.grad_images, a.grad_faces, a.grad_tex, c.ubox, c.K, c.pb.ctrl + 1, c.pb.ulist, (int)c.grid16.x,
           (int)c.grid16.y);
}

// det: the deterministic mode (every mode check_params accepts): 16x16-tile forward whatever tile_mode says, no pair
// buffer, fixed-point p2f accumulators after the default workspace layout
static int raster_forward(const float* face_vertices, const float* textures, float* images, float* soft_colors,
                          float* aggrs_info, float* p2f_info, const UmrRasterParams* p, void* workspace, void* stream,
                          bool det) {
    int rc = check_params<float>(p);
    if (rc) return rc;
    if (det && raster_side(p) > GATHER_MAX_RASTER) return UMR_ERR_TOO_LARGE;
    if (!face_vertices || !textures || !images || !aggrs_info || !workspace) return UMR_ERR_BAD_ARG;
    if (misaligned(workspace, 256)) return UMR_ERR_BAD_ARG;
    if ((rc = ensure_smem_attrs())) return rc;
    RasterCall c = raster_call(p, workspace, stream, !det && !is_generic(p));
    if (!c.K.aa && soft_colors == nullptr) soft_colors = images;
    c.K.vec_store = (c.K.aa && (c.S % 8) == 0 && (((uintptr_t)images | (uintptr_t)soft_colors | (uintptr_t)aggrs_info) & 15) == 0) ? 1 : 0;
    if ((rc = prep(c, face_vertices, nullptr))) return rc;
    // p2f sums: float accumulators in the workspace, or the deterministic mode's fixed-point words after it
    const size_t n = (size_t)c.B * c.F;
    void* acc = (char*)workspace + (det ? c.L.total : c.L.p2f_off);
    float* pacc = (c.softmax && p2f_info) ? (float*)acc : nullptr;
    if (pacc) {
        cudaError_t e = cudaMemsetAsync(acc, 0, det ? n * P2F_DET_WORDS * sizeof(unsigned long long) : n * 4 * sizeof(float),
                                        c.stream);
        if (e != cudaSuccess) return (int)e;
    }
    const float* bg = p->background_color;
    if (c.gen) {
        record(p->ev_kernel_start, c.stream);
        launch(c.softmax ? (det ? k_raster_fwd<1, true> : k_raster_fwd<1>) : k_raster_fwd<0>, c.grid16, CTA,
               raster_dyn_smem(c.F), c.stream, c.rec, c.box, textures, images, soft_colors, aggrs_info, pacc, c.ubox, c.K,
               p->eps, bg[0], bg[1], bg[2]);
    } else {
        // coarse bins -> tiled forward (saves pair records when a pair buffer is given)
        if ((rc = bin_coarse(c))) return rc;
        record(p->ev_kernel_start, c.stream);
        with_index(c.wide, [&](auto idx) {
            using IDX = decltype(idx);
            if (c.nc4 || det || forward_impl(p->tile_mode) == 3) {
                auto fwd3 = c.nc4 ? (det ? k_raster_fwd3<1, 4, IDX, true> : k_raster_fwd3<1, 4, IDX>)
                            : c.softmax ? (det ? k_raster_fwd3<1, 3, IDX, true> : k_raster_fwd3<1, 3, IDX>)
                                        : k_raster_fwd3<0, 3, IDX>;
                launch(fwd3, c.grid16, CTA, 0, c.stream, c.rec, c.box, (const IDX*)c.clist, c.ccount, textures, images,
                       soft_colors, aggrs_info, pacc, c.ubox, c.K, p->eps, bg[0], bg[1], bg[2], c.pb, c.ncb,
                       c.nc4 ? p->background_extra : 0.f, nullptr);
            } else {
                launch(c.softmax ? k_raster_fwd4<1, IDX> : k_raster_fwd4<0, IDX>, c.grid32, CTA, fwd4_dyn_smem(c.F, sizeof(IDX)),
                       c.stream, c.rec, c.box, (const IDX*)c.clist, c.ccount, textures, images, soft_colors, aggrs_info, pacc,
                       c.ubox, c.K, p->eps, bg[0], bg[1], bg[2], c.pb, c.ncb);
            }
        });
    }
    record(p->ev_kernel_stop, c.stream);
    if (pacc) {
        const unsigned grid = (unsigned)((n + 255) / 256);
        if (det) launch(k_p2f_finalize_det, grid, 256, 0, c.stream, (const unsigned long long*)acc, p2f_info, n);
        else launch(k_p2f_finalize, grid, 256, 0, c.stream, (const float*)acc, p2f_info, n);
    } else if (p2f_info) {  // hard mode never accumulates p2f (kernel.cu:417-431 is softmax-only) -> zeros
        cudaError_t e = cudaMemsetAsync(p2f_info, 0, n * 2 * sizeof(float), c.stream);
        if (e != cudaSuccess) return (int)e;
    }
    return (int)cudaGetLastError();
}

extern "C" int umr_raster_forward(const float* face_vertices, const float* textures, float* images,
                                  float* soft_colors, float* aggrs_info, float* p2f_info,
                                  const UmrRasterParams* p, void* workspace, void* stream_) {
    return raster_forward(face_vertices, textures, images, soft_colors, aggrs_info, p2f_info, p, workspace, stream_, false);
}

extern "C" int umr_raster_forward_deterministic(const float* face_vertices, const float* textures, float* images,
                                                float* soft_colors, float* aggrs_info, float* p2f_info,
                                                const UmrRasterParams* p, void* workspace, void* stream_) {
    return raster_forward(face_vertices, textures, images, soft_colors, aggrs_info, p2f_info, p, workspace, stream_, true);
}

// Visibility only: the hard z-buffer's winner per raster pixel (see k_raster_fwd3<2>).  aggrs_info [B,2,S,S] =
// (depth_min, float(face_index_min)) exactly as umr_raster_forward writes them with func_id_rgb = UMR_RGB_HARD.
extern "C" int umr_raster_visibility(const float* face_vertices, float* aggrs_info, uint8_t* visible_faces,
                                     const UmrRasterParams* p, void* workspace, void* stream_) {
    int rc = check_params<float>(p);
    if (rc) return rc;
    if (!face_vertices || (!aggrs_info && !visible_faces) || !workspace) return UMR_ERR_BAD_ARG;
    if (misaligned(workspace, 256)) return UMR_ERR_BAD_ARG;
    if (is_generic(p)) return UMR_ERR_UNSUPPORTED;  // euclidean distance / prod alpha / surface textures: UMR's configuration
    if ((rc = ensure_smem_attrs())) return rc;
    RasterCall c = raster_call(p, workspace, stream_, false);
    c.K.vec_store = (c.K.aa && (c.S % 8) == 0 && ((uintptr_t)aggrs_info & 15) == 0) ? 1 : 0;
    if (visible_faces) {
        cudaError_t e = cudaMemsetAsync(visible_faces, 0, (size_t)c.B * c.F, c.stream);
        if (e != cudaSuccess) return (int)e;
    }
    if ((rc = prep(c, face_vertices, nullptr)) || (rc = bin_coarse(c))) return rc;
    record(p->ev_kernel_start, c.stream);
    with_index(c.wide, [&](auto idx) {
        using IDX = decltype(idx);
        if (visible_faces && !aggrs_info)  // only the visible-face bytes: face-parallel z-buffer per 64x64 bin
            launch(k_visible_faces<IDX>, dim3(c.ncb, c.ncb, c.B), CTA, 0, c.stream, c.rec, (const IDX*)c.clist, c.ccount,
                   visible_faces, c.K);
        else
            launch(k_raster_fwd3<2, 3, IDX>, c.grid16, CTA, 0, c.stream, c.rec, c.box, (const IDX*)c.clist, c.ccount,
                   /*textures*/ nullptr, /*images*/ nullptr, /*colors_hi*/ nullptr, aggrs_info, /*p2f*/ nullptr, c.ubox, c.K,
                   p->eps, 0.f, 0.f, 0.f, c.pb, c.ncb, 0.f, visible_faces);
    });
    record(p->ev_kernel_stop, c.stream);
    return (int)cudaGetLastError();
}

// The split backward takes both gradients and UMR's configuration with 3 colour channels only (see umr_raster_backward_split).
static bool split_refused(const UmrRasterParams* p, const float* grad_faces, const float* grad_textures) {
    return !grad_faces || !grad_textures || is_generic(p) || p->color_channels == 4;
}

// split: umr_raster_backward_split
static int raster_backward(const float* face_vertices, const float* textures, const float* soft_colors, const float* aggrs_info,
                           const float* grad_images, float* grad_faces, float* grad_textures, const UmrRasterParams* p,
                           void* workspace, void* stream_, bool split) {
    int rc = check_params<float>(p);
    if (rc) return rc;
    if (split && split_refused(p, grad_faces, grad_textures)) return UMR_ERR_BAD_ARG;
    if (!face_vertices || !textures || !soft_colors || !aggrs_info || !grad_images || !workspace) return UMR_ERR_BAD_ARG;
    if (!grad_faces && !grad_textures) return UMR_ERR_BAD_ARG;  // nothing to compute
    if (misaligned(workspace, 256)) return UMR_ERR_BAD_ARG;
    if (p->color_channels == 4 && grad_textures) return UMR_ERR_UNSUPPORTED;  // part maps are constants (loss_utils.py:367-381)
    if (!grad_faces && is_generic(p)) return UMR_ERR_UNSUPPORTED;  // texture-only backward: streaming / pair kernels only
    if ((rc = ensure_smem_attrs())) return rc;
    const RasterCall c = raster_call(p, workspace, stream_, !is_generic(p));
    // The streamed backward re-derives its z-gradient factors from the records whenever it forms the colour terms of the
    // vertex gradients; a texture-only or split backward with a pair buffer needs them only for the recompute fallback, so
    // k_prep returns at once there when no tile is unsaved.
    if ((rc = prep(c, face_vertices, (c.pb.cap > 0 && (!grad_faces || split)) ? c.pb.ctrl + 1 : nullptr)) ||
        (rc = zero_grads(c, grad_faces, grad_textures)))
        return rc;
    unsigned lg = 0;
    if ((rc = list_grid(c, &lg))) return rc;
    // texel-gradient pre-reduction inside the warp (k_raster_bwd2<..., PRE>): pays when many pixels of an 8x4 block land
    // on one texel, i.e. when a face covers many more raster pixels than it has texels.
    const bool pre = (double)c.S * c.S >= (grad_faces ? TEXGRAD_PRE_RATIO_FULL : TEXGRAD_PRE_RATIO_TEXONLY) *
                                              (double)c.F * p->texture_size;
    const BwdArgs a{textures, soft_colors, aggrs_info, grad_images, grad_faces, grad_textures};
    record(p->ev_kernel_start, c.stream);
    if (c.gen)
        launch(c.softmax ? (grad_textures ? k_raster_bwd<1, true> : k_raster_bwd<1, false>)
                         : (grad_textures ? k_raster_bwd<0, true> : k_raster_bwd<0, false>),
               c.grid16, CTA, raster_dyn_smem(c.F), c.stream, c.rec, c.box, textures, soft_colors, aggrs_info, grad_images,
               grad_faces, grad_textures, c.ubox, c.K);
    else if (c.nc4) launch_pairs_backward<1, false, 4, false>(c, lg, pre, a);  // softmax, no texture gradient (above)
    else if (c.softmax && split) launch_pairs_backward<1, true, 3, true>(c, lg, pre, a);
    else if (c.softmax && grad_textures) launch_pairs_backward<1, true, 3, false>(c, lg, pre, a);
    else if (c.softmax) launch_pairs_backward<1, false, 3, false>(c, lg, pre, a);
    // hard colours: the vertex gradients have no colour terms, so the split backward is the full one
    else if (grad_textures) launch_pairs_backward<0, true, 3, false>(c, lg, pre, a);
    else launch_pairs_backward<0, false, 3, false>(c, lg, pre, a);
    record(p->ev_kernel_stop, c.stream);
    return (int)cudaGetLastError();
}

extern "C" int umr_raster_backward(const float* face_vertices, const float* textures,
                                   const float* soft_colors, const float* aggrs_info,
                                   const float* grad_images, float* grad_faces, float* grad_textures,
                                   const UmrRasterParams* p, void* workspace, void* stream_) {
    return raster_backward(face_vertices, textures, soft_colors, aggrs_info, grad_images, grad_faces, grad_textures, p, workspace,
                           stream_, false);
}

extern "C" int umr_raster_backward_split(const float* face_vertices, const float* textures,
                                         const float* soft_colors, const float* aggrs_info,
                                         const float* grad_images, float* grad_faces, float* grad_textures,
                                         const UmrRasterParams* p, void* workspace, void* stream_) {
    return raster_backward(face_vertices, textures, soft_colors, aggrs_info, grad_images, grad_faces, grad_textures, p, workspace,
                           stream_, true);
}

// Deterministic backward: k_prep, then the face-parallel gather k_raster_bwd_det (no pair buffer, no atomics).  Same inputs
// and outputs as umr_raster_backward; grad_faces == NULL (texture-only) is accepted.  split: see raster_backward.
static int raster_backward_det(const float* face_vertices, const float* textures, const float* soft_colors,
                               const float* aggrs_info, const float* grad_images, float* grad_faces, float* grad_textures,
                               const UmrRasterParams* p, void* workspace, void* stream_, bool split) {
    int rc = check_params<float>(p);
    if (rc) return rc;
    if (split && split_refused(p, grad_faces, grad_textures)) return UMR_ERR_BAD_ARG;
    if (raster_side(p) > GATHER_MAX_RASTER) return UMR_ERR_TOO_LARGE;  // as the forward
    if (!face_vertices || !textures || !soft_colors || !aggrs_info || !grad_images || !workspace) return UMR_ERR_BAD_ARG;
    if (!grad_faces && !grad_textures) return UMR_ERR_BAD_ARG;
    if (misaligned(workspace, 256)) return UMR_ERR_BAD_ARG;
    if (p->color_channels == 4 && grad_textures) return UMR_ERR_UNSUPPORTED;  // part maps are constants (loss_utils.py:367-381)
    const RasterCall c = raster_call(p, workspace, stream_, false);
    if ((rc = prep(c, face_vertices, nullptr)) || (rc = zero_grads(c, nullptr, grad_textures))) return rc;
    // RGB x TEXGRAD x GEN with 3 channels; hard colours: the split backward is the full one
    auto k = c.softmax ? (grad_textures ? (c.gen ? k_raster_bwd_det<float, 1, true, 3, true> : k_raster_bwd_det<float, 1, true, 3>)
                                        : (c.gen ? k_raster_bwd_det<float, 1, false, 3, true> : k_raster_bwd_det<float, 1, false, 3>))
                       : (grad_textures ? (c.gen ? k_raster_bwd_det<float, 0, true, 3, true> : k_raster_bwd_det<float, 0, true, 3>)
                                        : (c.gen ? k_raster_bwd_det<float, 0, false, 3, true> : k_raster_bwd_det<float, 0, false, 3>));
    if (c.nc4) k = k_raster_bwd_det<float, 1, false, 4>;
    else if (split && c.softmax) k = k_raster_bwd_det<float, 1, true, 3, false, true>;
    record(p->ev_kernel_start, c.stream);
    launch(k, gather_grid(c.K, c.B), CTA, 0, c.stream, c.rec, textures, soft_colors, aggrs_info, grad_images, grad_faces,
           grad_textures, c.K);
    record(p->ev_kernel_stop, c.stream);
    return (int)cudaGetLastError();
}

extern "C" int umr_raster_backward_deterministic(const float* face_vertices, const float* textures,
                                                 const float* soft_colors, const float* aggrs_info,
                                                 const float* grad_images, float* grad_faces, float* grad_textures,
                                                 const UmrRasterParams* p, void* workspace, void* stream_) {
    return raster_backward_det(face_vertices, textures, soft_colors, aggrs_info, grad_images, grad_faces, grad_textures, p,
                               workspace, stream_, false);
}

extern "C" int umr_raster_backward_split_deterministic(const float* face_vertices, const float* textures,
                                                       const float* soft_colors, const float* aggrs_info,
                                                       const float* grad_images, float* grad_faces, float* grad_textures,
                                                       const UmrRasterParams* p, void* workspace, void* stream_) {
    return raster_backward_det(face_vertices, textures, soft_colors, aggrs_info, grad_images, grad_faces, grad_textures, p,
                               workspace, stream_, true);
}

// =============================================================================================
// Silhouette render (DESIGN.md §12): the alpha plane and its vertex gradient, UMR's configuration only
// =============================================================================================
// Refused before any device work: what check_params refuses, the generic modes and the 4-channel render (UMR_ERR_BAD_ARG),
// and (det) a raster side past the deterministic limit.
static int check_silhouette_params(const UmrRasterParams* p, bool det) {
    int rc = check_params<float>(p);
    if (rc) return rc;
    if (is_generic(p) || p->color_channels == 4) return UMR_ERR_BAD_ARG;
    if (det && raster_side(p) > GATHER_MAX_RASTER) return UMR_ERR_TOO_LARGE;
    return UMR_OK;
}

// det: the deterministic twin -- the 16x16-tile forward whatever tile_mode says and no pair buffer (the silhouette forward
// has no float atomics either way, so its planes are those of the default call)
static int raster_forward_silhouette(const float* face_vertices, float* alpha, float* alpha_hi, const UmrRasterParams* p,
                                     void* workspace, void* stream_, bool det) {
    int rc = check_silhouette_params(p, det);
    if (rc) return rc;
    if (!face_vertices || !alpha || !workspace) return UMR_ERR_BAD_ARG;
    if (misaligned(face_vertices, 4) || misaligned(alpha, 4) || misaligned(alpha_hi, 4) || misaligned(workspace, 256))
        return UMR_ERR_BAD_ARG;
    if ((rc = ensure_smem_attrs())) return rc;
    const RasterCall c = raster_call(p, workspace, stream_, !det);
    if (!c.K.aa && alpha_hi == nullptr) alpha_hi = alpha;  // the raster is the image
    if ((rc = prep(c, face_vertices, nullptr)) || (rc = bin_coarse(c))) return rc;
    record(p->ev_kernel_start, c.stream);
    with_index(c.wide, [&](auto idx) {
        using IDX = decltype(idx);
        if (det || forward_impl(p->tile_mode) == 3)
            launch(k_raster_fwd3<RGB_SIL, 3, IDX>, c.grid16, CTA, 0, c.stream, c.rec, c.box, (const IDX*)c.clist, c.ccount,
                   /*textures*/ nullptr, alpha, alpha_hi, /*aggrs*/ nullptr, /*p2f*/ nullptr, c.ubox, c.K, p->eps, 0.f, 0.f, 0.f,
                   c.pb, c.ncb, 0.f, nullptr);
        else
            launch(k_raster_fwd4<RGB_SIL, IDX>, c.grid32, CTA, fwd4_dyn_smem(c.F, sizeof(IDX)), c.stream, c.rec, c.box,
                   (const IDX*)c.clist, c.ccount, nullptr, alpha, alpha_hi, nullptr, nullptr, c.ubox, c.K, p->eps, 0.f, 0.f,
                   0.f, c.pb, c.ncb);
    });
    record(p->ev_kernel_stop, c.stream);
    return (int)cudaGetLastError();
}

// det: k_prep, then the face-parallel gather (no pair buffer, no atomics); otherwise the streamed backward over the pairs the
// forward saved and the recompute backward for the tiles it could not save (or for every tile without a pair buffer)
static int raster_backward_silhouette(const float* face_vertices, const float* alpha_hi, const float* grad_alpha,
                                      float* grad_faces, const UmrRasterParams* p, void* workspace, void* stream_, bool det) {
    int rc = check_silhouette_params(p, det);
    if (rc) return rc;
    if (!face_vertices || !alpha_hi || !grad_alpha || !grad_faces || !workspace) return UMR_ERR_BAD_ARG;
    if (misaligned(face_vertices, 4) || misaligned(alpha_hi, 4) || misaligned(grad_alpha, 4) || misaligned(grad_faces, 4) ||
        misaligned(workspace, 256))
        return UMR_ERR_BAD_ARG;
    if ((rc = ensure_smem_attrs())) return rc;
    const RasterCall c = raster_call(p, workspace, stream_, !det);
    // the streamed silhouette backward reads no face record: with a pair buffer only the recompute fallback needs them, so
    // k_prep returns at once when no tile is unsaved
    if ((rc = prep(c, face_vertices, c.pb.cap > 0 ? c.pb.ctrl + 1 : nullptr))) return rc;
    unsigned lg = 0;
    if (!det && ((rc = zero_grads(c, grad_faces, nullptr)) || (rc = list_grid(c, &lg)))) return rc;
    record(p->ev_kernel_start, c.stream);
    if (det)
        launch(k_raster_bwd_det<float, RGB_SIL, false>, gather_grid(c.K, c.B), CTA, 0, c.stream, c.rec, nullptr, alpha_hi,
               nullptr, grad_alpha, grad_faces, nullptr, c.K);
    else
        launch_pairs_backward<RGB_SIL, false, 3, false>(c, lg, false, BwdArgs{nullptr, alpha_hi, nullptr, grad_alpha, grad_faces, nullptr});
    record(p->ev_kernel_stop, c.stream);
    return (int)cudaGetLastError();
}

extern "C" int umr_raster_forward_silhouette(const float* face_vertices, float* alpha, float* alpha_hi,
                                             const UmrRasterParams* p, void* workspace, void* stream_) {
    return raster_forward_silhouette(face_vertices, alpha, alpha_hi, p, workspace, stream_, false);
}

extern "C" int umr_raster_forward_silhouette_deterministic(const float* face_vertices, float* alpha, float* alpha_hi,
                                                           const UmrRasterParams* p, void* workspace, void* stream_) {
    return raster_forward_silhouette(face_vertices, alpha, alpha_hi, p, workspace, stream_, true);
}

extern "C" int umr_raster_backward_silhouette(const float* face_vertices, const float* alpha_hi, const float* grad_alpha,
                                              float* grad_faces, const UmrRasterParams* p, void* workspace, void* stream_) {
    return raster_backward_silhouette(face_vertices, alpha_hi, grad_alpha, grad_faces, p, workspace, stream_, false);
}

extern "C" int umr_raster_backward_silhouette_deterministic(const float* face_vertices, const float* alpha_hi,
                                                            const float* grad_alpha, float* grad_faces,
                                                            const UmrRasterParams* p, void* workspace, void* stream_) {
    return raster_backward_silhouette(face_vertices, alpha_hi, grad_alpha, grad_faces, p, workspace, stream_, true);
}
