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
#include "umr_b200.h"

namespace umr {

constexpr int TILE = 16;
constexpr int CTA = TILE * TILE;  // 256 threads, one pixel each
constexpr int CHUNK = 32;         // face records per TMA stage
constexpr int NSTAGE = 2;
constexpr int REC_F = 32;         // floats per record (128 B)

// record layout (float index)
constexpr int R_V = 0;     // 9 : x0 y0 z0 x1 y1 z1 x2 y2 z2
constexpr int R_INV = 9;   // 9 : barycentric inverse, row-major
constexpr int R_SYM = 18;  // 6 : s00 s01 s02 s11 s12 s22   (Gram + 1)
constexpr int R_BOX = 24;  // 4 : xlo xhi ylo yhi (cull box, already expanded by r)
constexpr int R_FLG = 28;  // 1 : bit0..2 obtuse corner, bit3 front-facing
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
    L.box_off = align256(n * REC_F * sizeof(float));
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
    float out[REC_F];
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
        float4* dst = reinterpret_cast<float4*>(rec + (size_t)i * REC_F);
#pragma unroll
        for (int k = 0; k < REC_F / 4; ++k)
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
// shared per-(pixel, face) math
// ---------------------------------------------------------------------------------------------
struct Frag {
    float w0, w1, w2;  // unclipped barycentrics
    float t0, t1, t2;  // closest-point barycentrics minus w
    float sign, dx, dy, dis, D;
};

// kernel.cu:325-326 evaluates (2.*i + 1. - S) / S in double and stores a float.  Numerator and
// denominator are integers < 2^24 (exact in float), and rounding a correctly rounded binary64 quotient
// to binary32 equals the correctly rounded binary32 quotient whenever the wide format carries at least
// 2p+2 = 50 bits (Figueroa's double-rounding theorem; binary64 has 53).  So one IEEE float division is
// bit-identical and ~4x cheaper than the double one.
__device__ __forceinline__ float pixel_coord(int i, int S) {
    return __fdiv_rn((float)(2 * i + 1 - S), (float)S);
}

// euclidean signed distance + sigmoid: kernel.cu:62-152, 380-383.  `rc` points at a staged record.
// Returns false when the pair is culled (outside and farther than the threshold).
__device__ __forceinline__ bool fragment(const float* __restrict__ rc, float xp, float yp, float thr,
                                         float sigma, Frag& fr) {
    const float w0 = rc[R_INV + 0] * xp + rc[R_INV + 1] * yp + rc[R_INV + 2];
    const float w1 = rc[R_INV + 3] * xp + rc[R_INV + 4] * yp + rc[R_INV + 5];
    const float w2 = rc[R_INV + 6] * xp + rc[R_INV + 7] * yp + rc[R_INV + 8];
    fr.w0 = w0; fr.w1 = w1; fr.w2 = w2;
    const float fx0 = rc[0], fy0 = rc[1], fx1 = rc[3], fy1 = rc[4], fx2 = rc[6], fy2 = rc[7];
    const float s00 = rc[R_SYM + 0], s01 = rc[R_SYM + 1], s02 = rc[R_SYM + 2];
    const float s11 = rc[R_SYM + 3], s12 = rc[R_SYM + 4], s22 = rc[R_SYM + 5];
    // inside pixels (kernel.cu:76-110) keep the nearest of the three edges; outside pixels (:111-147) project on the ONE
    // edge selected by the sign pattern of w (with the obtuse-corner correction) and clamp
    float dx, dy, t0, t1, t2;
    if (w0 > 0 && w1 > 0 && w2 > 0 && w0 < 1 && w1 < 1 && w2 < 1) {
        float best = 100000000.f;
        // edge k=0: v0=0,v1=1,v2=2    a = sym[0,:] - sym[1,:]
        {
            const float a0 = s00 - s01, a1 = s01 - s11, a2 = s02 - s12;
            float u0 = (w0 * a0 + w1 * a1 + w2 * a2 - a1) / (a0 - a1);
            float u1 = 1 - u0;
            float u2 = 0;
            u0 -= w0; u1 -= w1; u2 -= w2;
            const float ex = u0 * fx0 + u1 * fx1 + u2 * fx2;
            const float ey = u0 * fy0 + u1 * fy1 + u2 * fy2;
            const float d = ex * ex + ey * ey;
            dx = 0.f; dy = 0.f; t0 = t1 = t2 = 0.f;
            if (d < best) { best = d; dx = ex; dy = ey; t0 = u0; t1 = u1; t2 = u2; }
        }
        // edge k=1: v0=1,v1=2,v2=0    a = sym[1,:] - sym[2,:]
        {
            const float a0 = s01 - s02, a1 = s11 - s12, a2 = s12 - s22;
            float u1 = (w0 * a0 + w1 * a1 + w2 * a2 - a2) / (a1 - a2);
            float u2 = 1 - u1;
            float u0 = 0;
            u0 -= w0; u1 -= w1; u2 -= w2;
            const float ex = u0 * fx0 + u1 * fx1 + u2 * fx2;
            const float ey = u0 * fy0 + u1 * fy1 + u2 * fy2;
            const float d = ex * ex + ey * ey;
            if (d < best) { best = d; dx = ex; dy = ey; t0 = u0; t1 = u1; t2 = u2; }
        }
        // edge k=2: v0=2,v1=0,v2=1    a = sym[2,:] - sym[0,:]
        {
            const float a0 = s02 - s00, a1 = s12 - s01, a2 = s22 - s02;
            float u2 = (w0 * a0 + w1 * a1 + w2 * a2 - a0) / (a2 - a0);
            float u0 = 1 - u2;
            float u1 = 0;
            u0 -= w0; u1 -= w1; u2 -= w2;
            const float ex = u0 * fx0 + u1 * fx1 + u2 * fx2;
            const float ey = u0 * fy0 + u1 * fy1 + u2 * fy2;
            const float d = ex * ex + ey * ey;
            if (d < best) { best = d; dx = ex; dy = ey; t0 = u0; t1 = u1; t2 = u2; }
        }
        fr.sign = 1.f;
    } else {
        const uint32_t flg = __float_as_uint(rc[R_FLG]);
        int v0 = -1;
        if (w1 <= 0 && w2 <= 0) {
            v0 = 0;
            if ((flg & 1u) && (xp - fx0) * (fx2 - fx0) + (yp - fy0) * (fy2 - fy0) > 0) v0 = 2;
        } else if (w2 <= 0 && w0 <= 0) {
            v0 = 1;
            if ((flg & 2u) && (xp - fx1) * (fx0 - fx1) + (yp - fy1) * (fy0 - fy1) > 0) v0 = 0;
        } else if (w0 <= 0 && w1 <= 0) {
            v0 = 2;
            if ((flg & 4u) && (xp - fx2) * (fx1 - fx2) + (yp - fy2) * (fy1 - fy2) > 0) v0 = 1;
        } else if (w0 <= 0) v0 = 1;
        else if (w1 <= 0) v0 = 2;
        else if (w2 <= 0) v0 = 0;
        // all w > 0 but some w >= 1 (rounding): undefined in the reference (kernel.cu:128-139 runs
        // with v0 = -1).  Defined as "corner with the largest barycentric", like oracle B.
        if (v0 < 0) v0 = w0 >= w1 ? (w0 >= w2 ? 0 : 2) : (w1 >= w2 ? 1 : 2);
        float u0, u1, u2;
        if (v0 == 0) {  // v1 = 1, v2 = 2
            const float a0 = s00 - s01, a1 = s01 - s11, a2 = s02 - s12;
            u0 = (w0 * a0 + w1 * a1 + w2 * a2 - a1) / (a0 - a1);
            u1 = 1 - u0;
            u2 = 0;
        } else if (v0 == 1) {  // v1 = 2, v2 = 0
            const float a0 = s01 - s02, a1 = s11 - s12, a2 = s12 - s22;
            u1 = (w0 * a0 + w1 * a1 + w2 * a2 - a2) / (a1 - a2);
            u2 = 1 - u1;
            u0 = 0;
        } else {  // v0 = 2, v1 = 0, v2 = 1
            const float a0 = s02 - s00, a1 = s12 - s01, a2 = s22 - s02;
            u2 = (w0 * a0 + w1 * a1 + w2 * a2 - a0) / (a2 - a0);
            u0 = 1 - u2;
            u1 = 0;
        }
        // min(max(t, 0.), 1.) in double then float == float clamp (values are only selected)
        u0 = fminf(fmaxf(u0, 0.f), 1.f) - w0;
        u1 = fminf(fmaxf(u1, 0.f), 1.f) - w1;
        u2 = fminf(fmaxf(u2, 0.f), 1.f) - w2;
        t0 = u0; t1 = u1; t2 = u2;
        dx = t0 * fx0 + t1 * fx1 + t2 * fx2;
        dy = t0 * fy0 + t1 * fy1 + t2 * fy2;
        fr.sign = -1.f;
    }
    const float dis = dx * dx + dy * dy;
    if (fr.sign < 0 && dis >= thr) return false;
    fr.t0 = t0; fr.t1 = t1; fr.t2 = t2;
    fr.dx = dx; fr.dy = dy; fr.dis = dis;
    // 1. / (1. + exp(-sign * dis / sigma)): float exp, double add + divide, float result (:383)
    const float e = expf(-fr.sign * dis / sigma);
    fr.D = (float)(1. / (1. + (double)e));
    return true;
}

// NaN-aware note: fmaxf/fminf return the non-NaN operand whereas the reference's comparisons
// propagate differently; inputs with NaN coordinates are outside the supported domain.

__device__ __forceinline__ void clip_bary(float& w0, float& w1, float& w2) {  // kernel.cu:54-59
    const float hi = (float)(1 - 1e-5), lo = (float)1e-5;
    w0 = fmaxf(fminf(w0, hi), lo);
    w1 = fmaxf(fminf(w1, hi), lo);
    w2 = fmaxf(fminf(w2, hi), lo);
    const float s = fmaxf(w0 + w1 + w2, lo);
    w0 /= s; w1 /= s; w2 /= s;
}

__device__ __forceinline__ float depth_of(const float* __restrict__ rc, float c0, float c1, float c2) {
    // kernel.cu:403: 1. / (float sum) in double, stored as float == 1.f / sum in float (same theorem:
    // both operands are floats, the binary64 quotient is rounded once more to binary32).
    return __fdiv_rn(1.f, c0 / rc[2] + c1 / rc[5] + c2 / rc[8]);
}

__device__ __forceinline__ int texel_index(float c0, float c1, int R) {  // kernel.cu:180-190
    const int wx = (int)(c0 * R);
    const int wy = (int)(c1 * R);
    if ((c0 + c1) * R - wx - wy <= 1) return wy * R + wx;
    return (R - 1 - wy) * R + (R - 1 - wx);
}

struct Consts {
    float thr, sigma, gamma, near_, far_, inv_unused;
    float r_sigma, r_gamma, r_fn, r_nf;  // 1/sigma, 1/gamma, 1/(far-near), 1/(near-far): streamed backward only
    int F, T2, R, S, IS, aa, double_side;
    int dist, alpha, tex;  // mode ids (read only by the generic-mode kernels)
    int vec_store;         // 1: forward may use the shared-staged 128-bit store epilogue (alignment checked on host)
    size_t tex_bs;         // elements per texture (F*T2*3)
    int tex_div;           // consecutive images sharing one texture (1: per-image, B: one batch-shared texture)
};

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

// Texel-gradient sinks of bwd_pair_acc: the recompute backward adds a pair's texel gradient with REDs; the deterministic
// gather takes it out (address and values) and combines the warp's lanes in a fixed order instead.
struct TexRedSink {
    __device__ __forceinline__ void add3(float* p, float a, float b, float c) const { red_add3_global(p, a, b, c); }
    __device__ __forceinline__ void add(float* p, float v) const { red_add_global(p, v); }
};
// A pair adds to at most 9 consecutive floats (a surface texel's 3 channels, or a vertex texture's 3 corner colours) at
// ascending addresses: *addr = the first, val[k] = the value for *addr + k.
struct TexTakeSink {
    float** addr;
    float* val;
    __device__ __forceinline__ void add3(float* p, float a, float b, float c) const {
        *addr = p; val[0] = a; val[1] = b; val[2] = c;
    }
    __device__ __forceinline__ void add(float* p, float v) const {
        if (*addr == nullptr) *addr = p;
        val[p - *addr] = v;
    }
};

// ---------------------------------------------------------------------------------------------
// Modes UMR does not exercise (SURVEY.md §8f-3): hard / barycentric distance, hard / sum alpha, per-vertex
// textures.  They run through the generic per-pixel kernels k_raster_fwd / k_raster_bwd, which read the mode
// ids from Consts at run time; the UMR configuration (euclidean, prod, surface) has its own kernels.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool fragment_any(const float* __restrict__ rc, float xp, float yp, const Consts& K, Frag& fr) {
    if (K.dist == UMR_DIST_EUCLIDEAN) return fragment(rc, xp, yp, K.thr, K.sigma, fr);
    const float w0 = rc[R_INV + 0] * xp + rc[R_INV + 1] * yp + rc[R_INV + 2];
    const float w1 = rc[R_INV + 3] * xp + rc[R_INV + 4] * yp + rc[R_INV + 5];
    const float w2 = rc[R_INV + 6] * xp + rc[R_INV + 7] * yp + rc[R_INV + 8];
    fr.w0 = w0; fr.w1 = w1; fr.w2 = w2;
    fr.t0 = w0; fr.t1 = w1; fr.t2 = w2;  // kernel.cu:551 (barycentric backward uses the unclipped w)
    fr.sign = 0.f; fr.dx = 0.f; fr.dy = 0.f; fr.dis = 0.f;
    if (K.dist == UMR_DIST_HARD) {  // kernel.cu:370-372
        const bool inside = w0 <= 1 && w0 >= 0 && w1 <= 1 && w1 >= 0 && w2 <= 1 && w2 >= 0;
        fr.D = inside ? 1.f : 0.f;
        return inside;
    }
    // barycentric distance, kernel.cu:156-159, 374-377
    float m = w0 > w1 ? (w1 > w2 ? w2 : w1) : (w0 > w2 ? w2 : w0);
    const float dis = m > 0 ? m * m : -(m * m);
    if (-dis >= K.thr) return false;
    fr.dis = dis;
    fr.D = (float)(1. / (1. + (double)expf(-dis / K.sigma)));
    return true;
}

// colour channel k of face texture `tx` (surface: [T2,3] texels; vertex: [3,3] corner colours), kernel.cu:179-195
__device__ __forceinline__ void sample_texture(const float* __restrict__ tx, float c0, float c1, float c2, const Consts& K,
                                               float& r, float& g, float& b) {
    if (K.tex == UMR_TEX_SURFACE) {
        const float* t = tx + (size_t)texel_index(c0, c1, K.R) * 3;
        r = __ldg(t); g = __ldg(t + 1); b = __ldg(t + 2);
    } else {
        r = c0 * __ldg(tx + 0) + c1 * __ldg(tx + 3) + c2 * __ldg(tx + 6);
        g = c0 * __ldg(tx + 1) + c1 * __ldg(tx + 4) + c2 * __ldg(tx + 7);
        b = c0 * __ldg(tx + 2) + c1 * __ldg(tx + 5) + c2 * __ldg(tx + 8);
    }
}

// texture gradient of one pair: adds wgt * (g0,g1,g2) to the sampled texel (surface) or w_j * wgt * g to the
// three corner colours (vertex), kernel.cu:597-601 / 610-616 with the intended texel semantics (App. B-1)
template <class Sink = TexRedSink>
__device__ __forceinline__ void add_texture_grad(float* __restrict__ gt, float c0, float c1, float c2, const Consts& K,
                                                 float wgt, float g0, float g1, float g2, bool weighted, Sink sink = Sink()) {
    if (K.tex == UMR_TEX_SURFACE) {
        float* t = gt + (size_t)texel_index(c0, c1, K.R) * 3;
        sink.add(t + 0, weighted ? wgt * g0 : g0);
        sink.add(t + 1, weighted ? wgt * g1 : g1);
        sink.add(t + 2, weighted ? wgt * g2 : g2);
    } else {
        const float w[3] = {c0, c1, c2};
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            sink.add(gt + 3 * j + 0, weighted ? wgt * (w[j] * g0) : w[j] * g0);
            sink.add(gt + 3 * j + 1, weighted ? wgt * (w[j] * g1) : w[j] * g1);
            sink.add(gt + 3 * j + 2, weighted ? wgt * (w[j] * g2) : w[j] * g2);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// tile machinery shared by forward and backward
// ---------------------------------------------------------------------------------------------
constexpr int PT = 16;          // pixel-tile side of the pair-parallel backward kernel (32 is the A/B alternative)
constexpr int BOX_PIECE = 2048;  // cull boxes staged per TMA bulk copy (32 KB)
constexpr int NWARP = CTA / 32;

// dynamic shared memory: [ records NSTAGE*CHUNK*128 B | cull boxes min(F,BOX_PIECE)*16 B | list u16[F] ]
__host__ __device__ inline size_t smem_box_off() { return (size_t)NSTAGE * CHUNK * REC_F * 4; }
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
        cp_async16(s_rec + ((size_t)(c % NSTAGE) * CHUNK + j) * REC_F + q * 4, rec_img + (size_t)f * REC_F + q * 4);
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
                                                       const uint32_t* __restrict__ ubox, Consts K, float eps,
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
    const float gstep = 2.f / (float)(S - 1);
    const float gx = (px * 2 < S) ? (-1.f + gstep * px) : (1.f - gstep * (S - 1 - px));
    const float gy = (py * 2 < S) ? (-1.f + gstep * py) : (1.f - gstep * (S - 1 - py));

    for (int wb = 0; wb < F && !outside; wb += FACE_WINDOW) {
    const int n = build_tile_list(box + wb, min(F - wb, FACE_WINDOW), s_ext[0], s_ext[1], s_ext[2], s_ext[3], s_box, s_list,
                                  s_warp_cnt, &s_bar, bar_phase);
    // (build_tile_list ends with __syncthreads: the list is visible)
    any = any || n > 0;
    const float* rec_img = rec_all + ((size_t)b * F + wb) * REC_F;
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
        const float* chunk = s_rec + (size_t)st * CHUNK * REC_F;
        // p2f partial sums of this warp: lane j owns chunk face j (registers, no shared traffic)
        float own_x = 0.f, own_y = 0.f, own_w = 0.f;
        float4 bb = *reinterpret_cast<const float4*>(chunk + R_BOX);
        for (int j = 0; j < cnt; ++j) {
            const float* rc = chunk + j * REC_F;
            // prefetch the next cull box while this face is evaluated
            const float4 bbn = *reinterpret_cast<const float4*>(chunk + (j + 1 < cnt ? j + 1 : j) * REC_F + R_BOX);
            float a_x = 0.f, a_y = 0.f, a_w = 0.f;
            bool contrib = false;
            if (live && !(xp > bb.y || xp < bb.x || yp > bb.w || yp < bb.z)) {
                Frag fr;
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
        float* st = s_rec;  // 6 * 256 + 4 * 64 = 1792 floats <= NSTAGE * CHUNK * REC_F = 2048
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
// One (pixel, face) pair of the generic-mode backward for the deterministic gather (k_raster_bwd_det<..., GEN>): the
// per-pair body of k_raster_bwd (kernel.cu:577-654) statement for statement, with the texture gradient going to `sink`;
// writes the 9 vertex gradients to gv (zeroed by the caller) and sets `contrib` for a pair inside the depth range.
// k_raster_bwd keeps its inline copy: calling this function from it changes that kernel's SASS (its scheduling), and the
// default kernels stay bit-for-bit what they were.  The GPU tests hold both to oracle B.
// face_of() yields the face index (read where k_raster_bwd always read it: only for pairs inside the depth range).
template <int RGB, bool TEXGRAD, class Sink = TexRedSink, class FaceOf>
__device__ __forceinline__ void bwd_pair_generic(const float* __restrict__ rc, float xp, float yp, const Consts& K, FaceOf face_of,
                                                 float g0, float g1, float g2, float g3, float C0, float C1, float C2,
                                                 float C3, float ssum, float smax, const float* __restrict__ tex_img,
                                                 float* __restrict__ gtex_img, float* gv, bool& contrib, Sink sink = Sink()) {
    Frag fr;
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
            const int f = face_of();
            float gz0 = 0.f, gz1 = 0.f, gz2 = 0.f;
            if (RGB == 0) {
                if ((float)f == smax) {  // aggrs[1] = winning face id (:596)
                    if (TEXGRAD)
                        add_texture_grad(gtex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, 1.f, g0, g1, g2, false, sink);
                }
            } else if ((front || K.double_side) && (g0 != 0.f || g1 != 0.f || g2 != 0.f)) {
                const float zn = (K.far_ - zp) / (K.far_ - K.near_);
                const float s = fr.D * expf((zn - smax) / K.gamma) / ssum;  // :608
                if (s != 0.f) {
                    if (TEXGRAD)
                        add_texture_grad(gtex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, s, g0, g1, g2, true, sink);
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

template <int RGB, bool TEXGRAD>
__global__ void __launch_bounds__(CTA, 3) k_raster_bwd(const float* __restrict__ rec_all,
                                                       const float4* __restrict__ box_all,
                                                       const float* __restrict__ textures,
                                                       const float* __restrict__ colors_hi,
                                                       const float* __restrict__ aggrs,
                                                       const float* __restrict__ grad_images,
                                                       float* __restrict__ grad_faces, float* __restrict__ grad_tex,
                                                       const uint32_t* __restrict__ ubox, Consts K) {
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
    const float* rec_img = rec_all + ((size_t)b * F + wb) * REC_F;

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
        const float* chunk = s_rec + (size_t)st * CHUNK * REC_F;
        float own[9];  // vertex-gradient partial sums of this warp: lane j owns chunk face j
#pragma unroll
        for (int k = 0; k < 9; ++k) own[k] = 0.f;
        bool own_any = false;
        float4 bb = *reinterpret_cast<const float4*>(chunk + R_BOX);
        for (int j = 0; j < cnt; ++j) {
            const float* rc = chunk + j * REC_F;
            const float4 bbn = *reinterpret_cast<const float4*>(chunk + (j + 1 < cnt ? j + 1 : j) * REC_F + R_BOX);
            float gv[9];
#pragma unroll
            for (int k = 0; k < 9; ++k) gv[k] = 0.f;
            bool contrib = false;
            if (live && !(xp > bb.y || xp < bb.x || yp > bb.w || yp < bb.z)) {
                Frag fr;
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
                                    add_texture_grad(gtex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, 1.f, g0, g1, g2, false);
                            }
                        } else if ((front || K.double_side) && (g0 != 0.f || g1 != 0.f || g2 != 0.f)) {
                            const float zn = (K.far_ - zp) / (K.far_ - K.near_);
                            const float s = fr.D * expf((zn - smax) / K.gamma) / ssum;  // :608
                            if (s != 0.f) {
                                if (TEXGRAD)
                                    add_texture_grad(gtex_img + (size_t)f * K.T2 * 3, k0, k1, k2, K, s, g0, g1, g2, true);
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
template <int RGB, bool TEXGRAD>
__device__ __forceinline__ bool bwd_pair(const float* __restrict__ rc, float xp, float yp, const Consts& K, float g0,
                                         float g1, float g2, float g3, float C0, float C1, float C2, float C3,
                                         float ssum, float smax, int f, const float* __restrict__ tex_img,
                                         float* __restrict__ gtex_img, float* gv) {
    Frag fr;
    if (!fragment(rc, xp, yp, K.thr, K.sigma, fr)) return false;
    // alpha (prod): kernel.cu:577-585
    // g3 * ((1 - alpha) / max(1 - D, 1e-6)) in double (:584).  Interior pixels have alpha == 1: the quotient is
    // then exactly 0 and the double division would take its (very long) special-operand path, so the zero
    // cases are answered directly: x * 0 == 0 with the same sign rules.
    const float one_m_a = 1 - C3;
    float Cxy = (one_m_a == 0.f || g3 == 0.f)
                    ? g3 * one_m_a
                    : (float)((double)g3 * ((double)one_m_a / fmax((double)(1 - fr.D), 1e-6)));
    float k0 = fr.w0, k1 = fr.w1, k2 = fr.w2;
    clip_bary(k0, k1, k2);
    const float zp = depth_of(rc, k0, k1, k2);
    if (zp < K.near_ || zp > K.far_) return false;  // :592 drops the alpha gradient as well
    const uint32_t flg = __float_as_uint(rc[R_FLG]);
    const bool front = (flg & 8u) != 0;
    float gz0 = 0.f, gz1 = 0.f, gz2 = 0.f;
    if (RGB == 0) {
        if ((float)f == smax) {  // aggrs[1] = winning face id (:596)
            if (TEXGRAD) {
                float* gt = gtex_img + ((size_t)f * K.T2 + texel_index(k0, k1, K.R)) * 3;
                red_add_global(gt + 0, g0);
                red_add_global(gt + 1, g1);
                red_add_global(gt + 2, g2);
            }
        }
    } else if ((front || K.double_side) && (g0 != 0.f || g1 != 0.f || g2 != 0.f)) {
        // (no colour gradient at this pixel, e.g. silhouette-only losses: every term below is exactly 0)
        const float zn = (K.far_ - zp) / (K.far_ - K.near_);
        const float s = fr.D * expf((zn - smax) / K.gamma) / ssum;  // :608
        // s == 0 (softmax weight of an occluded face underflowed): texture gradient, C_rgb and the z
        // gradients are all exactly 0 -- skipping them also avoids ~9 IEEE divisions with zero numerators,
        // each of which would take the division's slow special-operand path.
        if (s != 0.f) {
            const size_t to = ((size_t)f * K.T2 + texel_index(k0, k1, K.R)) * 3;
            if (TEXGRAD) {
                red_add_global(gtex_img + to + 0, s * g0);
                red_add_global(gtex_img + to + 1, s * g1);
                red_add_global(gtex_img + to + 2, s * g2);
            }
            float Crgb = 0.f;
            Crgb += g0 * (__ldg(tex_img + to + 0) - C0);
            Crgb += g1 * (__ldg(tex_img + to + 1) - C1);
            Crgb += g2 * (__ldg(tex_img + to + 2) - C2);
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
    const float q = 2 * fr.sign * Cxy;      // :640
    gv[0] = q * (fr.t0 + fr.w0) * fr.dx;
    gv[1] = q * (fr.t0 + fr.w0) * fr.dy;
    gv[2] = gz0;
    gv[3] = q * (fr.t1 + fr.w1) * fr.dx;
    gv[4] = q * (fr.t1 + fr.w1) * fr.dy;
    gv[5] = gz1;
    gv[6] = q * (fr.t2 + fr.w2) * fr.dx;
    gv[7] = q * (fr.t2 + fr.w2) * fr.dy;
    gv[8] = gz2;
    return true;
}

// Register-lean variant used by the pair-parallel kernel: the 10 per-pixel inputs stay in shared memory
// (sp = &s_pix[0][pix], plane stride PT*PT) and are fetched where they are consumed, and the 9 gradients are
// added straight into the caller's accumulators -- this keeps the kernel at <= 64 registers (4 CTAs/SM).
template <int RGB, bool TEXGRAD, int NC = 3, class Sink = TexRedSink>
__device__ __forceinline__ bool bwd_pair_acc(const float* __restrict__ rc, float xp, float yp, const Consts& K,
                                             const float* __restrict__ sp, int f, const float* __restrict__ tex_img,
                                             float* __restrict__ gtex_img, float* acc, Sink sink = Sink()) {
    Frag fr;
    if (!fragment(rc, xp, yp, K.thr, K.sigma, fr)) return false;
    constexpr int NP = PT * PT, NPL = NC + 1, NV = 2 * NPL + 2;  // planes: g[NC], g_alpha, C[NC], alpha, ssum, smax
    const float g3 = sp[NC * NP];
    const float one_m_a = 1 - sp[(2 * NC + 1) * NP];
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
    } else if (front || K.double_side) {
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
// `bar_phase` carries the mbarrier parity across the tiles a CTA processes (list-driven launch).
template <int RGB, bool TEXGRAD, int NC = 3>
__device__ __forceinline__ void bwd_pairs_tile(const float* __restrict__ rec_all, const float4* __restrict__ box_all,
                                               const float* __restrict__ textures, const float* __restrict__ colors_hi,
                                               const float* __restrict__ aggrs, const float* __restrict__ grad_images,
                                               float* __restrict__ grad_faces, float* __restrict__ grad_tex,
                                               const uint32_t* __restrict__ ubox, const Consts& K, int bx, int by, int b,
                                               uint64_t* s_bar_p, uint32_t& bar_phase) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_rec = reinterpret_cast<float*>(smem_raw);
    float4* s_box = reinterpret_cast<float4*>(smem_raw + smem_box_off());
    uint16_t* s_list = reinterpret_cast<uint16_t*>(smem_raw + smem_list_off(K.F));
    __shared__ int s_warp_cnt[NWARP];
    __shared__ float s_ext[4];
    // PT x PT pixel tile (PT = 32 puts 4x the pairs in a chunk).
    constexpr int NPL = NC + 1, NV = 2 * NPL + 2;
    __shared__ float s_pix[NV][PT * PT];   // g[NC], g_alpha, C[NC], alpha, ssum, smax of the tile's pixels (row-major)
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
    const float* rec_img = rec_all + ((size_t)b * F + wb) * REC_F;

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
        for (int k = 0; k < NV; ++k) v[k] = (k == NV - 2) ? 1.f : 0.f;
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
            v[NV - 2] = __ldg(aggrs + ((size_t)b * 2 + 0) * np + p);
            v[NV - 1] = __ldg(aggrs + ((size_t)b * 2 + 1) * np + p);
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
        const float* chunk = s_rec + (size_t)st * CHUNK * REC_F;
        // ---- rectangles: thread (j = tid & 31, part = tid >> 5) tests 4 columns or 4 rows of face j
        {
            const int j = tid & 31, part = tid >> 5;
            if (j < cnt) {
                const float4 bb = *reinterpret_cast<const float4*>(chunk + j * REC_F + R_BOX);
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
                const float* rc = chunk + j * REC_F;
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
                    if (bwd_pair_acc<RGB, TEXGRAD, NC>(rc, s_xp[col], s_yp[row], K, &s_pix[0][pix], f, tex_img, gtex_img, acc))
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
template <int RGB, bool TEXGRAD, int NC = 3>
__global__ void __launch_bounds__(CTA, 3) k_raster_bwd_pairs(const float* __restrict__ rec_all, const float4* __restrict__ box_all,
                                                             const float* __restrict__ textures, const float* __restrict__ colors_hi,
                                                             const float* __restrict__ aggrs, const float* __restrict__ grad_images,
                                                             float* __restrict__ grad_faces, float* __restrict__ grad_tex,
                                                             const uint32_t* __restrict__ ubox, Consts K) {
    __shared__ uint64_t s_bar;
    if (threadIdx.x == 0) {
        mbar_init(&s_bar, 1);
        fence_mbar_init();
    }
    uint32_t phase = 0;  // (bwd_pairs_tile synchronises the CTA before the barrier is first used)
    bwd_pairs_tile<RGB, TEXGRAD, NC>(rec_all, box_all, textures, colors_hi, aggrs, grad_images, grad_faces, grad_tex, ubox, K,
                                 (int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z, &s_bar, phase);
}

// list-driven: with a pair buffer, only the tiles the forward could NOT save are recomputed.  The forward appended
// their ids to `ulist` (count in *ucount); a small persistent grid walks the list, so a render whose tiles were all
// saved pays one near-empty launch instead of one CTA per tile (35 us at C2 with the full grid).
template <int RGB, bool TEXGRAD, int NC = 3>
__global__ void __launch_bounds__(CTA, 3) k_raster_bwd_pairs_list(const float* __restrict__ rec_all, const float4* __restrict__ box_all,
                                                                  const float* __restrict__ textures, const float* __restrict__ colors_hi,
                                                                  const float* __restrict__ aggrs, const float* __restrict__ grad_images,
                                                                  float* __restrict__ grad_faces, float* __restrict__ grad_tex,
                                                                  const uint32_t* __restrict__ ubox, Consts K,
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
        bwd_pairs_tile<RGB, TEXGRAD, NC>(rec_all, box_all, textures, colors_hi, aggrs, grad_images, grad_faces, grad_tex, ubox, K,
                                     bx, by, b, &s_bar, phase);
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

// Conservative index range [i0, i1] of the pixels whose centre coordinate pixel_coord(i, S) lies in [lo, hi] (monotone in i;
// one index of slack on each side, the exact test runs per pixel).  NaN bounds keep every index, as the tile tests do.
__device__ __forceinline__ void det_span(float lo, float hi, int S, int& i0, int& i1) {
    const double a = ((double)lo * S + (S - 1)) * 0.5, c = ((double)hi * S + (S - 1)) * 0.5;
    i0 = a > 0.0 ? (a < (double)S ? (int)a - 1 : S) : 0;
    i1 = c < (double)(S - 1) ? (c >= 0.0 ? (int)c + 1 : -1) : S - 1;
    i0 = max(i0, 0);
    i1 = min(i1, S - 1);
}

// Face-parallel backward without atomics.  A (pixel, face) pair's gradient depends only on per-pixel constants and the face
// record, so every output gets exactly one writer: one warp owns a (texture group, face) pair and walks the group's images in
// ascending order and, in each, the face's cull box row by row (lanes across a row segment of 32 pixels), evaluating each pair
// with bwd_pair_acc -- the recompute backward's arithmetic.  Vertex gradients: a fixed shuffle tree, one plain store per image.
// Texel gradients: lanes that hit the same texel are summed in ascending lane order, and the lowest of them adds the sum into the
// warp-owned texels of the face (plain load / store; __syncwarp orders the steps).  GEN: the generic modes (distance, alpha
// and texture mode read at run time), evaluated with bwd_pair_generic -- k_raster_bwd's arithmetic; a vertex-texture pair adds
// to the face's 9 corner colours, which the warp sums the same way.
constexpr int DET_WARPS = CTA / 32;
template <int RGB, bool TEXGRAD, int NC = 3, bool GEN = false>
__global__ void __launch_bounds__(CTA) k_raster_bwd_det(const float* __restrict__ rec_all, const float* __restrict__ textures,
                                                        const float* __restrict__ colors_hi, const float* __restrict__ aggrs,
                                                        const float* __restrict__ grad_images, float* __restrict__ grad_faces,
                                                        float* __restrict__ grad_tex, Consts K) {
    constexpr int NPL = NC + 1, NV = 2 * NPL + 2, NP = PT * PT;
    static_assert(NP == CTA, "bwd_pair_acc reads the per-pixel planes with stride PT * PT: one slot per thread");
    __shared__ float s_pix[NV][NP];
    __shared__ __align__(16) float s_rc[DET_WARPS][REC_F];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int f = blockIdx.x * DET_WARPS + warp;
    if (f >= K.F) return;  // warp-uniform; the warps share no memory
    const int grp = blockIdx.y, S = K.S, F = K.F;
    const float* tex_img = textures + (size_t)grp * K.tex_bs;
    float* gtex_img = TEXGRAD ? grad_tex + (size_t)grp * K.tex_bs : nullptr;
    float* sp = &s_pix[0][threadIdx.x];
    const float* rc = s_rc[warp];
    const size_t np = (size_t)S * S;
    for (int i = 0; i < K.tex_div; ++i) {
        const int b = grp * K.tex_div + i;
        __syncwarp();
        s_rc[warp][lane] = __ldg(rec_all + ((size_t)b * F + f) * REC_F + lane);
        __syncwarp();
        const float4 bb = *reinterpret_cast<const float4*>(rc + R_BOX);
        int c0, c1, j0, j1;
        det_span(bb.x, bb.y, S, c0, c1);
        det_span(bb.z, bb.w, S, j0, j1);  // j = S - 1 - row
        float acc[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) acc[k] = 0.f;
        for (int py = S - 1 - j1; py <= S - 1 - j0; ++py) {
            const float yp = pixel_coord(S - 1 - py, S);
            if (yp > bb.w || yp < bb.z) continue;  // uniform
            for (int x0 = c0; x0 <= c1; x0 += 32) {
                const int px = x0 + lane;
                const float xp = pixel_coord(px, S);
                float* taddr = nullptr;
                float tval[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                if (px <= c1 && !(xp > bb.y || xp < bb.x)) {
                    const size_t p = (size_t)py * S + px;
                    if (K.aa) {  // avg_pool2d backward: g / 4
                        const size_t nq = (size_t)K.IS * K.IS;
                        const size_t q = (size_t)(py >> 1) * K.IS + (px >> 1);
#pragma unroll
                        for (int k = 0; k < NPL; ++k) sp[k * NP] = __ldg(grad_images + ((size_t)b * NPL + k) * nq + q) * 0.25f;
                    } else {
#pragma unroll
                        for (int k = 0; k < NPL; ++k) sp[k * NP] = __ldg(grad_images + ((size_t)b * NPL + k) * np + p);
                    }
#pragma unroll
                    for (int k = 0; k < NPL; ++k) sp[(NPL + k) * NP] = __ldg(colors_hi + ((size_t)b * NPL + k) * np + p);
                    sp[(NV - 2) * NP] = __ldg(aggrs + ((size_t)b * 2 + 0) * np + p);
                    sp[(NV - 1) * NP] = __ldg(aggrs + ((size_t)b * 2 + 1) * np + p);
                    if constexpr (GEN) {
                        float gv[9];
#pragma unroll
                        for (int k = 0; k < 9; ++k) gv[k] = 0.f;
                        bool hit = false;
                        bwd_pair_generic<RGB, TEXGRAD, TexTakeSink>(rc, xp, yp, K, [=] { return f; }, sp[0], sp[NP], sp[2 * NP], sp[3 * NP],
                                                                    sp[4 * NP], sp[5 * NP], sp[6 * NP], sp[7 * NP], sp[8 * NP],
                                                                    sp[9 * NP], tex_img, gtex_img, gv, hit, TexTakeSink{&taddr, tval});
                        if (hit) {
#pragma unroll
                            for (int k = 0; k < 9; ++k) acc[k] += gv[k];
                        }
                    } else {
                        bwd_pair_acc<RGB, TEXGRAD, NC, TexTakeSink>(rc, xp, yp, K, sp, f, tex_img, gtex_img, acc,
                                                                     TexTakeSink{&taddr, tval});
                    }
                }
                if (TEXGRAD) {
                    const bool has = taddr != nullptr;
                    uint32_t rem = __ballot_sync(0xffffffffu, has);
                    if (rem) {  // uniform
                        const uint32_t peers = __match_any_sync(0xffffffffu, (unsigned long long)(uintptr_t)taddr);
                        const bool vtx = GEN && K.tex != UMR_TEX_SURFACE;  // 9 corner-colour values instead of 3 texel channels
                        float sum[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                        while (rem) {  // ascending lane order
                            const int o = __ffs(rem) - 1;
                            rem &= rem - 1u;
                            const bool mine = (peers >> o) & 1u;
#pragma unroll
                            for (int k = 0; k < 9; ++k) {
                                if (k < 3 || vtx) {
                                    const float v = __shfl_sync(0xffffffffu, tval[k], o);
                                    if (mine) sum[k] += v;
                                }
                            }
                        }
                        if (has && lane == __ffs(peers) - 1) {
#pragma unroll
                            for (int k = 0; k < 9; ++k)
                                if (k < 3 || vtx) taddr[k] = taddr[k] + sum[k];
                        }
                        __syncwarp();
                    }
                }
            }
        }
#pragma unroll
        for (int k = 0; k < 9; ++k) acc[k] = warp_sum(acc[k]);
        if (grad_faces != nullptr && lane < 9) {
            float v = acc[0];
#pragma unroll
            for (int k = 1; k < 9; ++k) v = (lane == k) ? acc[k] : v;
            grad_faces[((size_t)b * F + f) * 9 + lane] = v;
        }
    }
}

}  // namespace umr

#include "raster_stream.cuh"
#include "raster_fwd3.cuh"
#include "raster_fwd4.cuh"

// =============================================================================================
// C ABI
// =============================================================================================
using namespace umr;

// k_raster_bwd2 instantiation for the call: texture-only (grad_faces == NULL) and warp-level texel pre-reduction variants
// exist for the texture-gradient kernels only
template <int RGBM, bool TG, int TS, typename IdxT>
static void launch_bwd2(dim3 grid, cudaStream_t stream, bool pre, const float* rec, const float* textures, const float* soft_colors,
                        const float* aggrs_info, const float* grad_images, float* grad_faces, float* grad_textures,
                        const Consts& K, const PairBuf& pb) {
#define UMR_BWD2_GO(GEOMV, PREV) \
    k_raster_bwd2<RGBM, TG, TS, 3, GEOMV, PREV, IdxT><<<grid, BWD2_THREADS, 0, stream>>>(rec, textures, soft_colors, aggrs_info, grad_images, \
                                                                                    grad_faces, grad_textures, K, pb)
    if constexpr (TG && RGBM == 1) {
        if (pre) { if (grad_faces) UMR_BWD2_GO(true, true); else UMR_BWD2_GO(false, true); }
        else { if (grad_faces) UMR_BWD2_GO(true, false); else UMR_BWD2_GO(false, false); }
    } else if constexpr (TG) {
        if (grad_faces) UMR_BWD2_GO(true, false); else UMR_BWD2_GO(false, false);
    } else {
        UMR_BWD2_GO(true, false);
    }
#undef UMR_BWD2_GO
}

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
    PairBuf pb;
    pb.ctrl = nullptr; pb.tile_head = nullptr; pb.ulist = nullptr; pb.blk_hdr = nullptr; pb.recs = nullptr; pb.cap = 0;
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
static bool is_generic(const UmrRasterParams* p);
static int check_params(const UmrRasterParams* p) {
    if (!p) return UMR_ERR_BAD_ARG;
    if (p->batch_size <= 0 || p->num_faces <= 0 || p->texture_size <= 0 || p->image_size <= 0)
        return UMR_ERR_BAD_ARG;
    if (p->num_faces > UMR_RASTER_MAX_FACES || p->batch_size > 65535) return UMR_ERR_TOO_LARGE;
    if (p->func_id_dist < 0 || p->func_id_dist > 2 || p->func_id_alpha < 0 || p->func_id_alpha > 2 ||
        p->texture_sample_type < 0 || p->texture_sample_type > 1)
        return UMR_ERR_UNSUPPORTED;
    if (p->texture_sample_type == UMR_TEX_VERTEX && p->texture_size != 3) return UMR_ERR_BAD_ARG;  // [B,F,3,3]
    if (p->shared_textures > 1 && p->batch_size % p->shared_textures != 0) return UMR_ERR_BAD_ARG;
    if (p->func_id_rgb != UMR_RGB_HARD && p->func_id_rgb != UMR_RGB_SOFTMAX) return UMR_ERR_UNSUPPORTED;
    if (p->color_channels != 0 && p->color_channels != 3 && p->color_channels != 4) return UMR_ERR_BAD_ARG;
    // 4 colour channels (the part-map render): UMR's own configuration only
    if (p->color_channels == 4 && (is_generic(p) || p->func_id_rgb != UMR_RGB_SOFTMAX)) return UMR_ERR_UNSUPPORTED;
    return UMR_OK;
}

// the UMR configuration has specialised kernels; every other mode combination takes the generic ones
static bool is_generic(const UmrRasterParams* p) {
    return p->func_id_dist != UMR_DIST_EUCLIDEAN || p->func_id_alpha != UMR_ALPHA_PROD ||
           p->texture_sample_type != UMR_TEX_SURFACE;
}

static Consts make_consts(const UmrRasterParams* p) {
    Consts K;
    K.thr = p->dist_eps * p->sigma_val;  // kernel.cu:333 (float * float)
    K.sigma = p->sigma_val;
    K.gamma = p->gamma_val;
    K.near_ = p->near_plane;
    K.far_ = p->far_plane;
    K.inv_unused = 0.f;
    K.r_sigma = (float)(1.0 / (double)p->sigma_val);
    K.r_gamma = (float)(1.0 / (double)p->gamma_val);
    K.r_fn = (float)(1.0 / ((double)p->far_plane - (double)p->near_plane));
    K.r_nf = (float)(1.0 / ((double)p->near_plane - (double)p->far_plane));
    K.F = p->num_faces;
    K.T2 = p->texture_size;
    K.R = (int)sqrt((double)p->texture_size);  // kernel.cu:685
    K.IS = p->image_size;
    K.aa = p->anti_aliasing ? 1 : 0;
    K.S = p->image_size * (K.aa ? 2 : 1);
    K.double_side = p->double_side ? 1 : 0;
    K.dist = p->func_id_dist;
    K.alpha = p->func_id_alpha;
    K.tex = p->texture_sample_type;
    K.vec_store = 0;
    K.tex_bs = (size_t)p->num_faces * p->texture_size * (p->color_channels == 4 ? 4 : 3);
    K.tex_div = p->shared_textures > 1 ? p->shared_textures : 1;
    return K;
}

// Opt every raster kernel into the full dynamic shared-memory range ONCE per device (not per call:
// the call may be inside a CUDA-graph capture).  A 65536-face window needs 8 KB + 32 KB + 128 KB.
static int ensure_smem_attrs() {
    static bool done[64] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    if (dev < 0 || dev >= 64 || done[dev]) return 0;
    int optin = 0;
    e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (e != cudaSuccess) return (int)e;
    cudaFuncAttributes fa;
#define UMR_SET(K)                                                                                  \
    e = cudaFuncGetAttributes(&fa, K);                                                               \
    if (e != cudaSuccess) return (int)e;                                                             \
    e = cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize,                         \
                             optin - (int)fa.sharedSizeBytes);                                       \
    if (e != cudaSuccess) return (int)e;
    UMR_SET((k_raster_fwd<0>)) UMR_SET((k_raster_fwd<1>)) UMR_SET((k_raster_fwd<1, true>))
    UMR_SET((k_raster_fwd4<0>)) UMR_SET((k_raster_fwd4<1>))
    UMR_SET((k_raster_fwd4<0, uint32_t>)) UMR_SET((k_raster_fwd4<1, uint32_t>))
    UMR_SET((k_raster_bwd<0, false>)) UMR_SET((k_raster_bwd<0, true>))
    UMR_SET((k_raster_bwd<1, false>)) UMR_SET((k_raster_bwd<1, true>))
    UMR_SET((k_raster_bwd_pairs<0, false>)) UMR_SET((k_raster_bwd_pairs<0, true>))
    UMR_SET((k_raster_bwd_pairs<1, false>)) UMR_SET((k_raster_bwd_pairs<1, true>))
    UMR_SET((k_raster_bwd_pairs_list<0, false>)) UMR_SET((k_raster_bwd_pairs_list<0, true>))
    UMR_SET((k_raster_bwd_pairs_list<1, false>)) UMR_SET((k_raster_bwd_pairs_list<1, true>))
#undef UMR_SET
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

// Coarse binning for the UMR-configuration kernels: u16 lists of F entries per bin, or (F > 65535) the wide pool, whose
// cursor is reset first.
static int launch_bin_coarse(const float4* box, const uint32_t* ubox, void* clist, int* ccount, int B, int F, int S,
                             const WorkspaceLayout& L, cudaStream_t stream) {
    const int ncb = (S + CB - 1) / CB;
    const size_t smem = (size_t)(F < BOX_PIECE ? F : BOX_PIECE) * 16;
    if (F <= NARROW_MAX_FACES) {
        k_bin_coarse<uint16_t><<<dim3(ncb, ncb, B), CTA, smem, stream>>>(box, ubox, (uint16_t*)clist, ccount, F, S);
        return 0;
    }
    const size_t nbin = (size_t)B * ncb * ncb;
    cudaError_t e = cudaMemsetAsync(ccount + 2 * nbin, 0, sizeof(unsigned long long), stream);
    if (e != cudaSuccess) return (int)e;
    k_bin_coarse<uint32_t><<<dim3(ncb, ncb, B), CTA, smem, stream>>>(box, ubox, (uint32_t*)clist, ccount, F, S, L.clist_cap);
    return 0;
}

// Deterministic-mode workspace: the default layout, then the fixed-point p2f accumulators (P2F_DET_WORDS int64 per face).
static size_t det_acc_bytes(int B, int F) { return align256((size_t)B * F * P2F_DET_WORDS * sizeof(unsigned long long)); }
// Rasters past the launch limit of the 16x16-tile grid (gridDim.y <= 65535) are refused; the p2f limb bound holds below it.
constexpr int DET_MAX_RASTER = 65535 * TILE;

extern "C" size_t umr_raster_workspace_bytes_deterministic(int32_t B, int32_t F, int32_t image_size, int32_t anti_aliasing) {
    if (B <= 0 || F <= 0 || image_size <= 0) return 0;
    return umr_raster_workspace_bytes(B, F, image_size, anti_aliasing) + det_acc_bytes(B, F);
}

// det: the deterministic mode (UMR's configuration only): 16x16-tile forward whatever tile_mode says, no pair buffer,
// fixed-point p2f accumulators after the default workspace layout
static int raster_forward(const float* face_vertices, const float* textures, float* images, float* soft_colors,
                          float* aggrs_info, float* p2f_info, const UmrRasterParams* p, void* workspace, void* stream_,
                          bool det) {
    int rc = check_params(p);
    if (rc) return rc;
    if (det && (int64_t)p->image_size * (p->anti_aliasing ? 2 : 1) > DET_MAX_RASTER) return UMR_ERR_TOO_LARGE;
    if (!face_vertices || !textures || !images || !aggrs_info || !workspace) return UMR_ERR_BAD_ARG;
    if (((uintptr_t)workspace & 255) != 0) return UMR_ERR_BAD_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    rc = ensure_smem_attrs();
    if (rc) return rc;
    const int B = p->batch_size, F = p->num_faces;
    Consts K = make_consts(p);
    if (!K.aa && soft_colors == nullptr) soft_colors = images;
    K.vec_store = (K.aa && (K.S % 8) == 0 && (((uintptr_t)images | (uintptr_t)soft_colors | (uintptr_t)aggrs_info) & 15) == 0) ? 1 : 0;
    const WorkspaceLayout L = ws_layout(B, F, K.S);
    char* ws = (char*)workspace;
    float* rec = (float*)(ws + L.rec_off);
    float4* box = (float4*)(ws + L.box_off);
    float* p2f_acc = (float*)(ws + L.p2f_off);
    uint32_t* ubox = (uint32_t*)(ws + L.ubox_off);
    int* ccount = (int*)(ws + L.ccount_off);
    void* clist = ws + L.clist_off;
    const bool wide = F > NARROW_MAX_FACES;
    const size_t n = (size_t)B * F;
    const float r = sqrtf(K.thr);  // kernel.cu:355 sqrt(threshold) in float
    {
        cudaError_t e0 = cudaMemsetAsync(ubox, 0, (size_t)B * 4 * sizeof(uint32_t), stream);
        if (e0 != cudaSuccess) return (int)e0;
    }
    k_prep<<<dim3((F + 255) / 256, B), 256, 0, stream>>>(face_vertices, rec, box, ubox, F, r);
    count_launch();
    const bool softmax = p->func_id_rgb == UMR_RGB_SOFTMAX;
    const bool want_p2f = p2f_info != nullptr;
    if (det) p2f_acc = (float*)(ws + L.total);
    if (want_p2f && softmax) {
        cudaError_t e = cudaMemsetAsync(p2f_acc, 0, det ? n * P2F_DET_WORDS * sizeof(unsigned long long) : n * 4 * sizeof(float),
                                        stream);
        if (e != cudaSuccess) return (int)e;
    }
    const dim3 grid((K.S + TILE - 1) / TILE, (K.S + TILE - 1) / TILE, B);
    const size_t smem = raster_dyn_smem(F);
    const bool gen = is_generic(p);
    float* pacc = (softmax && want_p2f) ? p2f_acc : nullptr;
    if (!gen) {
        // round-2 pipeline: coarse bins -> tiled forward (saves pair records when a pair buffer is given)
        const int ncb = (K.S + CB - 1) / CB;
        const PairBuf pb = det ? PairBuf{nullptr, nullptr, nullptr, nullptr, nullptr, 0u} : make_pairbuf(p, K.S);
        if (pb.cap > 0) {
            cudaError_t e = cudaMemsetAsync(pb.ctrl, 0, 16, stream);
            if (e != cudaSuccess) return (int)e;
        }
        count_launch(2);
        rc = launch_bin_coarse(box, ubox, clist, ccount, B, F, K.S, L, stream);
        if (rc) return rc;
        if (p->ev_kernel_start) cudaEventRecord((cudaEvent_t)p->ev_kernel_start, stream);
        const bool nc4 = p->color_channels == 4;
        const int impl = (nc4 || det) ? 3 : forward_impl(p->tile_mode);
#define UMR_FWD_ARGS(IDX) rec, box, (const IDX*)clist, ccount, textures, images, soft_colors, aggrs_info, pacc, ubox, K, p->eps, \
                     p->background_color[0], p->background_color[1], p->background_color[2], pb, ncb
#define UMR_FWD(IDX)                                                                                                        \
        if (det && nc4) {                                                                                                   \
            k_raster_fwd3<1, 4, IDX, true><<<grid, CTA, 0, stream>>>(UMR_FWD_ARGS(IDX), p->background_extra);               \
        } else if (det && softmax) {                                                                                        \
            k_raster_fwd3<1, 3, IDX, true><<<grid, CTA, 0, stream>>>(UMR_FWD_ARGS(IDX));                                    \
        } else if (nc4) {                                                                                                   \
            k_raster_fwd3<1, 4, IDX><<<grid, CTA, 0, stream>>>(UMR_FWD_ARGS(IDX), p->background_extra);                     \
        } else if (impl == 3) {                                                                                             \
            if (softmax) k_raster_fwd3<1, 3, IDX><<<grid, CTA, 0, stream>>>(UMR_FWD_ARGS(IDX));                             \
            else k_raster_fwd3<0, 3, IDX><<<grid, CTA, 0, stream>>>(UMR_FWD_ARGS(IDX));                                     \
        } else {                                                                                                            \
            const dim3 grid32((K.S + T4 - 1) / T4, (K.S + T4 - 1) / T4, B);                                                 \
            const size_t sm4 = fwd4_dyn_smem(F, sizeof(IDX));                                                               \
            if (softmax) k_raster_fwd4<1, IDX><<<grid32, CTA, sm4, stream>>>(UMR_FWD_ARGS(IDX));                            \
            else k_raster_fwd4<0, IDX><<<grid32, CTA, sm4, stream>>>(UMR_FWD_ARGS(IDX));                                    \
        }
        if (wide) { UMR_FWD(uint32_t) } else { UMR_FWD(uint16_t) }
#undef UMR_FWD
#undef UMR_FWD_ARGS
        if (p->ev_kernel_stop) cudaEventRecord((cudaEvent_t)p->ev_kernel_stop, stream);
    } else {
    if (p->ev_kernel_start) cudaEventRecord((cudaEvent_t)p->ev_kernel_start, stream);
    count_launch();
#define UMR_LAUNCH_FWD(RGBM)                                                                                 \
    if (det && RGBM == 1) k_raster_fwd<1, true><<<grid, CTA, smem, stream>>>(rec, box, textures, images, soft_colors,      \
                                                    aggrs_info, pacc, ubox, K, p->eps, p->background_color[0],       \
                                                    p->background_color[1], p->background_color[2]);                 \
    else k_raster_fwd<RGBM><<<grid, CTA, smem, stream>>>(rec, box, textures, images, soft_colors, aggrs_info, pacc, ubox, \
                                                    K, p->eps, p->background_color[0], p->background_color[1],       \
                                                    p->background_color[2])
    if (softmax) UMR_LAUNCH_FWD(1); else UMR_LAUNCH_FWD(0);
#undef UMR_LAUNCH_FWD
    if (p->ev_kernel_stop) cudaEventRecord((cudaEvent_t)p->ev_kernel_stop, stream);
    }
    if (want_p2f) {
        if (softmax) {
            count_launch();
            if (det)
                k_p2f_finalize_det<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((const unsigned long long*)p2f_acc, p2f_info, n);
            else
                k_p2f_finalize<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(p2f_acc, p2f_info, n);
        } else {  // hard mode never accumulates p2f (kernel.cu:417-431 is softmax-only) -> zeros
            cudaError_t e = cudaMemsetAsync(p2f_info, 0, n * 2 * sizeof(float), stream);
            if (e != cudaSuccess) return (int)e;
        }
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
    int rc = check_params(p);
    if (rc) return rc;
    if (!face_vertices || (!aggrs_info && !visible_faces) || !workspace) return UMR_ERR_BAD_ARG;
    if (((uintptr_t)workspace & 255) != 0) return UMR_ERR_BAD_ARG;
    if (is_generic(p)) return UMR_ERR_UNSUPPORTED;  // euclidean distance / prod alpha / surface textures: UMR's configuration
    cudaStream_t stream = (cudaStream_t)stream_;
    rc = ensure_smem_attrs();
    if (rc) return rc;
    const int B = p->batch_size, F = p->num_faces;
    Consts K = make_consts(p);
    K.vec_store = (K.aa && (K.S % 8) == 0 && ((uintptr_t)aggrs_info & 15) == 0) ? 1 : 0;
    const WorkspaceLayout L = ws_layout(B, F, K.S);
    char* ws = (char*)workspace;
    float* rec = (float*)(ws + L.rec_off);
    float4* box = (float4*)(ws + L.box_off);
    uint32_t* ubox = (uint32_t*)(ws + L.ubox_off);
    int* ccount = (int*)(ws + L.ccount_off);
    void* clist = ws + L.clist_off;
    cudaError_t e0 = cudaMemsetAsync(ubox, 0, (size_t)B * 4 * sizeof(uint32_t), stream);
    if (e0 != cudaSuccess) return (int)e0;
    if (visible_faces) {
        e0 = cudaMemsetAsync(visible_faces, 0, (size_t)B * F, stream);
        if (e0 != cudaSuccess) return (int)e0;
    }
    k_prep<<<dim3((F + 255) / 256, B), 256, 0, stream>>>(face_vertices, rec, box, ubox, F, sqrtf(K.thr));
    const int ncb = (K.S + CB - 1) / CB;
    rc = launch_bin_coarse(box, ubox, clist, ccount, B, F, K.S, L, stream);
    if (rc) return rc;
    const dim3 grid((K.S + TILE - 1) / TILE, (K.S + TILE - 1) / TILE, B);
    const PairBuf none{nullptr, nullptr, nullptr, nullptr, nullptr, 0u};
    if (p->ev_kernel_start) cudaEventRecord((cudaEvent_t)p->ev_kernel_start, stream);
#define UMR_VIS(IDX)                                                                                                          \
    if (visible_faces && !aggrs_info)   /* only the visible-face bytes: face-parallel z-buffer per 64x64 bin */              \
        k_visible_faces<IDX><<<dim3(ncb, ncb, B), CTA, 0, stream>>>(rec, (const IDX*)clist, ccount, visible_faces, K);       \
    else                                                                                                                      \
        k_raster_fwd3<2, 3, IDX><<<grid, CTA, 0, stream>>>(rec, box, (const IDX*)clist, ccount, /*textures*/ nullptr,        \
                                                           /*images*/ nullptr, /*colors_hi*/ nullptr, aggrs_info,             \
                                                           /*p2f*/ nullptr, ubox, K, p->eps, 0.f, 0.f, 0.f, none, ncb, 0.f,   \
                                                           visible_faces);
    if (F > NARROW_MAX_FACES) { UMR_VIS(uint32_t) } else { UMR_VIS(uint16_t) }
#undef UMR_VIS
    if (p->ev_kernel_stop) cudaEventRecord((cudaEvent_t)p->ev_kernel_stop, stream);
    count_launch(3);
    return (int)cudaGetLastError();
}

extern "C" int umr_raster_backward(const float* face_vertices, const float* textures,
                                   const float* soft_colors, const float* aggrs_info,
                                   const float* grad_images, float* grad_faces, float* grad_textures,
                                   const UmrRasterParams* p, void* workspace, void* stream_) {
    int rc = check_params(p);
    if (rc) return rc;
    if (!face_vertices || !textures || !soft_colors || !aggrs_info || !grad_images || !workspace) return UMR_ERR_BAD_ARG;
    if (!grad_faces && !grad_textures) return UMR_ERR_BAD_ARG;  // nothing to compute
    if (((uintptr_t)workspace & 255) != 0) return UMR_ERR_BAD_ARG;
    const bool nc4 = p->color_channels == 4;
    if (nc4 && grad_textures) return UMR_ERR_UNSUPPORTED;  // part maps are constants (loss_utils.py:367-381)
    cudaStream_t stream = (cudaStream_t)stream_;
    rc = ensure_smem_attrs();
    if (rc) return rc;
    const int B = p->batch_size, F = p->num_faces;
    const Consts K = make_consts(p);
    const WorkspaceLayout L = ws_layout(B, F, K.S);
    char* ws = (char*)workspace;
    float* rec = (float*)(ws + L.rec_off);
    float4* box = (float4*)(ws + L.box_off);
    uint32_t* ubox = (uint32_t*)(ws + L.ubox_off);
    const size_t n = (size_t)B * F;
    const bool wide = F > NARROW_MAX_FACES;
    const float r = sqrtf(K.thr);
    // the workspace is scratch (another render may have used it since forward): rebuild the records
    cudaError_t e = cudaMemsetAsync(ubox, 0, (size_t)B * 4 * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return (int)e;
    const bool gen = is_generic(p);
    const PairBuf pb = gen ? PairBuf{nullptr, nullptr, nullptr, nullptr, nullptr, 0u} : make_pairbuf(p, K.S);
    // The streamed backward re-derives its z-gradient factors from the records whenever it forms vertex gradients; a
    // texture-only backward with a pair buffer needs them only for the recompute fallback, so k_prep returns at once there
    // when no tile is unsaved.
    k_prep<<<dim3((F + 255) / 256, B), 256, 0, stream>>>(face_vertices, rec, box, ubox, F, r,
                                                         (pb.cap > 0 && !grad_faces) ? pb.ctrl + 1 : nullptr);
    count_launch();
    if (grad_faces) {
        e = cudaMemsetAsync(grad_faces, 0, n * 9 * sizeof(float), stream);
        if (e != cudaSuccess) return (int)e;
    } else if (gen) {
        return UMR_ERR_UNSUPPORTED;  // texture-only backward: streaming / pair kernels only
    }
    if (grad_textures) {
        e = cudaMemsetAsync(grad_textures, 0, (n / (p->shared_textures > 1 ? p->shared_textures : 1)) * p->texture_size * 3 * sizeof(float), stream);
        if (e != cudaSuccess) return (int)e;
    }
    const dim3 grid((K.S + TILE - 1) / TILE, (K.S + TILE - 1) / TILE, B);
    const size_t smem = raster_dyn_smem(F);
    const bool softmax = p->func_id_rgb == UMR_RGB_SOFTMAX;
#define UMR_LAUNCH_BWD(RGBM, TG)                                                                              \
    do {                                                                                                      \
        if (gen)                                                                                              \
            k_raster_bwd<RGBM, TG><<<grid, CTA, smem, stream>>>(rec, box, textures, soft_colors, aggrs_info,    \
                                                                grad_images, grad_faces, grad_textures, ubox, K); \
        else {                                                                                                \
            if (pb.cap > 0) {                                                                                 \
                count_launch();                                                                               \
                if (forward_impl(p->tile_mode) == 4 && wide)                                                  \
                    launch_bwd2<RGBM, TG, 32, uint32_t>(grid32, stream, tex_pre, rec, textures, soft_colors, aggrs_info, \
                                                        grad_images, grad_faces, grad_textures, K, pb);       \
                else if (forward_impl(p->tile_mode) == 4)                                                     \
                    launch_bwd2<RGBM, TG, 32, uint16_t>(grid32, stream, tex_pre, rec, textures, soft_colors, aggrs_info, \
                                                        grad_images, grad_faces, grad_textures, K, pb);       \
                else if (wide)                                                                                \
                    launch_bwd2<RGBM, TG, 16, uint32_t>(grid_pairs, stream, tex_pre, rec, textures, soft_colors, aggrs_info, \
                                                        grad_images, grad_faces, grad_textures, K, pb);       \
                else                                                                                          \
                    launch_bwd2<RGBM, TG, 16, uint16_t>(grid_pairs, stream, tex_pre, rec, textures, soft_colors, aggrs_info, \
                                                        grad_images, grad_faces, grad_textures, K, pb);       \
            }                                                                                                 \
            if (pb.cap > 0)                                                                                   \
                k_raster_bwd_pairs_list<RGBM, TG><<<list_grid, CTA, smem, stream>>>(                          \
                    rec, box, textures, soft_colors, aggrs_info, grad_images, grad_faces, grad_textures, ubox, K, \
                    pb.ctrl + 1, pb.ulist, (int)grid_pairs.x, (int)grid_pairs.y);                             \
            else                                                                                              \
                k_raster_bwd_pairs<RGBM, TG><<<grid_pairs, CTA, smem, stream>>>(rec, box, textures, soft_colors, aggrs_info, \
                                                                      grad_images, grad_faces, grad_textures, ubox, K); \
        }                                                                                                     \
    } while (0)
    const dim3 grid_pairs((K.S + PT - 1) / PT, (K.S + PT - 1) / PT, B);
    const dim3 grid32((K.S + T4 - 1) / T4, (K.S + T4 - 1) / T4, B);
    // texel-gradient pre-reduction inside the warp (k_raster_bwd2<..., PRE>): pays when many pixels of an 8x4 block land
    // on one texel, i.e. when a face covers many more raster pixels than it has texels.
    const bool tex_pre = (double)K.S * K.S >= (grad_faces ? TEXGRAD_PRE_RATIO_FULL : TEXGRAD_PRE_RATIO_TEXONLY) *
                                                  (double)F * p->texture_size;
    const size_t ntiles = (size_t)grid_pairs.x * grid_pairs.y * B;
    int sms = 0;
    rc = sm_count(&sms);
    if (rc) return rc;
    const size_t list_max = (size_t)3 * sms;  // 3 resident CTAs per SM walk the unsaved-tile list
    const unsigned list_grid = (unsigned)(ntiles < list_max ? ntiles : list_max);
    if (p->ev_kernel_start) cudaEventRecord((cudaEvent_t)p->ev_kernel_start, stream);
    count_launch();
    if (nc4) {  // 16x16 tiles, softmax, no texture gradient (check_params / above)
        if (pb.cap > 0) {
            count_launch();
            if (wide)
                k_raster_bwd2<1, false, 16, 4, true, false, uint32_t><<<grid_pairs, BWD2_THREADS, 0, stream>>>(
                    rec, textures, soft_colors, aggrs_info, grad_images, grad_faces, grad_textures, K, pb);
            else
                k_raster_bwd2<1, false, 16, 4><<<grid_pairs, BWD2_THREADS, 0, stream>>>(rec, textures, soft_colors, aggrs_info, grad_images, grad_faces,
                                                                                grad_textures, K, pb);
            k_raster_bwd_pairs_list<1, false, 4><<<list_grid, CTA, smem, stream>>>(rec, box, textures, soft_colors, aggrs_info, grad_images,
                                                                                   grad_faces, grad_textures, ubox, K, pb.ctrl + 1,
                                                                                   pb.ulist, (int)grid_pairs.x, (int)grid_pairs.y);
        } else {
            k_raster_bwd_pairs<1, false, 4><<<grid_pairs, CTA, smem, stream>>>(rec, box, textures, soft_colors, aggrs_info, grad_images,
                                                                               grad_faces, grad_textures, ubox, K);
        }
    } else if (softmax) {
        if (grad_textures) UMR_LAUNCH_BWD(1, true); else UMR_LAUNCH_BWD(1, false);
    } else {
        if (grad_textures) UMR_LAUNCH_BWD(0, true); else UMR_LAUNCH_BWD(0, false);
    }
#undef UMR_LAUNCH_BWD
    if (p->ev_kernel_stop) cudaEventRecord((cudaEvent_t)p->ev_kernel_stop, stream);
    return (int)cudaGetLastError();
}

// Deterministic backward: k_prep, then the face-parallel gather k_raster_bwd_det (no pair buffer, no atomics).  Same inputs
// and outputs as umr_raster_backward; grad_faces == NULL (texture-only) is accepted.
extern "C" int umr_raster_backward_deterministic(const float* face_vertices, const float* textures,
                                                 const float* soft_colors, const float* aggrs_info,
                                                 const float* grad_images, float* grad_faces, float* grad_textures,
                                                 const UmrRasterParams* p, void* workspace, void* stream_) {
    int rc = check_params(p);
    if (rc) return rc;
    if (!face_vertices || !textures || !soft_colors || !aggrs_info || !grad_images || !workspace) return UMR_ERR_BAD_ARG;
    if (!grad_faces && !grad_textures) return UMR_ERR_BAD_ARG;
    if (((uintptr_t)workspace & 255) != 0) return UMR_ERR_BAD_ARG;
    if ((int64_t)p->image_size * (p->anti_aliasing ? 2 : 1) > DET_MAX_RASTER) return UMR_ERR_TOO_LARGE;
    const bool gen = is_generic(p);
    const bool nc4 = p->color_channels == 4;
    if (nc4 && grad_textures) return UMR_ERR_UNSUPPORTED;  // part maps are constants (loss_utils.py:367-381)
    cudaStream_t stream = (cudaStream_t)stream_;
    const int B = p->batch_size, F = p->num_faces;
    const Consts K = make_consts(p);
    const WorkspaceLayout L = ws_layout(B, F, K.S);
    char* ws = (char*)workspace;
    float* rec = (float*)(ws + L.rec_off);
    float4* box = (float4*)(ws + L.box_off);
    uint32_t* ubox = (uint32_t*)(ws + L.ubox_off);
    const size_t n = (size_t)B * F;
    cudaError_t e = cudaMemsetAsync(ubox, 0, (size_t)B * 4 * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return (int)e;
    k_prep<<<dim3((F + 255) / 256, B), 256, 0, stream>>>(face_vertices, rec, box, ubox, F, sqrtf(K.thr));
    if (grad_textures) {
        e = cudaMemsetAsync(grad_textures, 0, (n / K.tex_div) * p->texture_size * 3 * sizeof(float), stream);
        if (e != cudaSuccess) return (int)e;
    }
    const dim3 grid((unsigned)((F + DET_WARPS - 1) / DET_WARPS), (unsigned)(B / K.tex_div));
    const bool softmax = p->func_id_rgb == UMR_RGB_SOFTMAX;
    if (p->ev_kernel_start) cudaEventRecord((cudaEvent_t)p->ev_kernel_start, stream);
#define UMR_BWD_DET(RGBM, TG, NCH)                                                                                        \
    do {                                                                                                                    \
        if (gen) k_raster_bwd_det<RGBM, TG, NCH, true><<<grid, CTA, 0, stream>>>(rec, textures, soft_colors, aggrs_info,     \
                                                                               grad_images, grad_faces, grad_textures, K); \
        else k_raster_bwd_det<RGBM, TG, NCH><<<grid, CTA, 0, stream>>>(rec, textures, soft_colors, aggrs_info, grad_images,  \
                                                                        grad_faces, grad_textures, K);                     \
    } while (0)
    if (nc4) k_raster_bwd_det<1, false, 4><<<grid, CTA, 0, stream>>>(rec, textures, soft_colors, aggrs_info, grad_images,
                                                                      grad_faces, grad_textures, K);
    else if (softmax) { if (grad_textures) UMR_BWD_DET(1, true, 3); else UMR_BWD_DET(1, false, 3); }
    else { if (grad_textures) UMR_BWD_DET(0, true, 3); else UMR_BWD_DET(0, false, 3); }
#undef UMR_BWD_DET
    if (p->ev_kernel_stop) cudaEventRecord((cudaEvent_t)p->ev_kernel_stop, stream);
    count_launch(2);
    return (int)cudaGetLastError();
}
