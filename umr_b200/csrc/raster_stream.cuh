// raster_stream.cuh -- round-2 raster pipeline: coarse binning, the pair buffer in which the forward
// (k_raster_fwd3 / k_raster_fwd4) SAVES one compact record per surviving (pixel, face) pair, and a streaming
// backward that consumes them.
// Included by raster.cu (same translation unit: -fmad=false, same exact-twin arithmetic helpers).
//
// Why: the round-1 backward re-derived fragment() (~13 IEEE divisions + a double sigmoid) for every pair the
// forward had already evaluated, behind 3 CTA barriers per 32-face chunk, with DRAM mostly idle;
// and every tile CTA re-scanned all F cull boxes in both passes.  Now:
//   k_bin_coarse     one CTA per 64x64-pixel bin scans the image's F cull boxes ONCE (TMA-staged, ordered
//                    ballot compaction) -> ascending face list per bin.  Tiles scan their bin's list
//                    (~100-200 entries) instead of F (1280 / 5120).
//   pair records     the forward writes one 32-byte record per surviving pair that passes the depth range
//                    (32-slot blocks, survivors compacted to the block front, block-SoA so a warp writes
//                    two fully coalesced 512-byte lines).  The z-gradient factors w_clip_k / z_k^2 are not
//                    saved: the backward re-derives them bit for bit from the face record and the pixel.
//   k_raster_bwd2    one CTA per tile streams the tile's blocks: no cull boxes, no fragment(), no barrier
//                    after the per-pixel inputs are staged; a warp owns a contiguous block range, so the 9
//                    vertex gradients are accumulated privately and flushed (shuffle reduce + 9 RED) once per
//                    (warp, face run).
// Tiles whose blocks do not fit the caller's pair buffer are marked UNSAVED and take the round-1 recompute
// kernel (k_raster_bwd_pairs) -- results are identical either way (tests/test_raster_stream_gpu.py).
#pragma once

namespace umr {

constexpr int CB = 64;             // coarse bin side in pixels (4 x 4 tiles)
constexpr int LCAP = 512;          // coarse-list window == longest tile-list segment held in shared memory
constexpr uint32_t SEG_NONE = 0xffffffffu;
constexpr int32_t TILE_EMPTY = -1, TILE_UNSAVED = -2;
constexpr int BLK_F4 = 64;         // float4 per block: 2 planes x 32 records

struct PairBuf {
    uint32_t* ctrl;      // [0] block cursor (== blocks wanted, may exceed cap), [1] tiles left unsaved
    int32_t* tile_head;  // [B * tiles]: first segment (block index), TILE_EMPTY or TILE_UNSAVED
    int32_t* ulist;      // [B * tiles]: ids of the unsaved tiles (count = ctrl[1]), walked by the recompute fallback
    uint32_t* blk_hdr;   // [cap]: per block  face | count << hdr_shift (16 narrow, 24 wide) ; per segment  [base] = #blocks, [base+1] = next
    float4* recs;        // [cap][2][32]
    uint32_t cap;        // blocks
};

struct PairBufLayout {
    size_t ctrl_off, head_off, ulist_off, hdr_off, rec_off, total;
};
inline PairBufLayout pair_layout(int B, int S, size_t cap_blocks) {
    PairBufLayout L;
    const size_t nt = (size_t)((S + TILE - 1) / TILE) * ((S + TILE - 1) / TILE) * B;
    L.ctrl_off = 0;
    L.head_off = 256;
    L.ulist_off = L.head_off + align256(nt * sizeof(int32_t));
    L.hdr_off = L.ulist_off + align256(nt * sizeof(int32_t));
    L.rec_off = L.hdr_off + align256(cap_blocks * sizeof(uint32_t));
    L.total = L.rec_off + cap_blocks * (size_t)BLK_F4 * sizeof(float4);
    return L;
}
// largest capacity (blocks) that fits `bytes`
inline size_t pair_capacity(int B, int S, size_t bytes) {
    const PairBufLayout z = pair_layout(B, S, 0);
    if (bytes <= z.total + 512) return 0;
    size_t cap = (bytes - z.total - 512) / ((size_t)BLK_F4 * sizeof(float4) + sizeof(uint32_t));
    while (cap > 0 && pair_layout(B, S, cap).total > bytes) --cap;
    return cap;
}

// ---------------------------------------------------------------------------------------------
// coarse binning: grid (ncb, ncb, B).
//   narrow (u16): clist[(b, cy, cx)][F], ccount[(b, cy, cx)] = list length
//   wide (u32):   ccount[(b, cy, cx)] = {length, offset of the list in the clist pool}; each bin counts its faces, reserves
//                 that many pool entries with one atomic on the pool cursor (ccount's tail) and fills them.  A bin that
//                 does not fit gets offset BIN_ALL_FACES: its consumers walk all F faces, which their own cull tests
//                 reduce to the same ascending list.
// ---------------------------------------------------------------------------------------------
template <typename IdxT>
struct CoarseBin {
    int n;           // entries
    const IdxT* cl;  // nullptr (wide only): entry i is face i
};
template <typename IdxT>
__device__ __forceinline__ CoarseBin<IdxT> coarse_bin(const IdxT* clist, const int* ccount, size_t cidx, int F) {
    if constexpr (sizeof(IdxT) == 2) {
        return {__ldg(ccount + cidx), clist + cidx * F};
    } else {
        const uint2 c = __ldg(reinterpret_cast<const uint2*>(ccount) + cidx);
        if (c.y == BIN_ALL_FACES) return {F, nullptr};
        return {(int)c.x, clist + c.y};
    }
}
template <typename IdxT>
__device__ __forceinline__ int bin_face(const CoarseBin<IdxT>& cb, int i) {
    if constexpr (sizeof(IdxT) == 2) return __ldg(cb.cl + i);
    else return cb.cl ? (int)__ldg(cb.cl + i) : i;
}

template <typename IdxT>
__global__ void __launch_bounds__(CTA) k_bin_coarse(const float4* __restrict__ box_all, const uint32_t* __restrict__ ubox,
                                                    IdxT* __restrict__ clist, int* __restrict__ ccount, int F, int S,
                                                    size_t pool_cap = 0) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float4* s_box = reinterpret_cast<float4*>(smem_raw);
    __shared__ uint64_t s_bar;
    __shared__ int s_warp_cnt[NWARP];
    __shared__ float s_ext[4];
    const int b = blockIdx.z;
    if (threadIdx.x == 0) {
        mbar_init(&s_bar, 1);
        fence_mbar_init();
    }
    tile_extents(S, s_ext, CB);
    __syncthreads();
    const size_t cidx = ((size_t)b * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    int n = 0;
    uint32_t bar_phase = 0;
    const float4* box = box_all + (size_t)b * F;
    if constexpr (sizeof(IdxT) == 2) {
        if (!tile_outside_union(ubox, b, s_ext))
            n = build_tile_list(box, F, s_ext[0], s_ext[1], s_ext[2], s_ext[3], s_box, clist + cidx * F, s_warp_cnt, &s_bar,
                                bar_phase);
        if (threadIdx.x == 0) ccount[cidx] = n;
    } else {
        __shared__ uint32_t s_off;
        if (!tile_outside_union(ubox, b, s_ext))
            n = build_tile_list<IdxT>(box, F, s_ext[0], s_ext[1], s_ext[2], s_ext[3], s_box, nullptr, s_warp_cnt, &s_bar,
                                      bar_phase);
        if (threadIdx.x == 0) {
            const size_t nbin = (size_t)gridDim.x * gridDim.y * gridDim.z;
            unsigned long long* cursor = reinterpret_cast<unsigned long long*>(ccount + 2 * nbin);
            uint32_t off = 0;
            if (n > 0) {
                const unsigned long long base = atomicAdd(cursor, (unsigned long long)n);
                off = base + (unsigned long long)n <= (unsigned long long)pool_cap ? (uint32_t)base : BIN_ALL_FACES;
            }
            s_off = off;
            reinterpret_cast<uint2*>(ccount)[cidx] = make_uint2((uint32_t)n, off);
        }
        __syncthreads();
        if (n > 0 && s_off != BIN_ALL_FACES)  // uniform: the second scan writes the list into the reserved entries
            build_tile_list<IdxT>(box, F, s_ext[0], s_ext[1], s_ext[2], s_ext[3], s_box, clist + s_off, s_warp_cnt, &s_bar,
                                  bar_phase);
    }
}

// ---------------------------------------------------------------------------------------------
// visible faces: which faces win at least one pixel of the hard z-buffer (kernel.cu:404-415) -- the [B,F] bytes TexCycle
// derives from the hard render's face-index plane (loss_utils.py:161-166).  FACE-parallel: one CTA per 64x64 bin keeps a
// z-buffer of packed (depth bits << 32 | face) keys in shared memory; each warp takes faces of the bin's list and tests only
// the pixels of the face's bounding box (+2 px; the whole cull box for thin faces, R_FLG bit 4), atomicMin keeps the
// nearest (lowest face index on ties, like the ascending strict-'<' walk).  No plane is written.  Work ~ sum of bounding
// boxes instead of pixels x candidate faces of k_raster_fwd3<2>.
// ---------------------------------------------------------------------------------------------
template <typename IdxT>
__global__ void __launch_bounds__(CTA) k_visible_faces(const float* __restrict__ rec_all, const IdxT* __restrict__ clist,
                                                       const int* __restrict__ ccount, uint8_t* __restrict__ vis, Consts K) {
    __shared__ unsigned long long s_z[CB * CB];   // 32 KB
    __shared__ float s_xp[CB], s_yp[CB];
    __shared__ int s_bg, s_next;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z, S = K.S, F = K.F;
    const int x0 = blockIdx.x * CB, y0 = blockIdx.y * CB;
    const int ncol = min(CB, S - x0), nrow = min(CB, S - y0);
    const size_t cidx = ((size_t)b * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    const CoarseBin<IdxT> cb = coarse_bin(clist, ccount, cidx, F);
    const int nc = cb.n;
    uint8_t* vb = vis + (size_t)b * F;
    if (nc == 0) {  // all background: face id -1, which the reference's indexing turns into face F-1 (see k_visible)
        if (tid == 0 && *reinterpret_cast<volatile uint8_t*>(vb + F - 1) == 0) vb[F - 1] = 1;
        return;
    }
    for (int i = tid; i < CB * CB; i += CTA) s_z[i] = ~0ull;
    if (tid < CB) s_xp[tid] = pixel_coord(x0 + tid, S);
    else if (tid < 2 * CB) s_yp[tid - CB] = pixel_coord(S - 1 - (y0 + tid - CB), S);
    if (tid == 0) { s_bg = 0; s_next = NWARP; }
    __syncthreads();
    const float* rec_img = rec_all + (size_t)b * F * REC_F;
    auto scan_face = [&](int i) {
        const int f = bin_face(cb, i);
        const float* rc = rec_img + (size_t)f * REC_F;
        if (lane == 0 && i + NWARP < nc)   // the warp's next face: pull its 128-byte record into L1 while this one is scanned
            asm volatile("prefetch.global.L1 [%0];" ::"l"(rec_img + (size_t)bin_face(cb, i + NWARP) * REC_F));
        const uint32_t flg = __float_as_uint(__ldg(rc + R_FLG));
        if (!(K.double_side || (flg & 8u))) return;   // back face of a single-sided render never wins (warp-uniform)
        // pixel rectangle to test: bounding box of the vertices widened by 2 pixels (an inside pixel lies in the box; the
        // margin covers the rounding of the index conversion), or the whole cull box for a thin face
        float xlo, xhi, ylo, yhi;
        if (flg & 16u) {
            xlo = __ldg(rc + R_BOX); xhi = __ldg(rc + R_BOX + 1); ylo = __ldg(rc + R_BOX + 2); yhi = __ldg(rc + R_BOX + 3);
        } else {
            const float ax = __ldg(rc + 0), ay = __ldg(rc + 1), bx = __ldg(rc + 3), by = __ldg(rc + 4), cx = __ldg(rc + 6), cy = __ldg(rc + 7);
            xlo = fminf(fminf(ax, bx), cx); xhi = fmaxf(fmaxf(ax, bx), cx);
            ylo = fminf(fminf(ay, by), cy); yhi = fmaxf(fmaxf(ay, by), cy);
        }
        // pixel_coord(i) = (2 i + 1 - S) / S  <=>  i = (x S + S - 1) / 2;  rows run top-down: y index j = S - 1 - row
        int c0 = (int)floorf((xlo * (float)S + (float)(S - 1)) * 0.5f) - 2 - x0;
        int c1 = (int)ceilf((xhi * (float)S + (float)(S - 1)) * 0.5f) + 2 - x0;
        const int j0 = (int)floorf((ylo * (float)S + (float)(S - 1)) * 0.5f) - 2;
        const int j1 = (int)ceilf((yhi * (float)S + (float)(S - 1)) * 0.5f) + 2;
        int r0 = (S - 1 - j1) - y0, r1 = (S - 1 - j0) - y0;
        if (!(xlo == xlo && xhi == xhi && ylo == ylo && yhi == yhi)) { c0 = 0; c1 = CB; r0 = 0; r1 = CB; }  // NaN face: whole bin
        c0 = max(c0, 0); c1 = min(c1, ncol - 1); r0 = max(r0, 0); r1 = min(r1, nrow - 1);
        const int w = c1 - c0 + 1, h = r1 - r0 + 1;
        if (w <= 0 || h <= 0) return;   // warp-uniform
        const float i00 = __ldg(rc + R_INV + 0), i01 = __ldg(rc + R_INV + 1), i02 = __ldg(rc + R_INV + 2);
        const float i10 = __ldg(rc + R_INV + 3), i11 = __ldg(rc + R_INV + 4), i12 = __ldg(rc + R_INV + 5);
        const float i20 = __ldg(rc + R_INV + 6), i21 = __ldg(rc + R_INV + 7), i22 = __ldg(rc + R_INV + 8);
        const float4 bb = __ldg(reinterpret_cast<const float4*>(rc + R_BOX));
        const int n = w * h;
        for (int p = lane; p < n; p += 32) {
            const int lr = p / w, col = c0 + (p - lr * w), row = r0 + lr;
            const float xp = s_xp[col], yp = s_yp[row];
            if (xp > bb.y || xp < bb.x || yp > bb.w || yp < bb.z) continue;   // the cull test of the full kernel (kernel.cu:32-38)
            const float w0 = i00 * xp + i01 * yp + i02;
            const float w1 = i10 * xp + i11 * yp + i12;
            const float w2 = i20 * xp + i21 * yp + i22;
            if (!(w0 <= 1 && w0 >= 0 && w1 <= 1 && w1 >= 0 && w2 <= 1 && w2 >= 0)) continue;   // kernel.cu:404
            bool pass = w0 > 0 && w1 > 0 && w2 > 0 && w0 < 1 && w1 < 1 && w2 < 1;
            if (!pass) {  // a barycentric exactly 0 or 1: the reference's outside branch decides (kernel.cu:380-383)
                Frag fr;
                pass = fragment(rc, xp, yp, K.thr, K.sigma, fr);
            }
            if (!pass) continue;
            float k0 = w0, k1 = w1, k2 = w2;
            clip_bary(k0, k1, k2);
            const float zp = depth_of(rc, k0, k1, k2);
            if (zp < K.near_ || zp > K.far_ || !(zp < 10000000.f)) continue;   // depth range (:399), initial depth_min (:341)
            // zp > 0 here (near_ >= 0 is assumed by the packed ordering; negative depths are ordered by the sign fix below)
            uint32_t zb = __float_as_uint(zp);
            zb = (zb & 0x80000000u) ? ~zb : (zb | 0x80000000u);   // total order of floats as unsigned integers
            atomicMin(&s_z[row * CB + col], ((unsigned long long)zb << 32) | (unsigned long long)(uint32_t)f);
        }
    };
    // faces are handed out dynamically (shared counter): their bounding boxes differ by an order of magnitude and a static
    // round-robin leaves warps waiting at the end-of-bin barrier (same-box A/B: 1.18 -> 0.97 ms at 32 x 2048^2)
    for (int i = warp; i < nc;) {
        scan_face(i);
        int nx = 0;
        if (lane == 0) nx = atomicAdd(&s_next, 1);
        i = __shfl_sync(0xffffffffu, nx, 0);
    }
    __syncthreads();
    bool bg = false;
    for (int i = tid; i < CB * CB; i += CTA) {
        const int row = i / CB, col = i - row * CB;
        if (row >= nrow || col >= ncol) continue;
        const unsigned long long key = s_z[i];
        if (key == ~0ull) { bg = true; continue; }
        uint8_t* m = vb + (uint32_t)(key & 0xffffffffull);
        if (*reinterpret_cast<volatile uint8_t*>(m) == 0) *m = 1;
    }
    if (bg) s_bg = 1;   // benign race: every writer stores 1
    __syncthreads();
    if (tid == 0 && s_bg && *reinterpret_cast<volatile uint8_t*>(vb + F - 1) == 0) vb[F - 1] = 1;
}

// ---------------------------------------------------------------------------------------------
// backward: stream the saved pair records of the tile
// ---------------------------------------------------------------------------------------------
// NC consecutive texel-gradient floats: RGB goes out as one 2-float vector RED + one scalar (common.cuh)
template <int NC>
__device__ __forceinline__ void red_add_texel(float* gt, const float* v) {
    if (NC == 3) {
        red_add3_global(gt, v[0], v[1], v[2]);
    } else {
#pragma unroll
        for (int c = 0; c < NC; ++c) red_add_global(gt + c, v[c]);
    }
}

constexpr int BWD2_CTAS = 5;  // 5 CTAs x 256 threads (48 registers)
constexpr int BWD2_THREADS = 256, BWD2_WARPS = BWD2_THREADS / 32;  // threads of one k_raster_bwd2 CTA (one tile)
// TS: side of the forward's tile (16: k_raster_fwd3, 32: k_raster_fwd4); one CTA streams one tile
// GEOM = false: the caller wants no gradient for the vertices (UMR's texture branch renders DETACHED geometry,
// experiments/train_s2.py:248) -- only the texel gradients are formed, the compiler drops the rest of the arithmetic.
// PRE = true: the texel gradients of a step are combined inside the warp before they go to global memory -- lanes that hit
// the same texel of the step's face (found with match.any) are summed by the lowest of them, which issues the only REDs.
// Pays only when a face covers hundreds of raster pixels per texel (raster.cu: TEXGRAD_PRE_RATIO_*); at UMR's shapes the
// plain vector REDs are faster.
// rec_all: the face records of k_prep (GEOM only): the z-gradient factors w_clip_k / z_k^2 are re-derived from them
// IdxT: face-index width of the block headers (hdr_shift)
template <int RGB, bool TEXGRAD, int TS, int NC = 3, bool GEOM = true, bool PRE = false, typename IdxT = uint16_t>  // NC colour channels; pixel planes: g[NC], g_alpha, C[NC], alpha, ssum, smax
__global__ void __launch_bounds__(BWD2_THREADS, BWD2_CTAS) k_raster_bwd2(const float* __restrict__ rec_all, const float* __restrict__ textures,
                                                        const float* __restrict__ colors_hi,
                                                        const float* __restrict__ aggrs, const float* __restrict__ grad_images,
                                                        float* __restrict__ grad_faces, float* __restrict__ grad_tex, Consts K,
                                                        PairBuf pb) {
    constexpr int NPL = NC + 1, NV = 2 * NPL + 2;
    __shared__ float s_pix[NV][TS * TS];  // g[NC], g_alpha, C[NC], alpha, ssum, smax (row-major tile pixels)
    __shared__ float s_xp[TS], s_yp[TS];  // pixel centres, built as the forward builds its tables (same bits)
    constexpr int NP = TS * TS;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z;
    const int S = K.S, F = K.F;
    const size_t tile_id = ((size_t)b * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    const int32_t head = __ldg(pb.tile_head + tile_id);
    if (head < 0) return;  // empty, or unsaved (k_raster_bwd_pairs handles it)
    const int x0 = blockIdx.x * TS, y0 = blockIdx.y * TS;
    if (GEOM) {
        if (tid < TS) s_xp[tid] = pixel_coord(x0 + tid, S);
        else if (tid < 2 * TS) s_yp[tid - TS] = pixel_coord(S - 1 - (y0 + tid - TS), S);
    }
    for (int pi = tid; pi < NP; pi += BWD2_THREADS) {
        const int px = x0 + (pi % TS), py = y0 + (pi / TS);
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
    __syncthreads();
    const float* tex_img = textures + (size_t)(b / K.tex_div) * K.tex_bs;
    float* gtex_img = TEXGRAD ? grad_tex + (size_t)(b / K.tex_div) * K.tex_bs : nullptr;
    float* gf_img = grad_faces + (size_t)b * F * 9;
    const float* rec_img = GEOM ? rec_all + (size_t)b * F * REC_F : nullptr;
    // the 128-byte face record of a step is pulled into L1 one step ahead: lanes 1-3 take the 32-byte sectors that hold
    // R_INV and R_IZ2
    auto prefetch_face = [&](int f) {
        if (lane >= 1 && lane < 4) asm volatile("prefetch.global.L1 [%0];" ::"l"(rec_img + (size_t)f * REC_F + 8 * lane));
    };

    float acc[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) acc[k] = 0.f;
    int cur_f = -1;
    auto flush = [&]() {
        if (GEOM && cur_f >= 0) {
#pragma unroll
            for (int k = 0; k < 9; ++k) acc[k] = warp_sum(acc[k]);
            if (lane < 9) {
                float v = acc[0];
#pragma unroll
                for (int k = 1; k < 9; ++k) v = (lane == k) ? acc[k] : v;
                if (v != 0.f) red_add_global(gf_img + (size_t)cur_f * 9 + lane, v);
            }
#pragma unroll
            for (int k = 0; k < 9; ++k) acc[k] = 0.f;
        }
    };

    uint32_t seg = (uint32_t)head;
    while (seg != SEG_NONE) {
        const uint32_t NB = __ldg(pb.blk_hdr + seg), next = __ldg(pb.blk_hdr + seg + 1);
        const uint32_t per = (NB + BWD2_WARPS - 1) / BWD2_WARPS;
        const uint32_t kbeg = min(NB, warp * per), kend = min(NB, kbeg + per);
        const uint32_t* hdrs = pb.blk_hdr + seg + 2;
        // The warp streams the records of its block range 32 at a time: blocks are only partly filled (survivors
        // of 32 candidates), so each step packs the unread records of up to 4 consecutive same-face blocks onto the
        // lanes -- (k, o) = current block and records of it already consumed.
        // block headers of the warp's range: ONE coalesced load per 32 blocks, kept in registers and read with shuffles
        // (a header load inside the loop would put a second global-memory latency in front of every record load)
        uint32_t k = kbeg, kwin = kbeg;
        uint32_t hw = (kbeg + lane < kend) ? __ldg(hdrs + kbeg + lane) : 0u;
        int o = 0;
        // plan(): the next step of the stream -- its face, whether this lane carries a record, and where the record is --
        // and advance (k, o).  Planning runs one step AHEAD of the arithmetic so that the step's two 16-byte lines per lane
        // can be prefetched into L1 while the previous step is being processed (the kernel is bound by the latency of
        // these loads).
        auto plan = [&](int& f_out, bool& act_out, const float4*& src_out) -> bool {
            while (k < kend) {
                if (k >= kwin + 32u) {  // warp-uniform
                    kwin = k;
                    hw = (k + lane < kend) ? __ldg(hdrs + k + lane) : 0u;
                }
                const uint32_t wend = min(kend, kwin + 32u);  // chains stop at the header window
                const int rel = (int)(k - kwin);
                const uint32_t h0 = __shfl_sync(0xffffffffu, hw, rel), h1 = __shfl_sync(0xffffffffu, hw, (rel + 1) & 31);
                const uint32_t h2 = __shfl_sync(0xffffffffu, hw, (rel + 2) & 31), h3 = __shfl_sync(0xffffffffu, hw, (rel + 3) & 31);
                constexpr int HS = hdr_shift<IdxT>();
                constexpr uint32_t HM = (1u << HS) - 1u;
                const int a0 = (int)(h0 >> HS) - o;
                if (a0 <= 0) { ++k; o = 0; continue; }  // block exhausted / empty (warp-uniform)
                const int f = (int)(h0 & HM);
                // records available in the following blocks while they belong to the same face (an empty block is transparent)
                int a1 = 0, a2 = 0, a3 = 0, nchain = 1;
                if (k + 1 < wend && ((h1 >> HS) == 0 || (int)(h1 & HM) == f)) {
                    a1 = (int)(h1 >> HS); nchain = 2;
                    if (k + 2 < wend && ((h2 >> HS) == 0 || (int)(h2 & HM) == f)) {
                        a2 = (int)(h2 >> HS); nchain = 3;
                        if (k + 3 < wend && ((h3 >> HS) == 0 || (int)(h3 & HM) == f)) { a3 = (int)(h3 >> HS); nchain = 4; }
                    }
                }
                const int p1 = a0, p2 = a0 + a1, p3 = p2 + a2, p4 = p3 + a3;
                int bi, pos;
                if (lane < p1) { bi = 0; pos = lane + o; }
                else if (lane < p2) { bi = 1; pos = lane - p1; }
                else if (lane < p3) { bi = 2; pos = lane - p2; }
                else { bi = 3; pos = lane - p3; }
                f_out = f;
                act_out = lane < p4;
                src_out = pb.recs + (size_t)(seg + 2 + k + bi) * BLK_F4 + pos;
                // advance the stream by min(32, p4) records: blocks consumed completely, then a partial one
                int left = min(32, p4), i = 0;
                const int av[4] = {a0, a1, a2, a3};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    if (i == q && q < nchain && left >= av[q]) { left -= av[q]; ++i; }
                }
                k += (uint32_t)i;
                o = (i == 0) ? o + left : ((i < nchain) ? left : 0);
                return true;
            }
            return false;
        };
        // The records of step i + 1 are prefetched into L1 while step i is processed, so the loads' latency is covered by a
        // whole step of arithmetic.
        auto prefetch2 = [&](bool act, const float4* p) {
            if (act) {
                asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
                asm volatile("prefetch.global.L1 [%0];" ::"l"(p + 32));
            }
        };
        int f_c = 0, f_n = 0;
        bool act_c = false, act_n = false;
        const float4 *src_c = nullptr, *src_n = nullptr;
        bool have = plan(f_c, act_c, src_c);
        if (have) prefetch2(act_c, src_c);
        if (GEOM && have) prefetch_face(f_c);
        while (have) {
            const bool have_n = plan(f_n, act_n, src_n);
            if (have_n) prefetch2(act_n, src_n);
            const int f = f_c;  // (warp-uniform, like f_n and have_n)
            if (f != cur_f) { flush(); cur_f = f; }
            if (GEOM && have_n && f_n != f) prefetch_face(f_n);
            int pre_tix = -1;   // PRE: this lane's texel of face f and its NC gradient terms (set below when it contributes)
            float pre_v[NC];
#pragma unroll
            for (int c = 0; c < NC; ++c) pre_v[c] = 0.f;
            if (act_c) {
                const float4* src = src_c;
                const float4 r0 = __ldg(src), r1 = __ldg(src + 32);
                const float D = r0.x, sdx = r0.y, sdy = r0.z, zn = r0.w;  // zn: normalised depth exactly as the forward formed it
                const uint32_t meta = __float_as_uint(r1.w);
                const int pix = TS == 16 ? (int)(meta & 0xffu) : (int)(meta & 0x3ffu);
                const int tix = TS == 16 ? (int)((meta >> 8) & 0x7fffffu) : (int)((meta >> 10) & 0x1fffffu);
                const bool front = (meta >> 31) != 0u;
                const float* sp = &s_pix[0][pix];
                float Cxy = 0.f;
                if (GEOM) {
                    const float g3 = sp[NC * NP];  // gradient of alpha
                    const float one_m_a = 1 - sp[(2 * NC + 1) * NP];
                    // g3 * ((1 - alpha) / max(1 - D, 1e-6)) (kernel.cu:584), in fp32 (the reference promotes to double;
                    // gradients are compared at 1e-4, see DESIGN.md "backward arithmetic")
                    Cxy = (one_m_a == 0.f || g3 == 0.f) ? g3 * one_m_a : g3 * __fdividef(one_m_a, fmaxf(1 - D, 1e-6f));
                }
                if (RGB == 0) {
                    if ((float)f == sp[(NV - 1) * NP]) {  // aggrs[1] = winning face id (:596)
                        if (TEXGRAD) {
                            float* gt = gtex_img + ((size_t)f * K.T2 + tix) * NC;
                            float g_[NC];
#pragma unroll
                            for (int c = 0; c < NC; ++c) g_[c] = sp[c * NP];
                            red_add_texel<NC>(gt, g_);
                        }
                    }
                } else if (front || K.double_side) {
                    float g[NC];
                    bool any = false;
#pragma unroll
                    for (int c = 0; c < NC; ++c) { g[c] = sp[c * NP]; any = any || g[c] != 0.f; }
                    if (any) {
                        const float s = __fdividef(D * expf((zn - sp[(NV - 1) * NP]) * K.r_gamma), sp[(NV - 2) * NP]);  // :608
                        if (s != 0.f) {
                            const size_t to = ((size_t)f * K.T2 + tix) * NC;
                            if (TEXGRAD) {
                                if (PRE) {
                                    pre_tix = tix;
#pragma unroll
                                    for (int c = 0; c < NC; ++c) pre_v[c] = s * g[c];
                                } else {
                                    float sg[NC];
#pragma unroll
                                    for (int c = 0; c < NC; ++c) sg[c] = s * g[c];
                                    red_add_texel<NC>(gtex_img + to, sg);
                                }
                            }
                            float Crgb = 0.f;
                            if (GEOM) {
#pragma unroll
                                for (int c = 0; c < NC; ++c) Crgb += g[c] * (__ldg(tex_img + to + c) - sp[(NPL + c) * NP]);
                                Crgb *= s;
                            }
                            if (GEOM && Crgb != 0.f) {
                                Cxy += __fdividef(Crgb, D);
                                const float zp = K.far_ - zn * (K.far_ - K.near_);
                                const float Cz = Crgb * K.r_gamma * K.r_nf * zp * zp;  // :624
                                // w_clip_k / z_k^2 (kernel.cu:624-627) exactly as the forward forms them: the w of
                                // fragment(), clip_bary, times the face record's 1 / z_k^2
                                const float* q = rec_img + (size_t)f * REC_F;
                                const float xp = s_xp[pix % TS], yp = s_yp[pix / TS];
                                float k0 = __ldg(q + R_INV + 0) * xp + __ldg(q + R_INV + 1) * yp + __ldg(q + R_INV + 2);
                                float k1 = __ldg(q + R_INV + 3) * xp + __ldg(q + R_INV + 4) * yp + __ldg(q + R_INV + 5);
                                float k2 = __ldg(q + R_INV + 6) * xp + __ldg(q + R_INV + 7) * yp + __ldg(q + R_INV + 8);
                                clip_bary(k0, k1, k2);
                                acc[2] += Cz * (k0 * __ldg(q + R_IZ2 + 0));
                                acc[5] += Cz * (k1 * __ldg(q + R_IZ2 + 1));
                                acc[8] += Cz * (k2 * __ldg(q + R_IZ2 + 2));
                            }
                        }
                    }
                }
                if (GEOM) {
                    Cxy *= D * (1 - D) * K.r_sigma;  // :632
                    const float q = 2 * Cxy;          // :640 (the sign rides in sdx / sdy)
                    acc[0] += q * r1.x * sdx;
                    acc[1] += q * r1.x * sdy;
                    acc[3] += q * r1.y * sdx;
                    acc[4] += q * r1.y * sdy;
                    acc[6] += q * r1.z * sdx;
                    acc[7] += q * r1.z * sdy;
                }
            }
            if (PRE && TEXGRAD && RGB == 1) {  // all 32 lanes are here (the stream loop is warp-uniform)
                const bool has = pre_tix >= 0;
                if (__any_sync(0xffffffffu, has)) {
                    const uint32_t lt_ = (1u << lane) - 1u;
                    const uint32_t pm = __match_any_sync(0xffffffffu, has ? (uint32_t)pre_tix : (0x80000000u | (uint32_t)lane));
                    const bool leader = (pm & lt_) == 0u;
                    uint32_t rest = (has && leader) ? (pm & ~(1u << lane)) : 0u;  // the other lanes on this leader's texel
                    float sum[NC];
#pragma unroll
                    for (int c = 0; c < NC; ++c) sum[c] = pre_v[c];
                    while (__any_sync(0xffffffffu, rest != 0u)) {
                        const int src = rest ? __ffs(rest) - 1 : lane;
                        const bool take = rest != 0u;
                        rest &= rest - 1u;
#pragma unroll
                        for (int c = 0; c < NC; ++c) {
                            const float t = __shfl_sync(0xffffffffu, pre_v[c], src);
                            if (take) sum[c] += t;
                        }
                    }
                    if (has && leader) {
                        float* gt = gtex_img + ((size_t)f * K.T2 + pre_tix) * NC;
                        red_add_texel<NC>(gt, sum);
                    }
                }
            }
            f_c = f_n; act_c = act_n; src_c = src_n; have = have_n;
        }
        seg = next;
    }
    flush();
}

}  // namespace umr
