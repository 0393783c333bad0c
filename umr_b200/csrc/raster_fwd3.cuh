// raster_fwd3.cuh -- forward of the round-2 pipeline, per-pixel formulation (included by raster.cu after
// raster_stream.cuh).  A pair-parallel forward spends its gain in lane utilisation on two
// extra CTA phases per sub-chunk, so the forward keeps the round-1 inner loop -- thread = pixel, faces walked in ascending
// index -- and gains: the tile list comes from the coarse bins (no scan of all F cull boxes), untouched tiles take a
// store-only fast path, a warp skips every face whose cull rectangle misses its 8x4 pixel block, and survivors are
// written as pair records for the streaming backward: one 32-slot block per (face, warp block met), face-major, so
// k_raster_bwd2 sees runs of blocks of the same face.
#pragma once

namespace umr {

// CTAs per SM: same-box A/B at C2: 3 CTAs (80 registers) and 5 CTAs (48 registers, 88 B of spills: 0.461 vs 0.386 ms) both lose
constexpr int FWD3_CTAS = 4;

// RGB: 0 = hard z-buffer colours, 1 = softmax aggregation, 2 = VISIBILITY ONLY -- the winning face of the hard z-buffer
// (aggrs planes: depth_min, face_index_min) and nothing else: no distance / sigmoid / alpha / colour arithmetic, no image
// planes.  That is all `MultiTextureLoss` keeps of its hard render (loss_utils.py:327-329: `_, p2f, aggr = hard_renderer(...)`,
// and p2f is zero in hard mode, kernel.cu:417-431).  Same winner as RGB = 0, bit for bit.
// RGB = RGB_SIL (3): SILHOUETTE -- the alpha plane alone: images is [B,is,is] (pooled alpha), colors_hi [B,S,S] (the
// full-resolution alpha for the backward, may be NULL), aggrs / p2f / textures are not touched.  No softmax weight, texel or
// colour work.  Alpha and the set of saved pairs are those of RGB = 0 / 1, bit for bit, and so is every record field the
// SPLIT walk reads for the alpha terms (and zn, as the softmax forward writes it); the texel field holds 0.
// IdxT: face-index width of the coarse lists, the tile list and the pair-block headers (uint16_t: F <= 65535)
// DET: p2f partials go to the fixed-point accumulators of the deterministic mode (red_p2f_fixed) instead of float REDs
template <int RGB, int NC = 3, typename IdxT = uint16_t, bool DET = false>  // NC colour channels (3, or 4: the part-map render of SURVEY.md 8f-2); planes = NC + 1 (alpha)
__global__ void __launch_bounds__(CTA, FWD3_CTAS) k_raster_fwd3(const float* __restrict__ rec_all, const float4* __restrict__ box_all,
                                                        const IdxT* __restrict__ clist, const int* __restrict__ ccount,
                                                        const float* __restrict__ textures, float* __restrict__ images,
                                                        float* __restrict__ colors_hi, float* __restrict__ aggrs,
                                                        float* __restrict__ p2f_acc, const uint32_t* __restrict__ ubox,
                                                        Consts<float> K, float eps, float bg0, float bg1, float bg2, PairBuf pb,
                                                        int ncb, float bg3 = 0.f,
                                                        uint8_t* __restrict__ vis_mask = nullptr) {  // RGB = 2: optional [B,F] "face is visible" bytes; aggrs may be NULL
    constexpr int NPL = NC + 1;                                      // image planes: colours + alpha
    constexpr bool VIS = RGB == 2;
    constexpr bool SIL = RGB == RGB_SIL;
    const float bgc[4] = {bg0, bg1, bg2, bg3};
    constexpr int WG = 16;                                           // list entries per warp group
    __shared__ __align__(128) float s_wrec[NWARP * 2 * WG * REC_LEN];  // 32 KB: warp-private record stages; reused by the store epilogue
    float* s_rec = s_wrec;
    __shared__ IdxT s_list[LCAP];
    __shared__ uint8_t s_meet[LCAP];          // bit w: the face's cull rectangle meets warp w's 8x4 pixel block
    __shared__ uint32_t s_boff[LCAP + 1];     // exclusive prefix of popc(s_meet): first pair block of the face
    __shared__ float s_xp[TILE], s_yp[TILE], s_ext[4];
    __shared__ int s_warp_cnt[NWARP];
    __shared__ uint32_t s_warp_blk[NWARP];
    __shared__ uint32_t s_segbase;
    __shared__ int s_save;
    __shared__ uint8_t s_pos[NWARP][WG];      // list offset of the r-th face of the warp's current issue mask

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z;
    const int S = K.S, F = K.F;
    const int tx0 = blockIdx.x * TILE, ty0 = blockIdx.y * TILE;
    const size_t np = (size_t)S * S;

    tile_extents(S, s_ext);
    if (tid < TILE) s_xp[tid] = pixel_coord(tx0 + tid, S);
    else if (tid < 2 * TILE) s_yp[tid - TILE] = pixel_coord(S - 1 - (ty0 + tid - TILE), S);
    if (tid == 0) s_save = pb.cap > 0 ? 1 : 0;
    __syncthreads();

    const size_t tile_id = ((size_t)b * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    const size_t cidx = ((size_t)b * ncb + (ty0 / CB)) * ncb + (tx0 / CB);
    const bool outside = tile_outside_union(ubox, b, s_ext);
    const CoarseBin<IdxT> cb = outside ? CoarseBin<IdxT>{0, nullptr} : coarse_bin(clist, ccount, cidx, F);
    const int nc = cb.n;

    if (nc == 0) {
        if (VIS) {
            // background pixels carry face id -1, which the reference's indexing turns into "face F-1 is visible"
            // (loss_utils.py:161-166, SURVEY.md App. B); reproduced like k_visible does
            if (vis_mask != nullptr && tid == 0) {
                uint8_t* m = vis_mask + (size_t)b * F + (F - 1);
                if (*reinterpret_cast<volatile uint8_t*>(m) == 0) *m = 1;
            }
            if (aggrs == nullptr) return;  // no planes wanted (uniform)
        }
        // ---- untouched tile (most of the image): every pixel holds the initial state.  Same arithmetic as the
        // general path (kernel.cu:335-348, 443-475), evaluated once, stored with 128-bit stores where possible.
        if (tid == 0 && pb.cap > 0) pb.tile_head[tile_id] = TILE_EMPTY;
        if (SIL) {  // alpha 1 - 1 = 0 everywhere, pooled ((0 + 0) + 0 + 0) * 0.25 = 0
            const int px = tx0 + (tid & (TILE - 1)), py = ty0 + (tid >> 4);
            if (px < S && py < S) {
                const size_t p = (size_t)py * S + px;
                const float a0 = (float)(1. - (double)1.f);
                if (colors_hi != nullptr) colors_hi[(size_t)b * np + p] = a0;
                if (K.aa) {
                    if ((px & 1) == 0 && (py & 1) == 0 && px + 1 < S && py + 1 < S)
                        images[(size_t)b * K.IS * K.IS + (size_t)(py >> 1) * K.IS + (px >> 1)] = (((a0 + a0) + a0) + a0) * 0.25f;
                } else if (images != colors_hi) {
                    images[(size_t)b * np + p] = a0;
                }
            }
            return;
        }
        const float ssum0 = expf(eps / K.gamma);
        float full[NC + 3], g0, g1;
        if (RGB != 1) {
#pragma unroll
            for (int k = 0; k < NC; ++k) full[k] = bgc[k];
            g0 = 10000000.f; g1 = -1.f;
        } else {
#pragma unroll
            for (int k = 0; k < NC; ++k) {
                const float q = bgc[k] * ssum0;
                full[k] = q == 0.f ? q : q / ssum0;
            }
            g0 = ssum0; g1 = eps;
        }
        full[NC] = (float)(1. - (double)1.f);  // alpha
        full[NC + 1] = g0; full[NC + 2] = g1;
        float pooled[NPL];
#pragma unroll
        for (int k = 0; k < NPL; ++k) pooled[k] = (((full[k] + full[k]) + full[k]) + full[k]) * 0.25f;
        if (K.aa && K.vec_store && tx0 + TILE <= S && ty0 + TILE <= S) {
            for (int i = tid; i < (NC + 3) * 64; i += CTA) {
                const int plane = i >> 6, rem = i & 63, row = rem >> 2, q = rem & 3;
                float x = full[0];
#pragma unroll
                for (int k = 1; k < NC + 3; ++k) x = (plane == k) ? full[k] : x;
                const float4 val = make_float4(x, x, x, x);
                const size_t off = (size_t)(ty0 + row) * S + tx0 + q * 4;
                if (plane < NPL) {
                    if (colors_hi != nullptr)
                        *reinterpret_cast<float4*>(colors_hi + ((size_t)b * NPL + plane) * np + off) = val;
                } else {
                    *reinterpret_cast<float4*>(aggrs + ((size_t)b * 2 + (plane - NPL)) * np + off) = val;
                }
            }
            if (!VIS && tid < NPL * 16) {
                const int k = tid >> 4, rem = tid & 15, row = rem >> 1, q = rem & 1;
                float x = pooled[0];
#pragma unroll
                for (int kk = 1; kk < NPL; ++kk) x = (k == kk) ? pooled[kk] : x;
                const int IS = K.IS;
                const size_t nq = (size_t)IS * IS;
                *reinterpret_cast<float4*>(images + ((size_t)b * NPL + k) * nq + (size_t)((ty0 >> 1) + row) * IS + (tx0 >> 1) + q * 4) =
                    make_float4(x, x, x, x);
            }
            return;
        }
        const int px = tx0 + (tid & (TILE - 1)), py = ty0 + (tid >> 4);
        if (px < S && py < S) {
            const size_t p = (size_t)py * S + px;
            aggrs[((size_t)b * 2 + 0) * np + p] = g0;
            aggrs[((size_t)b * 2 + 1) * np + p] = g1;
            if (colors_hi != nullptr) {
#pragma unroll
                for (int k = 0; k < NPL; ++k) colors_hi[((size_t)b * NPL + k) * np + p] = full[k];
            }
            if (VIS) {
            } else if (K.aa) {
                if ((px & 1) == 0 && (py & 1) == 0 && px + 1 < S && py + 1 < S) {
                    const size_t q = (size_t)(py >> 1) * K.IS + (px >> 1);
                    const size_t nq = (size_t)K.IS * K.IS;
#pragma unroll
                    for (int k = 0; k < NPL; ++k) images[((size_t)b * NPL + k) * nq + q] = pooled[k];
                }
            } else if (images != colors_hi) {
#pragma unroll
                for (int k = 0; k < NPL; ++k) images[((size_t)b * NPL + k) * np + p] = full[k];
            }
        }
        return;
    }

    // thread <-> pixel: warp = 8x4 block (map_pixel); coordinates from the shared tables (same bits as pixel_coord)
    const int lcol = (warp & 1) * 8 + (lane & 7), lrow = (warp >> 1) * 4 + (lane >> 3);
    const int px = tx0 + lcol, py = ty0 + lrow;
    const bool live = px < S && py < S;
    const float xp = s_xp[lcol], yp = s_yp[lrow];
    const int ncol = min(TILE, S - tx0), nrow = min(TILE, S - ty0);
    const float4* box = box_all + (size_t)b * F;
    const float* rec_img = rec_all + (size_t)b * F * REC_LEN;
    const float* tex_img = textures + (size_t)(b / K.tex_div) * K.tex_bs;
    const float ext0 = s_ext[0], ext1 = s_ext[1], ext2 = s_ext[2], ext3 = s_ext[3];

    // pixel state (kernel.cu:335-348)
    float acc_a = 1.f;
    float ssum = expf(eps / K.gamma);
    float smax = eps;
    float col[NC];
#pragma unroll
    for (int k = 0; k < NC; ++k) col[k] = RGB == 1 ? bgc[k] * ssum : bgc[k];
    float zmin = 10000000.f;
    int fid = -1;
    // torch-1.1 affine_grid (align_corners=True) coordinates of this pixel: linspace(-1, 1, S)
    // S = 1: torch 1.1's affine_grid takes linspace(-1, 1, 1) = [-1] (DESIGN.md §2), where 2 / 0 would give -1 + inf * 0 = NaN
    const float gstep = S > 1 ? 2.f / (float)(S - 1) : 0.f;
    const float gx = (px * 2 < S) ? (-1.f + gstep * px) : (1.f - gstep * (S - 1 - px));
    const float gy = (py * 2 < S) ? (-1.f + gstep * py) : (1.f - gstep * (S - 1 - py));

    int32_t head = TILE_EMPTY;     // meaningful in thread 0
    uint32_t prev_seg = SEG_NONE;  // meaningful in thread 0
    const uint32_t lt = (1u << lane) - 1u;
    const uint32_t wbit = 1u << warp, wlow = wbit - 1u;

    for (int w0 = 0; w0 < nc; w0 += LCAP) {
        // ---- tile-list segment: ordered compaction of this window's coarse entries that touch the tile ------
        const int nwin = min(LCAP, nc - w0);
        uint32_t masks[LCAP / CTA];
        IdxT fids[LCAP / CTA];
        uint8_t meets[LCAP / CTA];
        int cnt = 0;
#pragma unroll
        for (int r = 0; r < LCAP / CTA; ++r) {
            const int i = warp * (LCAP / NWARP) + r * 32 + lane;
            bool hit = false;
            uint32_t meet = 0;
            IdxT f = 0;
            if (i < nwin) {
                f = (IdxT)bin_face(cb, w0 + i);
                const float4 bb = __ldg(box + f);
                hit = !(ext0 > bb.y || ext1 < bb.x || ext2 > bb.w || ext3 < bb.z);
                if (hit) {
                    // which 8-column halves / 4-row bands hold a pixel passing the per-pixel cull test
                    // !(xp > hi || xp < lo || yp > hi || yp < lo) (kernel.cu:32-38)?  Same comparisons, so a NaN box
                    // stays "never culled" like the per-pixel form.
                    uint32_t cm = 0, rm = 0;
#pragma unroll
                    for (int q = 0; q < TILE; ++q) {
                        const float x = s_xp[q], y = s_yp[q];
                        if (q < ncol && !(x > bb.y || x < bb.x)) cm |= 1u << (q >> 3);
                        if (q < nrow && !(y > bb.w || y < bb.z)) rm |= 1u << (q >> 2);
                    }
#pragma unroll
                    for (int w = 0; w < NWARP; ++w)
                        if (((cm >> (w & 1)) & 1u) && ((rm >> (w >> 1)) & 1u)) meet |= 1u << w;
                }
            }
            masks[r] = __ballot_sync(0xffffffffu, hit);
            meets[r] = (uint8_t)meet;
            fids[r] = f;
            cnt += __popc(masks[r]);
        }
        if (lane == 0) s_warp_cnt[warp] = cnt;
        __syncthreads();
        int off = 0, n = 0;
#pragma unroll
        for (int w = 0; w < NWARP; ++w) {
            const int c = s_warp_cnt[w];
            if (w < warp) off += c;
            n += c;
        }
#pragma unroll
        for (int r = 0; r < LCAP / CTA; ++r) {
            if ((masks[r] >> lane) & 1u) {
                const int pos = off + __popc(masks[r] & lt);
                s_list[pos] = fids[r];
                s_meet[pos] = meets[r];
            }
            off += __popc(masks[r]);
        }
        __syncthreads();  // list + meet masks visible; s_warp_cnt reusable
        if (n == 0) continue;  // uniform

        // ---- block offsets: exclusive prefix of popc(meet) over the segment (2 entries per thread) ---------------
        {
            const int i0 = 2 * tid, i1 = 2 * tid + 1;
            const uint32_t v0 = i0 < n ? __popc((uint32_t)s_meet[i0]) : 0u, v1 = i1 < n ? __popc((uint32_t)s_meet[i1]) : 0u;
            uint32_t incl = v0 + v1;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += o;
            }
            if (lane == 31) s_warp_blk[warp] = incl;
            __syncthreads();
            uint32_t base = 0, total = 0;
#pragma unroll
            for (int w = 0; w < NWARP; ++w) {
                const uint32_t c = s_warp_blk[w];
                base += (w < warp) ? c : 0u;
                total += c;
            }
            const uint32_t excl = base + incl - (v0 + v1);
            if (i0 < n) s_boff[i0] = excl;
            if (i1 < n) s_boff[i1] = excl + v0;
            if (tid == 0) s_boff[n] = total;
        }
        __syncthreads();
        const uint32_t NBw = s_boff[n];
        if (NBw == 0) continue;  // uniform: no rectangle holds a pixel

        // ---- reserve the segment's blocks in the pair buffer --------------------------------------------------
        if (tid == 0 && *reinterpret_cast<volatile int*>(&s_save)) {  // thread 0 only (volatile: the read is not hoisted)
            const uint32_t base = atomicAdd(pb.ctrl, NBw + 2u);
            if ((uint64_t)base + NBw + 2u > (uint64_t)pb.cap) {
                s_save = 0;  // does not fit: the whole tile falls back to the recompute backward
                head = TILE_UNSAVED;
                pb.ulist[atomicAdd(pb.ctrl + 1, 1u)] = (int32_t)tile_id;
            } else {
                pb.blk_hdr[base] = NBw;
                pb.blk_hdr[base + 1] = SEG_NONE;
                if (prev_seg == SEG_NONE) head = (int32_t)base;
                else pb.blk_hdr[prev_seg + 1] = base;
                prev_seg = base;
                s_segbase = base + 2u;
            }
        }

        __syncthreads();  // s_save / s_segbase visible
        const bool save = s_save != 0;
        const uint32_t segbase = s_segbase;

        // ---- warp-autonomous main loop: NO CTA barrier.  Each warp walks the segment's faces in groups of WG list
        // entries, stages the records of the faces that meet ITS pixel block into a warp-private double buffer
        // (cp.async, 8 lanes x 16 B per record) and aggregates them in ascending face order.  Warps over empty parts of
        // the tile finish early instead of waiting at chunk barriers (30 % of the stall samples of the barrier version).
        float* wst = s_wrec + warp * (2 * WG * REC_LEN);
        const int ngroup = (n + WG - 1) / WG;
        auto issue = [&](int g) -> uint32_t {
            uint32_t m = 0;
            if (g < ngroup) {
                const int base = g * WG;
                m = __ballot_sync(0xffffffffu, lane < WG && base + lane < n && (s_meet[min(base + lane, n - 1)] & wbit));
                const int cntm = __popc(m);
                // rank -> list offset through a 16-byte per-warp table (the find-n-th-set-bit intrinsic is a software loop;
                // same-box A/B 0.385 -> 0.381 ms at C2)
                if ((m >> lane) & 1u) s_pos[warp][__popc(m & lt)] = (uint8_t)lane;
                __syncwarp();
                for (int r = lane >> 3; r < cntm; r += 4) {
                    const int e = s_pos[warp][r];  // list offset of the r-th face this warp needs
                    const int f = s_list[base + e];
                    cp_async16(wst + ((size_t)(g & 1) * WG + r) * REC_LEN + (lane & 7) * 4, rec_img + (size_t)f * REC_LEN + (lane & 7) * 4);
                }
            }
            __syncwarp();  // table reads done before the next issue() rewrites it
            cp_async_commit();
            return m;
        };
        uint32_t m_cur = issue(0);
        for (int g = 0; g < ngroup; ++g) {
            const uint32_t m_next = issue(g + 1);
            cp_async_wait<1>();  // group g has landed for this lane (g + 1 may still be in flight)
            __syncwarp();        // ... and for the other lanes of the warp
            const int base = g * WG;
            const float* stage = wst + (size_t)(g & 1) * WG * REC_LEN;
            float own_x = 0.f, own_y = 0.f, own_w = 0.f;  // p2f partial sums: lane r owns the r-th staged face
            uint32_t mm = m_cur;
            for (int r = 0; mm; ++r) {
                const int e = __ffs(mm) - 1;
                mm &= mm - 1u;
                const int jl = base + e;  // list position
                const uint32_t meet = s_meet[jl];
                const float* rc = stage + r * REC_LEN;
                const float4 bb = *reinterpret_cast<const float4*>(rc + R_BOX);
                float a_x = 0.f, a_y = 0.f, a_w = 0.f;
                bool contrib = false, emit = false;
                Frag<float> fr;
                float k0 = 0.f, k1 = 0.f, k2 = 0.f, zsave = 0.f;
                uint32_t tix = 0, front = 0;
                if (VIS) {
                    if (live && !(xp > bb.y || xp < bb.x || yp > bb.w || yp < bb.z)) {
                        // only a pixel inside the triangle (closed barycentric test, kernel.cu:404) can win the z-buffer
                        const float w0 = rc[R_INV + 0] * xp + rc[R_INV + 1] * yp + rc[R_INV + 2];
                        const float w1 = rc[R_INV + 3] * xp + rc[R_INV + 4] * yp + rc[R_INV + 5];
                        const float w2 = rc[R_INV + 6] * xp + rc[R_INV + 7] * yp + rc[R_INV + 8];
                        const bool inside = w0 <= 1 && w0 >= 0 && w1 <= 1 && w1 >= 0 && w2 <= 1 && w2 >= 0;
                        if (inside && (K.double_side || (__float_as_uint(rc[R_FLG]) & 8u))) {
                            // strictly inside pixels always pass the distance test (kernel.cu:380-383); a barycentric that is
                            // exactly 0 or 1 takes the reference's outside branch -- evaluate it as the full kernel does
                            bool pass = w0 > 0 && w1 > 0 && w2 > 0 && w0 < 1 && w1 < 1 && w2 < 1;
                            if (!pass) pass = fragment(rc, xp, yp, K.thr, K.sigma, fr);
                            if (pass) {
                                k0 = w0; k1 = w1; k2 = w2;
                                clip_bary(k0, k1, k2);
                                const float zp = depth_of(rc, k0, k1, k2);
                                if (!(zp < K.near_ || zp > K.far_) && zp < zmin) {
                                    zmin = zp;
                                    fid = s_list[jl];
                                }
                            }
                        }
                    }
                } else if (live && !(xp > bb.y || xp < bb.x || yp > bb.w || yp < bb.z)) {
                    if (fragment(rc, xp, yp, K.thr, K.sigma, fr)) {
                        acc_a = (float)((double)acc_a * (1. - (double)fr.D));  // kernel.cu:396
                        k0 = fr.w0; k1 = fr.w1; k2 = fr.w2;
                        clip_bary(k0, k1, k2);
                        const float zp = depth_of(rc, k0, k1, k2);
                        if (!(zp < K.near_ || zp > K.far_)) {
                            emit = true;  // kernel.cu:592: pairs outside the depth range get no gradient at all
                            front = (__float_as_uint(rc[R_FLG]) & 8u) ? 1u : 0u;
                            tix = SIL ? 0u : (uint32_t)texel_index(k0, k1, K.R);
                            const int f = s_list[jl];
                            zsave = zp;
                            if (SIL) {
                                zsave = (K.far_ - zp) / (K.far_ - K.near_);  // the softmax forward's zn (below)
                            } else if (RGB == 0) {
                                const bool inside = fr.w0 <= 1 && fr.w0 >= 0 && fr.w1 <= 1 && fr.w1 >= 0 &&
                                                    fr.w2 <= 1 && fr.w2 >= 0;
                                if (zp < zmin && inside && (K.double_side || front)) {
                                    zmin = zp;
                                    fid = f;
                                    const float* tp = tex_img + ((size_t)f * K.T2 + tix) * NC;
#pragma unroll
                                    for (int k = 0; k < NC; ++k) col[k] = __ldg(tp + k);
                                }
                            } else {
                                // normalised depth (kernel.cu:418); the backward needs THESE bits (its softmax weight is
                                // exp((zn - max) / gamma): 1 ulp of zn is a 5e-4 relative change of the weight)
                                const float zn = (K.far_ - zp) / (K.far_ - K.near_);
                                zsave = zn;
                                if (front || K.double_side) {
                                    float ed = 1.f;
                                    if (zn > smax) { ed = expf((smax - zn) / K.gamma); smax = zn; }
                                    const float ez = expf((zn - smax) / K.gamma);
                                    ssum = ed * ssum + ez * fr.D;
                                    const float a = ez * fr.D;
                                    // a == 0 with no max update: c = 1*c + 0*texel, p2f terms 0 -- skip the texel fetch (exact)
                                    if (a != 0.f || ed != 1.f) {
                                        a_x = a * gx; a_y = a * gy; a_w = a;
                                        contrib = a != 0.f;
                                        const float* tp = tex_img + ((size_t)f * K.T2 + tix) * NC;
#pragma unroll
                                        for (int k = 0; k < NC; ++k) col[k] = ed * col[k] + a * __ldg(tp + k);
                                    }
                                }
                            }
                        }
                    }
                }
                if (save) {  // uniform: one 32-slot block per (face, warp block met); survivors compacted to its front
                    const uint32_t m = __ballot_sync(0xffffffffu, emit);
                    const uint32_t blk = segbase + s_boff[jl] + (uint32_t)__popc(meet & wlow);
                    if (emit) {
                        float4* dst = pb.recs + (size_t)blk * BLK_F4 + __popc(m & lt);
                        // closest-point barycentrics as the reference forms them: t_k + w_k (kernel.cu:638-641)
                        const float u0 = fr.t0 + fr.w0, u1 = fr.t1 + fr.w1, u2 = fr.t2 + fr.w2;
                        // meta: pixel in bits 0-7, texel in bits 8-30 (T2 <= 2^23, make_pairbuf), front in bit 31
                        const uint32_t meta = (uint32_t)(lrow * TILE + lcol) | (tix << 8) | (front << 31);
                        dst[0] = make_float4(fr.D, fr.sign * fr.dx, fr.sign * fr.dy, zsave);
                        dst[32] = make_float4(u0, u1, u2, __uint_as_float(meta));
                    }
                    if (lane == 0) pb.blk_hdr[blk] = (uint32_t)s_list[jl] | ((uint32_t)__popc(m) << hdr_shift<IdxT>());
                }
                if (RGB == 1 && p2f_acc != nullptr) {
                    // p2f: warp-shuffle reduction (replaces the 4 global atomics per (pixel, face) of kernel.cu:427-430)
                    if (__any_sync(0xffffffffu, contrib)) {
                        a_x = warp_sum(a_x); a_y = warp_sum(a_y); a_w = warp_sum(a_w);
                        if (lane == r) { own_x += a_x; own_y += a_y; own_w += a_w; }
                    }
                }
            }
            if (RGB == 1 && p2f_acc != nullptr) {  // one global RED per (warp, face, component)
                if (own_w != 0.f) {  // lane r owns the r-th staged face of the group
                    const int e = __fns(m_cur, 0, lane + 1);
                    if constexpr (DET) {
                        red_p2f_fixed(reinterpret_cast<unsigned long long*>(p2f_acc) + ((size_t)b * F + s_list[base + e]) * P2F_DET_WORDS,
                                      own_x, own_y, own_w);
                    } else {
                    float* dst = p2f_acc + ((size_t)b * F + s_list[base + e]) * 4;
                    red_add4_global(dst, own_x, own_y, own_w, 0.f);  // the accumulator slots are 16-byte aligned (ws_layout)
                    }
                }
            }
            __syncwarp();  // every lane is done with stage g & 1 before issue(g + 2) overwrites it
            m_cur = m_next;
        }
        cp_async_wait<0>();
        __syncthreads();  // segment done: s_list / s_meet / s_boff / s_rec reusable
    }
    if (tid == 0 && pb.cap > 0) pb.tile_head[tile_id] = head;

    // ---- finalise (kernel.cu:443-475) + fused 2x2 pool + coalesced stores (as round 1) --------------------
    const float alpha = (float)(1. - (double)acc_a);  // kernel.cu:449-451
    if (SIL) {  // the alpha plane of the epilogue below: same value, same pooling sum
        float v = alpha;
        if (K.aa) {
            const float a01 = __shfl_xor_sync(0xffffffffu, v, 1);
            const float a10 = __shfl_xor_sync(0xffffffffu, v, 8);
            const float a11 = __shfl_xor_sync(0xffffffffu, v, 9);
            v = (((v + a01) + a10) + a11) * 0.25f;  // meaningful on the (even x, even y) lane
        }
        if (live) {
            const size_t p = (size_t)py * S + px;
            if (colors_hi != nullptr) colors_hi[(size_t)b * np + p] = alpha;
            if (K.aa) {
                if ((lane & 1) == 0 && (lane & 8) == 0)
                    images[(size_t)b * K.IS * K.IS + (size_t)(py >> 1) * K.IS + (px >> 1)] = v;
            } else if (images != colors_hi) {
                images[(size_t)b * np + p] = alpha;
            }
        }
        return;
    }
    if (VIS) {
        // face-visibility bytes (what TexCycle derives from the face-index plane with torch.unique, loss_utils.py:161-166):
        // test before set -- a stale 0 only repeats the store
        if (vis_mask != nullptr && live) {
            uint8_t* m = vis_mask + (size_t)b * F + (fid >= 0 ? fid : F - 1);  // -1 (background) marks face F-1, see above
            if (*reinterpret_cast<volatile uint8_t*>(m) == 0) *m = 1;
        }
        if (aggrs == nullptr) return;  // uniform
    }
    float v[NPL], hi[NPL], g0, g1;  // hi: full-resolution planes, v: pooled
    if (RGB != 1) {
#pragma unroll
        for (int k = 0; k < NC; ++k) hi[k] = col[k];
        g0 = zmin; g1 = (float)fid;
    } else {
#pragma unroll
        for (int k = 0; k < NC; ++k) hi[k] = col[k] == 0.f ? col[k] : col[k] / ssum;
        g0 = ssum; g1 = smax;
    }
    hi[NC] = alpha;
#pragma unroll
    for (int k = 0; k < NPL; ++k) v[k] = hi[k];
    if (K.aa) {
#pragma unroll
        for (int k = 0; k < NPL; ++k) {
            const float a01 = __shfl_xor_sync(0xffffffffu, v[k], 1);
            const float a10 = __shfl_xor_sync(0xffffffffu, v[k], 8);
            const float a11 = __shfl_xor_sync(0xffffffffu, v[k], 9);
            v[k] = (((v[k] + a01) + a10) + a11) * 0.25f;  // meaningful on the (even x, even y) lane
        }
    }
    if (K.aa && K.vec_store && tx0 + TILE <= S && ty0 + TILE <= S) {  // uniform: full tile, aligned buffers
        float* st = s_rec;  // (NC + 3) * 256 + (NC + 1) * 64 floats (2112 for NC = 4) <= 8192
        const int o = lrow * TILE + lcol;
#pragma unroll
        for (int k = 0; k < NPL; ++k) st[k * 256 + o] = hi[k];
        st[NPL * 256 + o] = g0; st[(NPL + 1) * 256 + o] = g1;
        if ((lane & 1) == 0 && (lane & 8) == 0) {
            const int po = (lrow >> 1) * (TILE / 2) + (lcol >> 1);
#pragma unroll
            for (int k = 0; k < NPL; ++k) st[(NC + 3) * 256 + k * 64 + po] = v[k];
        }
        __syncthreads();
        for (int i = tid; i < (NC + 3) * 64; i += CTA) {
            const int plane = i >> 6, rem = i & 63, row = rem >> 2, q = rem & 3;
            const float4 val = *reinterpret_cast<const float4*>(st + plane * 256 + row * TILE + q * 4);
            const size_t off = (size_t)(ty0 + row) * S + tx0 + q * 4;
            if (plane < NPL) {
                if (colors_hi != nullptr)
                    *reinterpret_cast<float4*>(colors_hi + ((size_t)b * NPL + plane) * np + off) = val;
            } else {
                *reinterpret_cast<float4*>(aggrs + ((size_t)b * 2 + (plane - NPL)) * np + off) = val;
            }
        }
        if (!VIS && tid < NPL * 16) {
            const int k = tid >> 4, rem = tid & 15, row = rem >> 1, q = rem & 1;
            const float4 val = *reinterpret_cast<const float4*>(st + (NC + 3) * 256 + k * 64 + row * (TILE / 2) + q * 4);
            const int IS = K.IS;
            const size_t nq = (size_t)IS * IS;
            *reinterpret_cast<float4*>(images + ((size_t)b * NPL + k) * nq + (size_t)((ty0 >> 1) + row) * IS + (tx0 >> 1) + q * 4) = val;
        }
        return;
    }
    if (live) {
        const size_t p = (size_t)py * S + px;
        aggrs[((size_t)b * 2 + 0) * np + p] = g0;
        aggrs[((size_t)b * 2 + 1) * np + p] = g1;
        if (colors_hi != nullptr) {
#pragma unroll
            for (int k = 0; k < NPL; ++k) colors_hi[((size_t)b * NPL + k) * np + p] = hi[k];
        }
    }
    if (VIS) {
    } else if (K.aa) {
        if (live && (lane & 1) == 0 && (lane & 8) == 0) {
            const int IS = K.IS;
            const size_t q = (size_t)(py >> 1) * IS + (px >> 1);
            const size_t nq = (size_t)IS * IS;
#pragma unroll
            for (int k = 0; k < NPL; ++k) images[((size_t)b * NPL + k) * nq + q] = v[k];
        }
    } else if (live && images != colors_hi) {
        const size_t p = (size_t)py * S + px;
#pragma unroll
        for (int k = 0; k < NPL; ++k) images[((size_t)b * NPL + k) * np + p] = hi[k];
    }
}

}  // namespace umr
