// raster_fwd4.cuh -- forward with DYNAMIC pixel-block scheduling (included by raster.cu after raster_fwd3.cuh).
//
// Why: in k_raster_fwd3 (one CTA = one 16x16 tile, warp w = the tile's w-th 8x4 pixel block) the warps over empty parts
// of a tile finish at once and then hold their registers until the tile's slowest warp is done, waiting at the end-of-tile
// barrier with part of the warp slots idle.  Here a
// CTA owns a 32x32 tile (32 pixel blocks of 8x4) and its 8 warps GRAB blocks from a shared counter: a warp that draws an
// empty block stores the background and takes the next one, so the tile's work spreads over all warps; the tile list
// (built once, cooperatively, from the coarse bin's list) is amortised over 4x more pixels.  Per block the arithmetic is
// k_raster_fwd3's: thread = pixel, faces in ascending index, records staged into a warp-private cp.async double buffer,
// pair records emitted per (face, pixel block met), face-major inside the tile.
//
// The tile list lives in shared memory (FWD4_CAP entries).  A tile whose coarse-bin list is longer than that (a very
// dense mesh region) takes the SLOW path: the list is processed in windows with a static block assignment (4 passes of
// 8 blocks, pixel state kept in registers across the windows of a pass) and the tile is left to the recompute backward.
#pragma once

namespace umr {

constexpr int T4 = 32;            // tile side
constexpr int FWD4_CAP = 1536;    // tile-list entries held in shared memory (10 bytes each)
constexpr int WG4 = 16;           // list entries per warp group

// bytes per list entry: block offset + meet mask + face index
__host__ __device__ inline size_t fwd4_dyn_smem(int F, size_t idx_bytes = 2) {
    return (size_t)(F < FWD4_CAP ? F : FWD4_CAP) * (8 + idx_bytes) + 16;
}

// IdxT: face-index width of the coarse lists, the tile list and the pair-block headers (uint16_t: F <= 65535)
template <int RGB, typename IdxT = uint16_t>
__global__ void __launch_bounds__(CTA, 4) k_raster_fwd4(const float* __restrict__ rec_all, const float4* __restrict__ box_all,
                                                        const IdxT* __restrict__ clist, const int* __restrict__ ccount,
                                                        const float* __restrict__ textures, float* __restrict__ images,
                                                        float* __restrict__ colors_hi, float* __restrict__ aggrs,
                                                        float* __restrict__ p2f_acc, const uint32_t* __restrict__ ubox,
                                                        Consts K, float eps, float bg0, float bg1, float bg2, PairBuf pb,
                                                        int ncb) {
    extern __shared__ __align__(16) unsigned char smem_dyn[];
    const int F = K.F;
    const int LC = F < FWD4_CAP ? F : FWD4_CAP;                               // list capacity
    uint32_t* s_boff = reinterpret_cast<uint32_t*>(smem_dyn);                 // [LC + 1]
    uint32_t* s_meet = s_boff + (LC + 1);                                     // [LC]  bit q: rectangle meets pixel block q
    IdxT* s_list = reinterpret_cast<IdxT*>(s_meet + LC);                      // [LC]
    __shared__ __align__(128) float s_wrec[NWARP * 2 * WG4 * REC_F];          // 32 KB: warp-private record stages
    __shared__ float s_xp[T4], s_yp[T4], s_ext[4];
    __shared__ int s_warp_cnt[NWARP];
    __shared__ uint32_t s_warp_blk[NWARP];
    __shared__ uint32_t s_segbase;
    __shared__ int s_save, s_next;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z;
    const int S = K.S;
    const int tx0 = blockIdx.x * T4, ty0 = blockIdx.y * T4;
    const size_t np = (size_t)S * S;

    tile_extents_at(S, s_ext, T4, (int)blockIdx.x, (int)blockIdx.y);
    if (tid < T4) s_xp[tid] = pixel_coord(tx0 + tid, S);
    else if (tid < 2 * T4) s_yp[tid - T4] = pixel_coord(S - 1 - (ty0 + tid - T4), S);
    if (tid == 0) { s_save = pb.cap > 0 ? 1 : 0; s_next = 0; }
    __syncthreads();

    const size_t tile_id = ((size_t)b * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    const size_t cidx = ((size_t)b * ncb + (ty0 / CB)) * ncb + (tx0 / CB);
    const bool outside = tile_outside_union(ubox, b, s_ext);
    const CoarseBin<IdxT> cb = outside ? CoarseBin<IdxT>{0, nullptr} : coarse_bin(clist, ccount, cidx, F);
    const int nc = cb.n;

    // the initial pixel state, finalised (kernel.cu:335-348, 443-475): what an untouched pixel stores
    const float ssum0 = expf(eps / K.gamma);
    float e0, e1, e2, eg0, eg1;
    if (RGB == 0) {
        e0 = bg0; e1 = bg1; e2 = bg2;
        eg0 = 10000000.f; eg1 = -1.f;
    } else {
        const float q0 = bg0 * ssum0, q1 = bg1 * ssum0, q2 = bg2 * ssum0;
        e0 = q0 == 0.f ? q0 : q0 / ssum0;
        e1 = q1 == 0.f ? q1 : q1 / ssum0;
        e2 = q2 == 0.f ? q2 : q2 / ssum0;
        eg0 = ssum0; eg1 = eps;
    }

    if (nc == 0) {
        // ---- untouched tile: store-only, 128-bit stores where the tile is full and the buffers are aligned
        if (tid == 0 && pb.cap > 0) pb.tile_head[tile_id] = TILE_EMPTY;
        const float alpha = (float)(1. - (double)1.f);
        const float full[6] = {e0, e1, e2, alpha, eg0, eg1};
        float pooled[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) pooled[k] = (((full[k] + full[k]) + full[k]) + full[k]) * 0.25f;
        if (K.aa && K.vec_store && tx0 + T4 <= S && ty0 + T4 <= S) {
            for (int i = tid; i < 6 * T4 * (T4 / 4); i += CTA) {  // 6 planes x 32 rows x 8 float4
                const int plane = i / (T4 * (T4 / 4)), rem = i % (T4 * (T4 / 4)), row = rem >> 3, q = rem & 7;
                float x = full[0];
#pragma unroll
                for (int k = 1; k < 6; ++k) x = (plane == k) ? full[k] : x;
                const float4 val = make_float4(x, x, x, x);
                const size_t off = (size_t)(ty0 + row) * S + tx0 + q * 4;
                if (plane < 4) {
                    if (colors_hi != nullptr)
                        *reinterpret_cast<float4*>(colors_hi + ((size_t)b * 4 + plane) * np + off) = val;
                } else {
                    *reinterpret_cast<float4*>(aggrs + ((size_t)b * 2 + (plane - 4)) * np + off) = val;
                }
            }
            {   // 4 pooled planes x 16 rows x 4 float4 = 256 stores
                const int k = tid >> 6, rem = tid & 63, row = rem >> 2, q = rem & 3;
                float x = pooled[0];
#pragma unroll
                for (int kk = 1; kk < 4; ++kk) x = (k == kk) ? pooled[kk] : x;
                const int IS = K.IS;
                const size_t nq = (size_t)IS * IS;
                *reinterpret_cast<float4*>(images + ((size_t)b * 4 + k) * nq + (size_t)((ty0 >> 1) + row) * IS + (tx0 >> 1) + q * 4) =
                    make_float4(x, x, x, x);
            }
            return;
        }
        for (int pi = tid; pi < T4 * T4; pi += CTA) {
            const int px = tx0 + (pi & (T4 - 1)), py = ty0 + (pi >> 5);
            if (px >= S || py >= S) continue;
            const size_t p = (size_t)py * S + px;
            aggrs[((size_t)b * 2 + 0) * np + p] = eg0;
            aggrs[((size_t)b * 2 + 1) * np + p] = eg1;
            if (colors_hi != nullptr) {
#pragma unroll
                for (int k = 0; k < 4; ++k) colors_hi[((size_t)b * 4 + k) * np + p] = full[k];
            }
            if (K.aa) {
                if ((px & 1) == 0 && (py & 1) == 0) {
                    const size_t q = (size_t)(py >> 1) * K.IS + (px >> 1);
                    const size_t nq = (size_t)K.IS * K.IS;
#pragma unroll
                    for (int k = 0; k < 4; ++k) images[((size_t)b * 4 + k) * nq + q] = pooled[k];
                }
            } else if (images != colors_hi) {
#pragma unroll
                for (int k = 0; k < 4; ++k) images[((size_t)b * 4 + k) * np + p] = full[k];
            }
        }
        return;
    }

    const int ncol = min(T4, S - tx0), nrow = min(T4, S - ty0);
    const float4* box = box_all + (size_t)b * F;
    const float* rec_img = rec_all + (size_t)b * F * REC_F;
    const float* tex_img = textures + (size_t)(b / K.tex_div) * K.tex_bs;
    const float ext0 = s_ext[0], ext1 = s_ext[1], ext2 = s_ext[2], ext3 = s_ext[3];
    const uint32_t lt = (1u << lane) - 1u;

    // ---- tile list: ordered compaction of the coarse entries [w0, w0 + nwin) that touch the tile (cooperative) -------
    auto build_list = [&](int w0, int nwin) -> int {
        int n = 0;
        for (int r0 = 0; r0 < nwin; r0 += CTA) {
            const int i = r0 + tid;
            bool hit = false;
            uint32_t meet = 0;
            IdxT f = 0;
            if (i < nwin) {
                f = (IdxT)bin_face(cb, w0 + i);
                const float4 bb = __ldg(box + f);
                hit = !(ext0 > bb.y || ext1 < bb.x || ext2 > bb.w || ext3 < bb.z);
                if (hit) {
                    // 8-column bands / 4-row bands holding a pixel that passes the per-pixel cull test (kernel.cu:32-38);
                    // same comparisons, so a NaN box stays "never culled"
                    uint32_t cm = 0, rm = 0;
#pragma unroll 8
                    for (int q = 0; q < T4; ++q) {
                        const float x = s_xp[q], y = s_yp[q];
                        if (q < ncol && !(x > bb.y || x < bb.x)) cm |= 1u << (q >> 3);
                        if (q < nrow && !(y > bb.w || y < bb.z)) rm |= 1u << (q >> 2);
                    }
#pragma unroll
                    for (int r = 0; r < 8; ++r)
                        if ((rm >> r) & 1u) meet |= cm << (4 * r);  // block q = r * 4 + c
                }
            }
            const uint32_t m = __ballot_sync(0xffffffffu, hit);
            if (lane == 0) s_warp_cnt[warp] = __popc(m);
            __syncthreads();
            int off = n, tot = 0;
#pragma unroll
            for (int w = 0; w < NWARP; ++w) {
                const int c = s_warp_cnt[w];
                if (w < warp) off += c;
                tot += c;
            }
            if (hit) {
                const int pos = off + __popc(m & lt);
                s_list[pos] = f;
                s_meet[pos] = meet;
            }
            n += tot;
            __syncthreads();  // entries visible; s_warp_cnt reusable
        }
        return n;
    };
    const bool slow = nc > LC;  // uniform: the bin's list does not fit the shared tile list -> windowed static path below
    float* wst = s_wrec + warp * (2 * WG4 * REC_F);
    const float gstep = 2.f / (float)(S - 1);

    struct PixelState { float acc_a, ssum, smax, c0, c1, c2, zmin; int fid; };
    auto init_state = [&](PixelState& st) {  // kernel.cu:335-348
        st.acc_a = 1.f; st.ssum = ssum0; st.smax = eps;
        if (RGB == 1) { st.c0 = bg0 * ssum0; st.c1 = bg1 * ssum0; st.c2 = bg2 * ssum0; }
        else { st.c0 = bg0; st.c1 = bg1; st.c2 = bg2; }
        st.zmin = 10000000.f; st.fid = -1;
    };

    // ---- one pixel block (8x4, block q of the tile) against the n list entries currently in shared memory: the warp walks
    // the entries in groups of WG4, stages the records of the faces meeting ITS block into its private cp.async double
    // buffer and aggregates them in ascending face order.  No CTA barrier inside.
    auto run_groups = [&](int q, int n, bool save, uint32_t segbase, PixelState& st) {
        const uint32_t qbit = 1u << q, qlow = qbit - 1u;
        const int lcol = (q & 3) * 8 + (lane & 7), lrow = (q >> 2) * 4 + (lane >> 3);
        const int px = tx0 + lcol, py = ty0 + lrow;
        const bool live = px < S && py < S;
        const float xp = s_xp[lcol], yp = s_yp[lrow];
        // torch-1.1 affine_grid (align_corners=True) coordinates of this pixel: linspace(-1, 1, S)
        const float gx = (px * 2 < S) ? (-1.f + gstep * px) : (1.f - gstep * (S - 1 - px));
        const float gy = (py * 2 < S) ? (-1.f + gstep * py) : (1.f - gstep * (S - 1 - py));
        float acc_a = st.acc_a, ssum = st.ssum, smax = st.smax, c0 = st.c0, c1 = st.c1, c2 = st.c2, zmin = st.zmin;
        int fid = st.fid;
        const int ngroup = (n + WG4 - 1) / WG4;
        auto issue = [&](int g) -> uint32_t {
            uint32_t m = 0;
            if (g < ngroup) {
                const int base = g * WG4;
                m = __ballot_sync(0xffffffffu, lane < WG4 && base + lane < n && (s_meet[min(base + lane, n - 1)] & qbit));
                const int cntm = __popc(m);
                for (int r = lane >> 3; r < cntm; r += 4) {
                    const int e = __fns(m, 0, r + 1);  // list offset of the r-th face this block needs
                    const int f = s_list[base + e];
                    cp_async16(wst + ((size_t)(g & 1) * WG4 + r) * REC_F + (lane & 7) * 4, rec_img + (size_t)f * REC_F + (lane & 7) * 4);
                }
            }
            cp_async_commit();
            return m;
        };
        uint32_t m_cur = issue(0);
        for (int g = 0; g < ngroup; ++g) {
            const uint32_t m_next = issue(g + 1);
            cp_async_wait<1>();  // group g has landed for this lane (g + 1 may still be in flight)
            __syncwarp();        // ... and for the other lanes of the warp
            const int base = g * WG4;
            const float* stage = wst + (size_t)(g & 1) * WG4 * REC_F;
            float own_x = 0.f, own_y = 0.f, own_w = 0.f;  // p2f partial sums: lane r owns the r-th staged face
            uint32_t mm = m_cur;
            for (int r = 0; mm; ++r) {
                const int e = __ffs(mm) - 1;
                mm &= mm - 1u;
                const int jl = base + e;  // list position
                const float* rc = stage + r * REC_F;
                const float4 bb = *reinterpret_cast<const float4*>(rc + R_BOX);
                float a_x = 0.f, a_y = 0.f, a_w = 0.f;
                bool contrib = false, emit = false;
                Frag fr;
                float k0 = 0.f, k1 = 0.f, k2 = 0.f, zsave = 0.f;
                uint32_t tix = 0, front = 0;
                if (live && !(xp > bb.y || xp < bb.x || yp > bb.w || yp < bb.z)) {
                    if (fragment(rc, xp, yp, K.thr, K.sigma, fr)) {
                        acc_a = (float)((double)acc_a * (1. - (double)fr.D));  // kernel.cu:396
                        k0 = fr.w0; k1 = fr.w1; k2 = fr.w2;
                        clip_bary(k0, k1, k2);
                        const float zp = depth_of(rc, k0, k1, k2);
                        if (!(zp < K.near_ || zp > K.far_)) {
                            emit = true;  // kernel.cu:592: pairs outside the depth range get no gradient at all
                            front = (__float_as_uint(rc[R_FLG]) & 8u) ? 1u : 0u;
                            tix = (uint32_t)texel_index(k0, k1, K.R);
                            const int f = s_list[jl];
                            zsave = zp;
                            if (RGB == 0) {
                                const bool inside = fr.w0 <= 1 && fr.w0 >= 0 && fr.w1 <= 1 && fr.w1 >= 0 &&
                                                    fr.w2 <= 1 && fr.w2 >= 0;
                                if (zp < zmin && inside && (K.double_side || front)) {
                                    zmin = zp;
                                    fid = f;
                                    const float* tp = tex_img + ((size_t)f * K.T2 + tix) * 3;
                                    c0 = __ldg(tp); c1 = __ldg(tp + 1); c2 = __ldg(tp + 2);
                                }
                            } else {
                                // normalised depth (kernel.cu:418); the backward needs THESE bits (DESIGN.md §2)
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
                                        const float* tp = tex_img + ((size_t)f * K.T2 + tix) * 3;
                                        c0 = ed * c0 + a * __ldg(tp);
                                        c1 = ed * c1 + a * __ldg(tp + 1);
                                        c2 = ed * c2 + a * __ldg(tp + 2);
                                    }
                                }
                            }
                        }
                    }
                }
                if (save) {  // uniform: one 32-slot block per (face, pixel block met); survivors compacted to its front
                    const uint32_t m = __ballot_sync(0xffffffffu, emit);
                    const uint32_t blk = segbase + s_boff[jl] + (uint32_t)__popc(s_meet[jl] & qlow);
                    if (emit) {
                        float4* dst = pb.recs + (size_t)blk * BLK_F4 + __popc(m & lt);
                        // closest-point barycentrics as the reference forms them: t_k + w_k (kernel.cu:638-641)
                        const float u0 = fr.t0 + fr.w0, u1 = fr.t1 + fr.w1, u2 = fr.t2 + fr.w2;
                        // meta: pixel in bits 0-9, texel in bits 10-30 (T2 <= 2^21, make_pairbuf), front in bit 31
                        const uint32_t meta = (uint32_t)(lrow * T4 + lcol) | (tix << 10) | (front << 31);
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
            if (RGB == 1 && p2f_acc != nullptr) {  // one global RED per (pixel block, face, component)
                if (own_w != 0.f) {  // lane r owns the r-th staged face of the group
                    const int e = __fns(m_cur, 0, lane + 1);
                    float* dst = p2f_acc + ((size_t)b * F + s_list[base + e]) * 4;
                    red_add_global(dst + 0, own_x);
                    red_add_global(dst + 1, own_y);
                    red_add_global(dst + 2, own_w);
                }
            }
            __syncwarp();  // every lane is done with stage g & 1 before issue(g + 2) overwrites it
            m_cur = m_next;
        }
        cp_async_wait<0>();  // (the trailing empty group) -- the stages are reused by the next block / window
        __syncwarp();
        st.acc_a = acc_a; st.ssum = ssum; st.smax = smax; st.c0 = c0; st.c1 = c1; st.c2 = c2; st.zmin = zmin; st.fid = fid;
    };

    // ---- finalise (kernel.cu:443-475), fused 2x2 pool, stores of one 8x4 block ---------------------------------
    auto store_block = [&](int q, const PixelState& st) {
        const int lcol = (q & 3) * 8 + (lane & 7), lrow = (q >> 2) * 4 + (lane >> 3);
        const int px = tx0 + lcol, py = ty0 + lrow;
        const bool live = px < S && py < S;
        const float alpha = (float)(1. - (double)st.acc_a);  // kernel.cu:449-451
        float o0, o1, o2, g0, g1;
        if (RGB == 0) {
            o0 = st.c0; o1 = st.c1; o2 = st.c2;
            g0 = st.zmin; g1 = (float)st.fid;
        } else {
            o0 = st.c0 == 0.f ? st.c0 : st.c0 / st.ssum;
            o1 = st.c1 == 0.f ? st.c1 : st.c1 / st.ssum;
            o2 = st.c2 == 0.f ? st.c2 : st.c2 / st.ssum;
            g0 = st.ssum; g1 = st.smax;
        }
        float v[4] = {o0, o1, o2, alpha};
        if (K.aa) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float a01 = __shfl_xor_sync(0xffffffffu, v[k], 1);
                const float a10 = __shfl_xor_sync(0xffffffffu, v[k], 8);
                const float a11 = __shfl_xor_sync(0xffffffffu, v[k], 9);
                v[k] = (((v[k] + a01) + a10) + a11) * 0.25f;  // meaningful on the (even x, even y) lane
            }
        }
        if (live) {  // a warp store covers 4 rows x 32 bytes (full sectors)
            const size_t p = (size_t)py * S + px;
            aggrs[((size_t)b * 2 + 0) * np + p] = g0;
            aggrs[((size_t)b * 2 + 1) * np + p] = g1;
            if (colors_hi != nullptr) {
                colors_hi[((size_t)b * 4 + 0) * np + p] = o0;
                colors_hi[((size_t)b * 4 + 1) * np + p] = o1;
                colors_hi[((size_t)b * 4 + 2) * np + p] = o2;
                colors_hi[((size_t)b * 4 + 3) * np + p] = alpha;
            }
            if (K.aa) {
                if ((lane & 1) == 0 && (lane & 8) == 0) {
                    const int IS = K.IS;
                    const size_t qq = (size_t)(py >> 1) * IS + (px >> 1);
                    const size_t nq = (size_t)IS * IS;
#pragma unroll
                    for (int k = 0; k < 4; ++k) images[((size_t)b * 4 + k) * nq + qq] = v[k];
                }
            } else if (images != colors_hi) {
                images[((size_t)b * 4 + 0) * np + p] = o0;
                images[((size_t)b * 4 + 1) * np + p] = o1;
                images[((size_t)b * 4 + 2) * np + p] = o2;
                images[((size_t)b * 4 + 3) * np + p] = alpha;
            }
        }
    };
    // the tile's four 16x16 tiles go to the recompute backward
    auto mark_unsaved = [&]() {
        const int t16x = (S + TILE - 1) / TILE, t16y = t16x;
        for (int dy = 0; dy < 2; ++dy)
            for (int dx = 0; dx < 2; ++dx) {
                const int bx = blockIdx.x * 2 + dx, by = blockIdx.y * 2 + dy;
                if (bx < t16x && by < t16y) pb.ulist[atomicAdd(pb.ctrl + 1, 1u)] = (int32_t)(((size_t)b * t16y + by) * t16x + bx);
            }
    };

    if (slow) {
        // ---- SLOW path (coarse list longer than the shared tile list): windows of LC entries, static block assignment
        // (pass p: warp w owns block p * 8 + w, its pixel state lives in registers across the windows), no record saving
        if (tid == 0 && pb.cap > 0) { pb.tile_head[tile_id] = TILE_UNSAVED; mark_unsaved(); }
        for (int pass = 0; pass < 4; ++pass) {
            const int q = pass * NWARP + warp;
            PixelState st;
            init_state(st);
            for (int w0 = 0; w0 < nc; w0 += LC) {
                const int n = build_list(w0, min(LC, nc - w0));
                run_groups(q, n, false, 0u, st);
                __syncthreads();  // every warp is done with this window's list before it is rebuilt
            }
            store_block(q, st);
        }
        return;
    }

    const int n = build_list(0, nc);
    // ---- block offsets: exclusive prefix of popc(meet) over the list ------------------------------------------
    {
        uint32_t running = 0;
        for (int r0 = 0; r0 < n; r0 += CTA) {
            const int i = r0 + tid;
            const uint32_t v = i < n ? (uint32_t)__popc(s_meet[i]) : 0u;
            uint32_t incl = v;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += o;
            }
            if (lane == 31) s_warp_blk[warp] = incl;
            __syncthreads();
            uint32_t base = running, total = 0;
#pragma unroll
            for (int w = 0; w < NWARP; ++w) {
                const uint32_t c = s_warp_blk[w];
                base += (w < warp) ? c : 0u;
                total += c;
            }
            if (i < n) s_boff[i] = base + incl - v;
            running += total;
            __syncthreads();  // s_warp_blk reusable
        }
        if (tid == 0) s_boff[n] = running;
    }
    __syncthreads();
    const uint32_t NBw = s_boff[n];

    // ---- reserve the tile's blocks in the pair buffer (one segment per tile) -----------------------------------
    if (tid == 0) {
        int32_t head = TILE_EMPTY;
        const int save_prev = *reinterpret_cast<volatile int*>(&s_save);  // read by thread 0 only (volatile: not hoisted)
        if (save_prev && NBw > 0) {
            const uint32_t base = atomicAdd(pb.ctrl, NBw + 2u);
            if ((uint64_t)base + NBw + 2u > (uint64_t)pb.cap) {
                s_save = 0;  // does not fit: the tile falls back to the recompute backward
                head = TILE_UNSAVED;
                mark_unsaved();
            } else {
                pb.blk_hdr[base] = NBw;
                pb.blk_hdr[base + 1] = SEG_NONE;
                head = (int32_t)base;
                s_segbase = base + 2u;
            }
        }
        if (pb.cap > 0) pb.tile_head[tile_id] = head;
    }
    __syncthreads();  // s_save / s_segbase visible
    const bool save = s_save != 0 && NBw > 0;
    const uint32_t segbase = s_segbase;

    // ---- warps grab 8x4 pixel blocks until the tile is done: no CTA barrier below this line ---------------------
    for (;;) {
        int q = 0;
        if (lane == 0) q = atomicAdd(&s_next, 1);
        q = __shfl_sync(0xffffffffu, q, 0);
        if (q >= (T4 / 8) * (T4 / 4)) break;
        PixelState st;
        init_state(st);
        run_groups(q, n, save, segbase, st);
        store_block(q, st);
    }
}

}  // namespace umr
