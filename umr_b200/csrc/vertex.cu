// vertex.cu -- fused vertex pipeline around the rasteriser (SURVEY.md §8f-1).
//
// One kernel replaces ~70 tiny torch launches per render of the reference host path:
//   nnutils/geom_utils.py:74-91,119-165  orthographic_proj_withz (quaternion rotate via two Hamilton
//                                        products, scale, translate, z offset)
//   nnutils/smr.py:36                    y *= -1
//   SoftRas/functional/look_at.py:48-60  v - eye, rotation = identity for an eye on the z axis
//   SoftRas/functional/orthogonal.py     x, y *= viewing_scale
//   SoftRas/functional/face_vertices.py  gather vertices -> [B,F,3,3]
//   SoftRas/lighting.py:50-57 + mesh.py:112-118 + functional/{ambient,directional}_lighting.py
//                                        per-face light = Ia*ca + Id*cd*relu(n . d)   (optional)
// and its backward (scatter of the per-face-corner gradients to vertices, projection backward to
// vertices and the 7-dof camera) replaces the matching autograd chain.
//
// Compiled with -fmad=false and written in the reference's operation order, so the forward is
// bit-identical to the torch-op chain (every torch elementwise op rounds to fp32).
//
// CorrLossChamfer's kernels are templated on the scalar type; the float64 entry points at the end of this file
// (DESIGN.md §10) run their double instantiations with the deterministic float32 launchers.
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "common.cuh"
#include "umr_b200.h"

namespace umr {

template <typename T>
struct Cam {
    T s, tx, ty, q0, q1, q2, q3;
};

template <typename T>
__device__ __forceinline__ Cam<T> load_cam(const T* __restrict__ cams, int b) {
    const T* c = cams + (size_t)b * 7;
    Cam<T> k;
    k.s = __ldg(c); k.tx = __ldg(c + 1); k.ty = __ldg(c + 2);
    k.q0 = __ldg(c + 3); k.q1 = __ldg(c + 4); k.q2 = __ldg(c + 5); k.q3 = __ldg(c + 6);
    return k;
}

// quat_rotate (geom_utils.py:147-165): r = q (x) (0, X) (x) conj(q), products written out in the
// reference's order (hamilton_product, :119-144).
template <typename T>
__device__ __forceinline__ void quat_rotate(const Cam<T>& k, T x, T y, T z, T& r1, T& r2, T& r3) {
    const T b0 = k.q0, b1 = -k.q1, b2 = -k.q2, b3 = -k.q3;  // conjugate
    const T a0 = x * T(0);                                   // X[:, :, [0]] * 0
    // t = (0, X) (x) conj(q)
    const T t0 = a0 * b0 - x * b1 - y * b2 - z * b3;
    const T t1 = a0 * b1 + x * b0 + y * b3 - z * b2;
    const T t2 = a0 * b2 - x * b3 + y * b0 + z * b1;
    const T t3 = a0 * b3 + x * b2 - y * b1 + z * b0;
    // r = q (x) t
    r1 = k.q0 * t1 + k.q1 * t0 + k.q2 * t3 - k.q3 * t2;
    r2 = k.q0 * t2 - k.q1 * t3 + k.q2 * t0 + k.q3 * t1;
    r3 = k.q0 * t3 + k.q1 * t2 - k.q2 * t1 + k.q3 * t0;
}

struct ProjCfg {
    float offset_z;   // smr.py:66  (5.0)
    float eye_z;      // smr.py:60  eye = (0, 0, eye_z), eye_z = -2.732
    float view_scale; // orthogonal scale (1.0)
    int flip_y;       // smr.py:36
};

// raster-space position of one vertex; also returns the pre-look_at position (used for normals,
// mesh.py:112-118 takes them before the transform)
__device__ __forceinline__ void project(const Cam<float>& k, const ProjCfg& c, float x, float y, float z, float* out,
                                        float* pre) {
    float r1, r2, r3;
    quat_rotate(k, x, y, z, r1, r2, r3);
    float px = k.s * r1 + k.tx;
    float py = k.s * r2 + k.ty;
    float pz = k.s * r3 + c.offset_z;
    if (c.flip_y) py = py * -1.f;
    pre[0] = px; pre[1] = py; pre[2] = pz;
    // look_at with eye on the z axis: R = I, v - eye; then orthogonal(scale)
    out[0] = (px - 0.f) * c.view_scale;
    out[1] = (py - 0.f) * c.view_scale;
    out[2] = pz - c.eye_z;
}

struct LightCfg {
    int enabled;
    float ia, id;            // intensities
    float ca[3], cd[3];      // colours
    float dir[3];            // light direction
};

__global__ void __launch_bounds__(256) k_project_faces(const float* __restrict__ verts, const float* __restrict__ cams,
                                                       const int32_t* __restrict__ faces, float* __restrict__ fv,
                                                       float* __restrict__ light, int V, int F, int H, int64_t faces_bstride,
                                                       ProjCfg pc, LightCfg lc) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (f >= F) return;
    const auto k = load_cam(cams, b);
    const int vb = b / H;  // vertex / face batch item: H consecutive renders (camera hypotheses) share one mesh
    const int32_t* fi = faces + (size_t)vb * faces_bstride + (size_t)f * 3;
    float out[9], pre[9];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int v = __ldg(fi + c);
        if ((unsigned)v >= (unsigned)V) {
            // face index outside [0, V): never read out of bounds.  The face becomes NaN (the reference's torch
            // indexing raises a device-side assert here, face_vertices.py:22); NaN surfaces in every loss downstream.
            const float nan = __int_as_float(0x7fc00000);
            out[3 * c] = out[3 * c + 1] = out[3 * c + 2] = nan;
            pre[3 * c] = pre[3 * c + 1] = pre[3 * c + 2] = nan;
            continue;
        }
        const float* p = verts + ((size_t)vb * V + v) * 3;
        project(k, pc, __ldg(p), __ldg(p + 1), __ldg(p + 2), out + 3 * c, pre + 3 * c);
    }
    float* o = fv + ((size_t)b * F + f) * 9;
#pragma unroll
    for (int i = 0; i < 9; ++i) o[i] = out[i];
    if (lc.enabled && light != nullptr) {
        // mesh.py:114-116: v10 = v0 - v1, v12 = v2 - v1, n = normalize(cross(v12, v10), eps=1e-6)
        const float ax = pre[6] - pre[3], ay = pre[7] - pre[4], az = pre[8] - pre[5];  // v12
        const float bx = pre[0] - pre[3], by = pre[1] - pre[4], bz = pre[2] - pre[5];  // v10
        const float nx = ay * bz - az * by, ny = az * bx - ax * bz, nz = ax * by - ay * bx;
        const float nrm = fmaxf(sqrtf(nx * nx + ny * ny + nz * nz), 1e-6f);
        const float cosv = fmaxf((nx / nrm) * lc.dir[0] + (ny / nrm) * lc.dir[1] + (nz / nrm) * lc.dir[2], 0.f);
        float* l = light + ((size_t)b * F + f) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) l[c] = lc.ia * lc.ca[c] + lc.id * (lc.cd[c] * cosv);
    }
}

// backward A: per face -> add d(light)/d(corners) to the corner gradients, scatter to gproj[B,V,3]
// DET: `gproj` is the per-(render, face, corner) term array [B,F,3,3] (plain stores, zeros for a face with an index
// outside [0, V)), summed per vertex by k_vertex_gather.
template <bool DET>
__global__ void __launch_bounds__(256) k_scatter_face_grads(const float* __restrict__ verts, const float* __restrict__ cams,
                                                            const int32_t* __restrict__ faces, const float* __restrict__ gfv,
                                                            const float* __restrict__ glight, float* __restrict__ gproj,
                                                            int V, int F, int H, int64_t faces_bstride, ProjCfg pc, LightCfg lc) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (f >= F) return;
    const int vb = b / H;  // vertex / face batch item: H consecutive renders (camera hypotheses) share one mesh
    const int32_t* fi = faces + (size_t)vb * faces_bstride + (size_t)f * 3;
    int vid[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) vid[c] = __ldg(fi + c);
    // face with an index outside [0, V) (forward wrote NaN for it): never write out of bounds
    if ((unsigned)vid[0] >= (unsigned)V || (unsigned)vid[1] >= (unsigned)V || (unsigned)vid[2] >= (unsigned)V) {
        if (DET) {
            float* q = gproj + ((size_t)b * F + f) * 9;
#pragma unroll
            for (int i = 0; i < 9; ++i) q[i] = 0.f;
        }
        return;
    }
    float g[9];
    const float* gi = gfv + ((size_t)b * F + f) * 9;
    // d/d(pre) of out: x,y scaled by view_scale, z unchanged
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        g[3 * c + 0] = __ldg(gi + 3 * c + 0) * pc.view_scale;
        g[3 * c + 1] = __ldg(gi + 3 * c + 1) * pc.view_scale;
        g[3 * c + 2] = __ldg(gi + 3 * c + 2);
    }
    if (lc.enabled && glight != nullptr) {
        const float* gl = glight + ((size_t)b * F + f) * 3;
        const float gc = lc.id * (lc.cd[0] * __ldg(gl) + lc.cd[1] * __ldg(gl + 1) + lc.cd[2] * __ldg(gl + 2));
        if (gc != 0.f) {
            const auto k = load_cam(cams, b);
            float out[9], pre[9];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float* p = verts + ((size_t)vb * V + vid[c]) * 3;
                project(k, pc, __ldg(p), __ldg(p + 1), __ldg(p + 2), out + 3 * c, pre + 3 * c);
            }
            const float ax = pre[6] - pre[3], ay = pre[7] - pre[4], az = pre[8] - pre[5];
            const float bx = pre[0] - pre[3], by = pre[1] - pre[4], bz = pre[2] - pre[5];
            const float nx = ay * bz - az * by, ny = az * bx - ax * bz, nz = ax * by - ay * bx;
            const float len = sqrtf(nx * nx + ny * ny + nz * nz);
            const float nrm = fmaxf(len, 1e-6f);
            const float hx = nx / nrm, hy = ny / nrm, hz = nz / nrm;
            const float cosv = hx * lc.dir[0] + hy * lc.dir[1] + hz * lc.dir[2];
            if (cosv > 0.f) {
                // dL/dn_hat = gc * dir ; through n_hat = n / max(|n|, eps)
                float Gx = gc * lc.dir[0], Gy = gc * lc.dir[1], Gz = gc * lc.dir[2];
                if (len > 1e-6f) {
                    const float d = hx * Gx + hy * Gy + hz * Gz;
                    Gx = (Gx - hx * d) / nrm; Gy = (Gy - hy * d) / nrm; Gz = (Gz - hz * d) / nrm;
                } else {
                    Gx /= nrm; Gy /= nrm; Gz /= nrm;
                }
                // n = a x b  (a = v12, b = v10):  dL/da = b x G,  dL/db = G x a
                const float dax = by * Gz - bz * Gy, day = bz * Gx - bx * Gz, daz = bx * Gy - by * Gx;
                const float dbx = Gy * az - Gz * ay, dby = Gz * ax - Gx * az, dbz = Gx * ay - Gy * ax;
                // a = v2 - v1, b = v0 - v1
                g[6] += dax; g[7] += day; g[8] += daz;
                g[0] += dbx; g[1] += dby; g[2] += dbz;
                g[3] -= dax + dbx; g[4] -= day + dby; g[5] -= daz + dbz;
            }
        }
    }
    if (DET) {
        float* q = gproj + ((size_t)b * F + f) * 9;
#pragma unroll
        for (int i = 0; i < 9; ++i) q[i] = g[i];
    } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float* q = gproj + ((size_t)b * V + vid[c]) * 3;
            atomicAdd(q + 0, g[3 * c + 0]);
            atomicAdd(q + 1, g[3 * c + 1]);
            atomicAdd(q + 2, g[3 * c + 2]);
        }
    }
}

// backward B: per vertex -> grad_vertices (direct store) and grad_cams (block reduce + 7 atomics)
// DET: `gverts` is indexed by render (the per-render term array [B,V,3] when H > 1, summed by k_hypothesis_sum), and
// `gcams` is the slot array [B][gridDim.x][7]: each CTA stores its partial, k_cam_finalize sums the slots.
template <bool DET>
__global__ void __launch_bounds__(256) k_project_backward(const float* __restrict__ verts, const float* __restrict__ cams,
                                                          const float* __restrict__ gproj, float* __restrict__ gverts,
                                                          float* __restrict__ gcams, int V, int H, ProjCfg pc) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    const int vb = b / H;  // H consecutive renders (camera hypotheses) share one vertex set
    float gc[7] = {0, 0, 0, 0, 0, 0, 0};
    if (v < V) {
        const auto k = load_cam(cams, b);
        const float* p = verts + ((size_t)vb * V + v) * 3;
        const float X = __ldg(p), Y = __ldg(p + 1), Z = __ldg(p + 2);
        const float* gp = gproj + ((size_t)b * V + v) * 3;
        float gx = __ldg(gp), gy = __ldg(gp + 1);
        const float gz = __ldg(gp + 2);
        if (pc.flip_y) gy = -gy;
        float r1, r2, r3;
        quat_rotate(k, X, Y, Z, r1, r2, r3);
        gc[0] = gx * r1 + gy * r2 + gz * r3;  // d/ds
        gc[1] = gx;                            // d/dtx
        gc[2] = gy;                            // d/dty
        // G = dL/dr
        const float Gx = k.s * gx, Gy = k.s * gy, Gz = k.s * gz;
        const float vx = k.q1, vy = k.q2, vz = k.q3, q0 = k.q0;
        const float vv = vx * vx + vy * vy + vz * vz;
        const float vG = vx * Gx + vy * Gy + vz * Gz;
        const float vX = vx * X + vy * Y + vz * Z;
        const float XG = X * Gx + Y * Gy + Z * Gz;
        // r = (q0^2 - v.v) X + 2 (v.X) v + 2 q0 (v x X)
        // dL/dX = (q0^2 - v.v) G + 2 (v.G) v - 2 q0 (v x G)
        const float c0 = q0 * q0 - vv;
        const float cx = vy * Gz - vz * Gy, cy = vz * Gx - vx * Gz, cz = vx * Gy - vy * Gx;  // v x G
        if (gverts != nullptr) {
            float* o = gverts + ((size_t)(DET ? b : vb) * V + v) * 3;
            const float o0 = c0 * Gx + 2.f * vG * vx - 2.f * q0 * cx;
            const float o1 = c0 * Gy + 2.f * vG * vy - 2.f * q0 * cy;
            const float o2 = c0 * Gz + 2.f * vG * vz - 2.f * q0 * cz;
            if (DET || H == 1) { o[0] = o0; o[1] = o1; o[2] = o2; }
            else { atomicAdd(o, o0); atomicAdd(o + 1, o1); atomicAdd(o + 2, o2); }  // sum over the hypotheses (zero-filled by the host)
        }
        // dL/dq0 = G . (2 q0 X + 2 (v x X))
        const float wx = vy * Z - vz * Y, wy = vz * X - vx * Z, wz = vx * Y - vy * X;  // v x X
        gc[3] = 2.f * (q0 * XG + (Gx * wx + Gy * wy + Gz * wz));
        // dL/dv = -2 (X.G) v + 2 (v.G) X + 2 (v.X) G + 2 q0 (X x G)
        const float ex = Y * Gz - Z * Gy, ey = Z * Gx - X * Gz, ez = X * Gy - Y * Gx;  // X x G
        gc[4] = 2.f * (-XG * vx + vG * X + vX * Gx + q0 * ex);
        gc[5] = 2.f * (-XG * vy + vG * Y + vX * Gy + q0 * ey);
        gc[6] = 2.f * (-XG * vz + vG * Z + vX * Gz + q0 * ez);
    }
    if (gcams == nullptr) return;
    __shared__ float s[8][7];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < 7; ++i) {
        const float r = warp_sum(gc[i]);
        if (lane == 0) s[warp][i] = r;
    }
    __syncthreads();
    if (threadIdx.x < 7) {
        float r = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) r += s[w][threadIdx.x];
        if (DET) gcams[((size_t)b * gridDim.x + blockIdx.x) * 7 + threadIdx.x] = r;
        else atomicAdd(gcams + (size_t)b * 7 + threadIdx.x, r);
    }
}

// Deterministic backward, per-vertex sums of k_scatter_face_grads<true>'s corner terms: gproj[b][v] = the terms of v's
// incidence entries in render b, added in ascending table order.  The table lists positions face * 3 + corner of the
// flattened faces: rows v over V vertices when the faces are shared, rows vb * V + v over the Bv meshes otherwise (their
// positions then lie in mesh vb's [vb * F * 3, (vb + 1) * F * 3)).
__global__ void __launch_bounds__(256) k_vertex_gather(const float* __restrict__ terms, const int32_t* __restrict__ rowptr,
                                                       const int32_t* __restrict__ incidence, float* __restrict__ gproj,
                                                       int V, int F, int H, int batched) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (v >= V) return;
    const int vb = b / H;
    const size_t row = batched ? (size_t)vb * V + v : (size_t)v;
    const int64_t base = batched ? (int64_t)vb * F * 3 : 0;
    const float* tb = terms + (size_t)b * F * 9;
    float g0 = 0.f, g1 = 0.f, g2 = 0.f;
    const int k1 = __ldg(rowptr + row + 1);
    for (int k = __ldg(rowptr + row); k < k1; ++k) {
        const float* t = tb + (size_t)(__ldg(incidence + k) - base) * 3;
        g0 += t[0]; g1 += t[1]; g2 += t[2];
    }
    float* o = gproj + ((size_t)b * V + v) * 3;
    o[0] = g0; o[1] = g1; o[2] = g2;
}

// gverts[vb][v] = the per-render terms [B,V,3] of the H hypotheses of mesh vb, added in ascending h
__global__ void __launch_bounds__(256) k_hypothesis_sum(const float* __restrict__ terms, float* __restrict__ gverts, int V,
                                                        int H) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    const int vb = blockIdx.y;
    if (v >= V) return;
    float g0 = 0.f, g1 = 0.f, g2 = 0.f;
    for (int h = 0; h < H; ++h) {
        const float* t = terms + ((size_t)(vb * H + h) * V + v) * 3;
        g0 += t[0]; g1 += t[1]; g2 += t[2];
    }
    float* o = gverts + ((size_t)vb * V + v) * 3;
    o[0] = g0; o[1] = g1; o[2] = g2;
}

// gcams[b][i] = render b's CTA slots [nslot][7] added in ascending CTA order
__global__ void k_cam_finalize(const float* __restrict__ slots, float* __restrict__ gcams, int B, int nslot) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= B * 7) return;
    const int b = t / 7, i = t - b * 7;
    const float* s = slots + (size_t)b * nslot * 7 + i;
    float r = 0.f;
    for (int w = 0; w < nslot; ++w) r += s[(size_t)w * 7];
    gcams[t] = r;
}


// ---------------------------------------------------------------------------------------------
// CorrLossChamfer (nnutils/loss_utils.py:194-248) in one kernel per direction.  The reference projects the selected part
// vertices with ~60 tiny torch kernels (quaternion products through stack / cat), runs distChamfer once per part (bmm +
// min), concatenates and averages; its backward is ~150 more launches including a radix sort for the index_put.  Here one
// CTA per render: project the NS selected vertices (same arithmetic as k_project_faces: quat_rotate, scale, translate),
// nearest target of the vertex's own part in the defined fp32 order of k_chamfer_nn (losses.cu), weighted mean.
// ---------------------------------------------------------------------------------------------
template <typename T>
struct CorrCfg {
    const T* tgt[4];   // [B, m[g], 2] target points of part g
    int m[4];          // target counts
    int end[4];        // exclusive end of part g in the concatenated vertex selection (loss_utils.py:211-216 `nums`)
    T w[4];            // per-part weights (loss_utils.py:210: [1, 1, 0, 0])
};

template <typename T>
__device__ __forceinline__ int corr_part(const CorrCfg<T>& c, int j) { return j < c.end[0] ? 0 : (j < c.end[1] ? 1 : (j < c.end[2] ? 2 : 3)); }

template <typename T>
__global__ void __launch_bounds__(256) k_corr_fwd(const T* __restrict__ verts, int64_t verts_bstride, const T* __restrict__ cams,
                                                  const int32_t* __restrict__ sel, CorrCfg<T> c, T* __restrict__ vert2d,
                                                  int32_t* __restrict__ nn, T* __restrict__ loss, int NS) {
    __shared__ T s_part[8];
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const auto k = load_cam(cams, b);
    T acc = 0;  // meaningful in lane 0
    for (int j = warp; j < NS; j += 8) {
        const T* p = verts + (size_t)b * verts_bstride + (size_t)__ldg(sel + j) * 3;
        T r1, r2, r3;
        quat_rotate(k, __ldg(p), __ldg(p + 1), __ldg(p + 2), r1, r2, r3);
        const T qx = k.s * r1 + k.tx, qy = k.s * r2 + k.ty;   // orthographic_proj_withz(...)[:, :, :2] (geom_utils.py:74-91)
        const int g = corr_part(c, j);
        const T* tb = c.tgt[g] + (size_t)b * c.m[g] * 2;
        const T qq = add_rn(mul_rn(qx, qx), mul_rn(qy, qy));
        T best = (T)INFINITY;
        int bi = 0x7fffffff;
        for (int t = lane; t < c.m[g]; t += 32) {
            const T kx = __ldg(tb + 2 * t), ky = __ldg(tb + 2 * t + 1);
            const T kk = add_rn(mul_rn(kx, kx), mul_rn(ky, ky));
            const T zz = add_rn(mul_rn(qx, kx), mul_rn(qy, ky));
            const T P = sub_rn(add_rn(qq, kk), mul_rn(T(2), zz));  // chamfer_python.py:63, as k_chamfer_nn
            if (P < best) { best = P; bi = t; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const T ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
        if (lane == 0) {
            vert2d[((size_t)b * NS + j) * 2 + 0] = qx;
            vert2d[((size_t)b * NS + j) * 2 + 1] = qy;
            nn[(size_t)b * NS + j] = bi;
            acc += best * c.w[g];   // d_to_target * weight (loss_utils.py:236)
        }
    }
    if (lane == 0) s_part[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        T t = 0;
        for (int w = 0; w < 8; ++w) t += s_part[w];   // fixed order: deterministic
        loss[b] = t / (T)NS;                          // torch.mean(torch.cat(terms, 1), 1) (:239)
    }
}

// per-vertex backward of r = quat_rotate(q, X); p = s r + t given G = dL/dp with dL/dpz = 0: adds to gc[7] (scale, tx, ty,
// q0..q3) and returns dL/dX (the derivation of k_project_backward).  float32 carries the zero z gradient through (s * 0 and
// a 0 * r3 term), float64 uses an exact 0 with no r3 term; they differ only for a non-finite scale or r3 and in the sign
// of a zero, and each precision keeps its bits.
template <typename T>
__device__ __forceinline__ void project_point_backward(const Cam<T>& k, T X, T Y, T Z, T gx, T gy, T* gc, T& o0, T& o1, T& o2) {
    constexpr bool F32 = std::is_same<T, float>::value;
    T r1, r2, r3;
    quat_rotate(k, X, Y, Z, r1, r2, r3);
    gc[0] += F32 ? gx * r1 + gy * r2 + T(0) * r3 : gx * r1 + gy * r2;
    gc[1] += gx;
    gc[2] += gy;
    const T Gx = k.s * gx, Gy = k.s * gy, Gz = F32 ? k.s * T(0) : T(0);
    const T vx = k.q1, vy = k.q2, vz = k.q3, q0 = k.q0;
    const T vv = vx * vx + vy * vy + vz * vz;
    const T vG = vx * Gx + vy * Gy + vz * Gz;
    const T vX = vx * X + vy * Y + vz * Z;
    const T XG = X * Gx + Y * Gy + Z * Gz;
    const T c0 = q0 * q0 - vv;
    const T cx = vy * Gz - vz * Gy, cy = vz * Gx - vx * Gz, cz = vx * Gy - vy * Gx;  // v x G
    o0 = c0 * Gx + T(2) * vG * vx - T(2) * q0 * cx;
    o1 = c0 * Gy + T(2) * vG * vy - T(2) * q0 * cy;
    o2 = c0 * Gz + T(2) * vG * vz - T(2) * q0 * cz;
    const T wx = vy * Z - vz * Y, wy = vz * X - vx * Z, wz = vx * Y - vy * X;  // v x X
    gc[3] += T(2) * (q0 * XG + (Gx * wx + Gy * wy + Gz * wz));
    const T ex = Y * Gz - Z * Gy, ey = Z * Gx - X * Gz, ez = X * Gy - Y * Gx;  // X x G
    gc[4] += T(2) * (-XG * vx + vG * X + vX * Gx + q0 * ex);
    gc[5] += T(2) * (-XG * vy + vG * Y + vX * Gy + q0 * ey);
    gc[6] += T(2) * (-XG * vz + vG * Z + vX * Gz + q0 * ez);
}

// backward: grad_loss [B] (per render), optional grad_vert2d [B,NS,2] -> grad_verts [B,V,3] (zero-filled by the host,
// atomics: a vertex may sit in several parts) and grad_cams [B,7].  Targets are constants (the reference's are data).
// DET: `gverts` is the per-(render, j) term array [B,NS,3] (plain stores), summed per vertex by k_gather3.  Float64 runs
// only the DET form.
template <typename T, bool DET>
__global__ void __launch_bounds__(256) k_corr_bwd(const T* __restrict__ verts, int64_t verts_bstride, const T* __restrict__ cams,
                                                  const int32_t* __restrict__ sel, CorrCfg<T> c, const T* __restrict__ vert2d,
                                                  const int32_t* __restrict__ nn, const T* __restrict__ grad_loss,
                                                  const T* __restrict__ grad_vert2d, T* __restrict__ gverts,
                                                  T* __restrict__ gcams, int NS, int V) {
    __shared__ T s[8][7];
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const auto k = load_cam(cams, b);
    const T gl = __ldg(grad_loss + b) / (T)NS;
    T gc[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int j = threadIdx.x; j < NS; j += 256) {
        const int g = corr_part(c, j);
        const int vi = __ldg(sel + j);
        const T* p = verts + (size_t)b * verts_bstride + (size_t)vi * 3;
        const T qx = __ldg(vert2d + ((size_t)b * NS + j) * 2), qy = __ldg(vert2d + ((size_t)b * NS + j) * 2 + 1);
        const T* t = c.tgt[g] + ((size_t)b * c.m[g] + __ldg(nn + (size_t)b * NS + j)) * 2;
        const T gd = gl * c.w[g];
        // d/dq of (|q|^2 + |t|^2 - 2 q.t) = 2 q - 2 t (chamfer_python.py:63; the argmin is piecewise constant)
        T gx = gd * (T(2) * qx - T(2) * __ldg(t)), gy = gd * (T(2) * qy - T(2) * __ldg(t + 1));
        if (grad_vert2d != nullptr) {
            gx += __ldg(grad_vert2d + ((size_t)b * NS + j) * 2);
            gy += __ldg(grad_vert2d + ((size_t)b * NS + j) * 2 + 1);
        }
        T o0, o1, o2;
        project_point_backward(k, __ldg(p), __ldg(p + 1), __ldg(p + 2), gx, gy, gc, o0, o1, o2);
        if (gverts != nullptr) {
            if (DET) {
                T* o = gverts + ((size_t)b * NS + j) * 3;
                o[0] = o0; o[1] = o1; o[2] = o2;
            } else {
                T* o = gverts + ((size_t)b * V + vi) * 3;
                atomicAdd(o, o0); atomicAdd(o + 1, o1); atomicAdd(o + 2, o2);
            }
        }
    }
    if (gcams == nullptr) return;
#pragma unroll
    for (int i = 0; i < 7; ++i) {
        const T r = warp_sum(gc[i]);
        if (lane == 0) s[warp][i] = r;
    }
    __syncthreads();
    if (threadIdx.x < 7) {
        T r = 0;
        for (int w = 0; w < 8; ++w) r += s[w][threadIdx.x];
        gcams[(size_t)b * 7 + threadIdx.x] = r;   // one CTA per render: plain store
    }
}

}  // namespace umr

using namespace umr;

static ProjCfg make_pc(const UmrProjectParams* p) {
    ProjCfg c;
    c.offset_z = p->offset_z; c.eye_z = p->eye_z; c.view_scale = p->viewing_scale; c.flip_y = p->flip_y ? 1 : 0;
    return c;
}
static LightCfg make_lc(const UmrProjectParams* p) {
    LightCfg l;
    l.enabled = p->light_enabled ? 1 : 0;
    l.ia = p->light_intensity_ambient; l.id = p->light_intensity_directional;
    for (int i = 0; i < 3; ++i) {
        l.ca[i] = p->light_color_ambient[i]; l.cd[i] = p->light_color_directional[i]; l.dir[i] = p->light_direction[i];
    }
    return l;
}

extern "C" int umr_project_faces_forward(const float* vertices, const float* cams, const int32_t* faces,
                                         float* face_vertices, float* light, const UmrProjectParams* p, void* stream_) {
    if (!vertices || !cams || !faces || !face_vertices || !p) return UMR_ERR_BAD_ARG;
    if (p->batch_size <= 0 || p->num_vertices <= 0 || p->num_faces <= 0) return UMR_ERR_BAD_ARG;
    if (p->batch_size > 65535) return UMR_ERR_TOO_LARGE;
    const int H = p->num_hypotheses > 1 ? p->num_hypotheses : 1;
    if (p->batch_size % H != 0) return UMR_ERR_BAD_ARG;
    launch(k_project_faces, dim3((p->num_faces + 255) / 256, p->batch_size), 256, 0, (cudaStream_t)stream_, vertices, cams,
           faces, face_vertices, light, p->num_vertices, p->num_faces, H, p->faces_batch_stride, make_pc(p), make_lc(p));
    return (int)cudaGetLastError();
}

extern "C" int umr_project_faces_backward(const float* vertices, const float* cams, const int32_t* faces,
                                          const float* grad_face_vertices, const float* grad_light, float* grad_proj,
                                          float* grad_vertices, float* grad_cams, const UmrProjectParams* p,
                                          void* stream_) {
    if (!vertices || !cams || !faces || !grad_face_vertices || !grad_proj || !p) return UMR_ERR_BAD_ARG;
    if (p->batch_size <= 0 || p->num_vertices <= 0 || p->num_faces <= 0) return UMR_ERR_BAD_ARG;
    if (p->batch_size > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const int B = p->batch_size, V = p->num_vertices, F = p->num_faces;
    const int H = p->num_hypotheses > 1 ? p->num_hypotheses : 1;
    if (B % H != 0) return UMR_ERR_BAD_ARG;
    cudaError_t e = cudaMemsetAsync(grad_proj, 0, (size_t)B * V * 3 * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    if (H > 1 && grad_vertices) e = cudaMemsetAsync(grad_vertices, 0, (size_t)(B / H) * V * 3 * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    if (grad_cams) {
        e = cudaMemsetAsync(grad_cams, 0, (size_t)B * 7 * sizeof(float), st);
        if (e != cudaSuccess) return (int)e;
    }
    launch(k_scatter_face_grads<false>, dim3((F + 255) / 256, B), 256, 0, st, vertices, cams, faces, grad_face_vertices,
           grad_light, grad_proj, V, F, H, p->faces_batch_stride, make_pc(p), make_lc(p));
    launch(k_project_backward<false>, dim3((V + 255) / 256, B), 256, 0, st, vertices, cams, grad_proj, grad_vertices, grad_cams,
           V, H, make_pc(p));
    return (int)cudaGetLastError();
}

// Deterministic backward (include/umr_b200.h): corner terms to the workspace, a per-vertex gather over the caller's
// incidence table, the default projection backward with per-render vertex terms and per-CTA camera slots, then the
// ascending sums over the hypotheses and the slots.  Workspace: terms [B,F,9] | vertex terms [B,V,3] | slots
// [B][ceil(V/256)][7], all float.
extern "C" size_t umr_project_faces_workspace_bytes_deterministic(int32_t B, int32_t V, int32_t F) {
    if (B <= 0 || V <= 0 || F <= 0) return 0;
    return (size_t)B * (9 * (size_t)F + 3 * (size_t)V + 7 * (size_t)((V + 255) / 256)) * sizeof(float);
}
extern "C" int umr_project_faces_backward_deterministic(const float* vertices, const float* cams, const int32_t* faces,
                                                        const float* grad_face_vertices, const float* grad_light,
                                                        float* grad_proj, float* grad_vertices, float* grad_cams,
                                                        const UmrProjectParams* p, const int32_t* vert_rowptr,
                                                        const int32_t* vert_incidence, void* workspace, void* stream_) {
    if (!vertices || !cams || !faces || !grad_face_vertices || !grad_proj || !p) return UMR_ERR_BAD_ARG;
    if (!vert_rowptr || !vert_incidence || !workspace) return UMR_ERR_BAD_ARG;
    if (p->batch_size <= 0 || p->num_vertices <= 0 || p->num_faces <= 0) return UMR_ERR_BAD_ARG;
    if (p->batch_size > 65535) return UMR_ERR_TOO_LARGE;
    cudaStream_t st = (cudaStream_t)stream_;
    const int B = p->batch_size, V = p->num_vertices, F = p->num_faces;
    const int H = p->num_hypotheses > 1 ? p->num_hypotheses : 1;
    if (B % H != 0) return UMR_ERR_BAD_ARG;
    const unsigned nslot = (unsigned)((V + 255) / 256);
    float* terms = (float*)workspace;
    float* vterms = terms + (size_t)B * F * 9;
    float* slots = vterms + (size_t)B * V * 3;
    float* gv = (grad_vertices && H > 1) ? vterms : grad_vertices;
    launch(k_scatter_face_grads<true>, dim3((F + 255) / 256, B), 256, 0, st, vertices, cams, faces, grad_face_vertices,
           grad_light, terms, V, F, H, p->faces_batch_stride, make_pc(p), make_lc(p));
    launch(k_vertex_gather, dim3(nslot, B), 256, 0, st, terms, vert_rowptr, vert_incidence, grad_proj, V, F, H,
           p->faces_batch_stride != 0 ? 1 : 0);
    launch(k_project_backward<true>, dim3(nslot, B), 256, 0, st, vertices, cams, grad_proj, gv, grad_cams ? slots : nullptr, V,
           H, make_pc(p));
    if (grad_vertices && H > 1) launch(k_hypothesis_sum, dim3(nslot, B / H), 256, 0, st, vterms, grad_vertices, V, H);
    if (grad_cams) launch(k_cam_finalize, (B * 7 + 255) / 256, 256, 0, st, slots, grad_cams, B, (int)nslot);
    return (int)cudaGetLastError();
}

template <typename T>
static int make_corr_cfg(CorrCfg<T>& c, const T* const* targets, const int32_t* target_counts, const int32_t* part_ends,
                         const T* weights, int NS) {
    int prev = 0;
    for (int g = 0; g < 4; ++g) {
        if (!targets[g] || target_counts[g] <= 0 || part_ends[g] < prev) return UMR_ERR_BAD_ARG;
        c.tgt[g] = targets[g]; c.m[g] = target_counts[g]; c.end[g] = part_ends[g]; c.w[g] = weights[g];
        prev = part_ends[g];
    }
    return prev == NS ? UMR_OK : UMR_ERR_BAD_ARG;
}

// float32 and float64
template <typename T>
static int corr_chamfer_forward(const T* vertices, int64_t vertices_batch_stride, const T* cams, const int32_t* selection,
                                const T* const* targets, const int32_t* target_counts, const int32_t* part_ends,
                                const T* weights, T* vert2d, int32_t* nearest, T* loss, int32_t B, int32_t NS, void* stream_) {
    if (!vertices || !cams || !selection || !targets || !target_counts || !part_ends || !weights || !vert2d || !nearest ||
        !loss || B <= 0 || NS <= 0)
        return UMR_ERR_BAD_ARG;
    CorrCfg<T> c;
    const int rc = make_corr_cfg(c, targets, target_counts, part_ends, weights, NS);
    if (rc) return rc;
    launch(k_corr_fwd<T>, B, 256, 0, (cudaStream_t)stream_, vertices, vertices_batch_stride, cams, selection, c, vert2d,
           nearest, loss, NS);
    return (int)cudaGetLastError();
}

extern "C" int umr_corr_chamfer_forward(const float* vertices, int64_t vertices_batch_stride, const float* cams,
                                        const int32_t* selection, const float* const* targets, const int32_t* target_counts,
                                        const int32_t* part_ends, const float* weights, float* vert2d, int32_t* nearest,
                                        float* loss, int32_t B, int32_t NS, void* stream_) {
    return corr_chamfer_forward(vertices, vertices_batch_stride, cams, selection, targets, target_counts, part_ends, weights,
                                vert2d, nearest, loss, B, NS, stream_);
}

extern "C" int umr_corr_chamfer_backward(const float* vertices, int64_t vertices_batch_stride, const float* cams,
                                         const int32_t* selection, const float* const* targets, const int32_t* target_counts,
                                         const int32_t* part_ends, const float* weights, const float* vert2d,
                                         const int32_t* nearest, const float* grad_loss, const float* grad_vert2d,
                                         float* grad_vertices, float* grad_cams, int32_t B, int32_t NS, int32_t V, void* stream_) {
    if (!vertices || !cams || !selection || !targets || !target_counts || !part_ends || !weights || !vert2d || !nearest ||
        !grad_loss || B <= 0 || NS <= 0 || V <= 0)
        return UMR_ERR_BAD_ARG;
    CorrCfg<float> c;
    const int rc = make_corr_cfg(c, targets, target_counts, part_ends, weights, NS);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream_;
    if (grad_vertices) {
        cudaError_t e = cudaMemsetAsync(grad_vertices, 0, (size_t)B * V * 3 * sizeof(float), st);
        if (e != cudaSuccess) return (int)e;
    }
    launch(k_corr_bwd<float, false>, B, 256, 0, st, vertices, vertices_batch_stride, cams, selection, c, vert2d, nearest,
           grad_loss, grad_vert2d, grad_vertices, grad_cams, NS, V);
    return (int)cudaGetLastError();
}

// Deterministic float32 and float64 backward (include/umr_b200.h): k_corr_bwd<T, true> stores the per-(render, j) vertex
// terms in the workspace, k_gather3 sums them per vertex in ascending j.  grad_cams is the kernel's plain store.
template <typename T>
static size_t corr_chamfer_workspace_bytes(int32_t B, int32_t NS) {
    if (B <= 0 || NS <= 0) return 0;
    return (size_t)B * NS * 3 * sizeof(T);
}
template <typename T>
static int corr_chamfer_backward_gather(const T* vertices, int64_t vertices_batch_stride, const T* cams, const int32_t* selection,
                                        const T* const* targets, const int32_t* target_counts, const int32_t* part_ends,
                                        const T* weights, const T* vert2d, const int32_t* nearest, const T* grad_loss,
                                        const T* grad_vert2d, T* grad_vertices, T* grad_cams, int32_t B, int32_t NS, int32_t V,
                                        const int32_t* vert_rowptr, const int32_t* vert_selection, void* workspace,
                                        void* stream_) {
    if (!vertices || !cams || !selection || !targets || !target_counts || !part_ends || !weights || !vert2d || !nearest ||
        !grad_loss || B <= 0 || NS <= 0 || V <= 0)
        return UMR_ERR_BAD_ARG;
    if (grad_vertices && (!vert_rowptr || !vert_selection || !workspace)) return UMR_ERR_BAD_ARG;
    if (B > 65535) return UMR_ERR_TOO_LARGE;
    CorrCfg<T> c;
    const int rc = make_corr_cfg(c, targets, target_counts, part_ends, weights, NS);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream_;
    T* terms = grad_vertices ? (T*)workspace : nullptr;
    launch(k_corr_bwd<T, true>, B, 256, 0, st, vertices, vertices_batch_stride, cams, selection, c, vert2d, nearest, grad_loss,
           grad_vert2d, terms, grad_cams, NS, V);
    if (grad_vertices)
        launch(k_gather3<T>, dim3((V + 255) / 256, B), 256, 0, st, terms, vert_rowptr, vert_selection, grad_vertices, V,
               (int64_t)NS);
    return (int)cudaGetLastError();
}

extern "C" size_t umr_corr_chamfer_workspace_bytes_deterministic(int32_t B, int32_t NS) {
    return corr_chamfer_workspace_bytes<float>(B, NS);
}
extern "C" int umr_corr_chamfer_backward_deterministic(const float* vertices, int64_t vertices_batch_stride, const float* cams,
                                                       const int32_t* selection, const float* const* targets,
                                                       const int32_t* target_counts, const int32_t* part_ends,
                                                       const float* weights, const float* vert2d, const int32_t* nearest,
                                                       const float* grad_loss, const float* grad_vert2d, float* grad_vertices,
                                                       float* grad_cams, int32_t B, int32_t NS, int32_t V,
                                                       const int32_t* vert_rowptr, const int32_t* vert_selection,
                                                       void* workspace, void* stream_) {
    return corr_chamfer_backward_gather(vertices, vertices_batch_stride, cams, selection, targets, target_counts, part_ends,
                                        weights, vert2d, nearest, grad_loss, grad_vert2d, grad_vertices, grad_cams, B, NS, V,
                                        vert_rowptr, vert_selection, workspace, stream_);
}

// float64 (include/umr_b200.h, "float64 loss kernels")
extern "C" int umr_corr_chamfer_forward_f64(const double* vertices, int64_t vertices_batch_stride, const double* cams,
                                            const int32_t* selection, const double* const* targets,
                                            const int32_t* target_counts, const int32_t* part_ends, const double* weights,
                                            double* vert2d, int32_t* nearest, double* loss, int32_t B, int32_t NS,
                                            void* stream_) {
    return corr_chamfer_forward(vertices, vertices_batch_stride, cams, selection, targets, target_counts, part_ends, weights,
                                vert2d, nearest, loss, B, NS, stream_);
}
extern "C" size_t umr_corr_chamfer_workspace_bytes_f64(int32_t B, int32_t NS) { return corr_chamfer_workspace_bytes<double>(B, NS); }
extern "C" int umr_corr_chamfer_backward_f64(const double* vertices, int64_t vertices_batch_stride, const double* cams,
                                             const int32_t* selection, const double* const* targets,
                                             const int32_t* target_counts, const int32_t* part_ends, const double* weights,
                                             const double* vert2d, const int32_t* nearest, const double* grad_loss,
                                             const double* grad_vert2d, double* grad_vertices, double* grad_cams, int32_t B,
                                             int32_t NS, int32_t V, const int32_t* vert_rowptr, const int32_t* vert_selection,
                                             void* workspace, void* stream_) {
    return corr_chamfer_backward_gather(vertices, vertices_batch_stride, cams, selection, targets, target_counts, part_ends,
                                        weights, vert2d, nearest, grad_loss, grad_vert2d, grad_vertices, grad_cams, B, NS, V,
                                        vert_rowptr, vert_selection, workspace, stream_);
}
