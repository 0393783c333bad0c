"""CPU oracle for SoftRas `functional.voxelization` -- TEST INFRASTRUCTURE ONLY.

voxelization_np restates the reference (functional/voxelization.py:41-58, cuda/voxelization_cuda_kernel.cu:30-190) in
numpy float32 or float64 (the faces' dtype, like AT_DISPATCH_FLOATING_TYPES), one rounding per operation in the
reference's order (numpy never contracts to FMA).  The interior fill is the reference's fixed point computed directly:
the empty voxels 6-connected through empty voxels to an empty boundary voxel (connected-component labelling), and the
result is 1 minus that set.  Cases the reference leaves undefined are defined as in DESIGN.md §8: a NaN / inf depth or
vertex marks nothing.

fill_runs is the word-parallel run fill the kernel uses along the packed axis, at any word width, for an exhaustive
check against a bit-by-bit fill.
"""
import numpy as np
from scipy import ndimage

# (y slot, x slot, z slot) coordinates of voxelize_sub1's three calls: faces permuted [2,1,0], [0,2,1], unpermuted
AXES = ((2, 1, 0), (0, 2, 1), (0, 1, 2))


def fill_up(s, e, bits):
    """Run fill toward the high bits: (e & ~(e + s)) | s, with s ⊆ e, in `bits`-bit words."""
    m = (1 << bits) - 1
    return ((e & ~((e + s) & m)) | s) & m


def _brev(x, bits):
    x = np.asarray(x, np.uint64)
    r = np.zeros_like(x)
    for i in range(bits):
        r |= ((x >> np.uint64(i)) & np.uint64(1)) << np.uint64(bits - 1 - i)
    return r


def fill_runs(s, e, bits):
    """Every bit of e in a run of set bits of e that holds a bit of s (s ⊆ e): fill_up, then the same on the
    bit-reversed words toward the low bits."""
    s = np.asarray(s, np.uint64)
    e = np.asarray(e, np.uint64)
    u = fill_up(s, e, bits)
    return _brev(fill_up(_brev(u, bits), _brev(e, bits), bits), bits)


def _regions(a, b, y1d, x1d, y2d, x2d, det, vs, dt):
    """Column ranges [lo, hi] per face that hold every column the float test can pass: a box widened by 2 + L/4 for faces
    with u * L^2 / |det| <= 2^-16 (wider and stricter than the kernel's, DESIGN.md §8), the whole grid otherwise."""
    u = float(np.finfo(dt).eps) / 2
    with np.errstate(all="ignore"):
        e1 = [np.asarray(v, np.float64) for v in (y1d, x1d)]
        e2 = [np.asarray(v, np.float64) for v in (y2d, x2d)]
        L2 = np.maximum(e1[0] ** 2 + e1[1] ** 2, e2[0] ** 2 + e2[1] ** 2)
        good = (u * L2 <= 2.0 ** -16 * np.abs(np.asarray(det, np.float64))) & (L2 <= 1e30)
        good &= np.isfinite(a).all(1) & np.isfinite(b).all(1)
        m = 2.0 + np.sqrt(np.where(good, L2, 0.0)) / 4
        a64, b64 = a.astype(np.float64), b.astype(np.float64)
        ylo = np.where(good, np.floor(a64.min(1) - m), 0).clip(0, vs - 1)
        yhi = np.where(good, np.ceil(a64.max(1) + m), vs - 1).clip(-1, vs - 1)
        xlo = np.where(good, np.floor(b64.min(1) - m), 0).clip(0, vs - 1)
        xhi = np.where(good, np.ceil(b64.max(1) + m), vs - 1).clip(-1, vs - 1)
        outside = (np.where(good, np.ceil(a64.max(1) + m), 0) < 0) | (np.where(good, np.floor(a64.min(1) - m), 0) > vs - 1)
        outside |= (np.where(good, np.ceil(b64.max(1) + m), 0) < 0) | (np.where(good, np.floor(b64.min(1) - m), 0) > vs - 1)
    yhi = np.where(outside, -1, yhi)
    return ylo.astype(np.int64), yhi.astype(np.int64), xlo.astype(np.int64), xhi.astype(np.int64)


def _surface(f, vs, occ):
    """voxelize_sub1 for the three projections of one batch item's faces f [F,3,3] (already scaled), into occ."""
    dt = f.dtype.type
    for ys, xs, zs in AXES:
        a, b, c = f[:, :, ys], f[:, :, xs], f[:, :, zs]
        with np.errstate(all="ignore"):
            y1d, x1d, z1d = a[:, 1] - a[:, 0], b[:, 1] - b[:, 0], c[:, 1] - c[:, 0]
            y2d, x2d, z2d = a[:, 2] - a[:, 0], b[:, 2] - b[:, 0], c[:, 2] - c[:, 0]
            det = x1d * y2d - x2d * y1d
        ylo, yhi, xlo, xhi = _regions(a, b, y1d, x1d, y2d, x2d, det, vs, f.dtype)
        keep = np.nonzero((det != 0) & (yhi >= ylo) & (xhi >= xlo))[0]
        ny, nx = yhi - ylo + 1, xhi - xlo + 1
        # chunks of faces with similar box sizes, about 2M columns per chunk
        order = keep[np.argsort(ny[keep] * nx[keep], kind="stable")]
        start = 0
        while start < len(order):
            ky, kx = ny[order[start]], nx[order[start]]
            end = start + 1
            while end < len(order):
                ky2, kx2 = max(ky, ny[order[end]]), max(kx, nx[order[end]])
                if (end - start + 1) * ky2 * kx2 > 2_000_000:
                    break
                ky, kx, end = ky2, kx2, end + 1
            sel = order[start:end]
            start = end
            y = ylo[sel, None, None] + np.arange(ky)[None, :, None]
            x = xlo[sel, None, None] + np.arange(kx)[None, None, :]
            valid = (y <= yhi[sel, None, None]) & (x <= xhi[sel, None, None])
            with np.errstate(all="ignore"):
                ypd = y.astype(dt) - a[sel, 0, None, None]
                xpd = x.astype(dt) - b[sel, 0, None, None]
                d = det[sel, None, None]
                t1 = (y2d[sel, None, None] * xpd - x2d[sel, None, None] * ypd) / d
                t2 = ((-y1d[sel, None, None]) * xpd + x1d[sel, None, None] * ypd) / d
                ok = valid & (t1 >= 0) & (t2 >= 0) & ~(1 < t1 + t2)
                zf = np.floor(t1 * z1d[sel, None, None] + t2 * z2d[sel, None, None] + c[sel, 0, None, None])
                ok &= (zf >= 0) & (zf < vs)  # NaN / inf: nothing
            fi, yi, xi = np.nonzero(ok)
            Y, X, Z = y[fi, yi, 0], x[fi, 0, xi], zf[fi, yi, xi].astype(np.int64)
            for dy in (0, 1):
                for dx in (0, 1):
                    m = (Y - dy >= 0) & (X - dx >= 0)
                    idx = [None] * 3
                    idx[ys], idx[xs], idx[zs] = Y[m] - dy, X[m] - dx, Z[m]
                    occ[idx[0], idx[1], idx[2]] = True


def occupancy_np(faces, size, normalize=False):
    """Steps 1-4 of the contract: bool [B,vs,vs,vs], surface and vertex voxels."""
    faces = np.asarray(faces)
    assert faces.dtype in (np.float32, np.float64) and faces.ndim == 4 and faces.shape[2:] == (3, 3)
    dt = faces.dtype.type
    f = faces.copy() if normalize else (faces * dt(size)).astype(faces.dtype)
    B, vs = f.shape[0], int(size)
    occ = np.zeros((B, vs, vs, vs), bool)
    for bi in range(B):
        _surface(f[bi], vs, occ[bi])
        with np.errstate(all="ignore"):
            v = np.floor(f[bi].reshape(-1, 3))
            ok = ((v >= 0) & (v < vs)).all(1)  # voxelize_sub2; NaN / inf: nothing
        vi = v[ok].astype(np.int64)
        occ[bi, vi[:, 0], vi[:, 1], vi[:, 2]] = True
    return occ


def outside_np(occ):
    """The reference's sub3/sub4 fixed point: empty voxels 6-connected through empty voxels to an empty boundary voxel."""
    vis = np.zeros_like(occ)
    struct = ndimage.generate_binary_structure(3, 1)
    for bi in range(occ.shape[0]):
        lab, _ = ndimage.label(~occ[bi], structure=struct)
        shell = np.concatenate([lab[0].ravel(), lab[-1].ravel(), lab[:, 0].ravel(), lab[:, -1].ravel(),
                                lab[:, :, 0].ravel(), lab[:, :, -1].ravel()])
        seeds = np.unique(shell[shell > 0])
        vis[bi] = np.isin(lab, seeds)
    return vis


def voxelization_np(faces, size, normalize=False):
    """faces [B,F,3,3] float32 / float64 -> int32 [B,size,size,size] (functional/voxelization.py:41-58)."""
    return (~outside_np(occupancy_np(faces, size, normalize))).astype(np.int32)


def box_faces(lo, hi, open_side=None):
    """Closed axis-aligned box [lo, hi]^3 as 12 triangles [12,3,3] (float64; cast as needed).  open_side = (axis, 0 | 1)
    leaves out the two triangles of that side."""
    lo, hi = np.broadcast_to(np.asarray(lo, np.float64), (3,)), np.broadcast_to(np.asarray(hi, np.float64), (3,))
    tris = []
    for ax in range(3):
        u, v = [a for a in range(3) if a != ax]
        for side, val in ((0, lo[ax]), (1, hi[ax])):
            if open_side == (ax, side):
                continue
            q = []
            for cu, cv in ((lo[u], lo[v]), (hi[u], lo[v]), (hi[u], hi[v]), (lo[u], hi[v])):
                p = np.zeros(3)
                p[ax], p[u], p[v] = val, cu, cv
                q.append(p)
            tris += [[q[0], q[1], q[2]], [q[0], q[2], q[3]]]
    return np.asarray(tris)


def box_with_hole(lo, hi, axis, side, hole_lo, hole_hi):
    """Box [lo, hi]^3 whose side (axis, side) has a square hole [hole_lo, hole_hi]^2 in the other two coordinates: the
    side is tiled by 8 rectangles (16 triangles) around the hole."""
    faces = [box_faces(lo, hi, open_side=(axis, side))]
    u, v = [a for a in range(3) if a != axis]
    val = hi if side else lo
    cuts = [lo, hole_lo, hole_hi, hi]
    for i in range(3):
        for j in range(3):
            if i == 1 and j == 1:
                continue
            q = []
            for cu, cv in ((cuts[i], cuts[j]), (cuts[i + 1], cuts[j]), (cuts[i + 1], cuts[j + 1]), (cuts[i], cuts[j + 1])):
                p = np.zeros(3)
                p[axis], p[u], p[v] = val, cu, cv
                q.append(p)
            faces.append(np.asarray([[q[0], q[1], q[2]], [q[0], q[2], q[3]]]))
    return np.concatenate(faces)
