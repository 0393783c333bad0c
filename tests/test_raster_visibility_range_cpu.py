"""Without a GPU: each visibility scene of raster_range_scenes.py has the property test_raster_visibility_range_gpu.py
relies on, by float32 restatements of the kernels' arithmetic (raster.cu is built -fmad=false, so each float operation
is one IEEE operation and the restatements are exact), and umr_raster_visibility refuses bad arguments before any
CUDA call."""
import ctypes

import numpy as np

import raster_range_scenes as rs
from umr_b200 import _lib, raster

OK, UNSUPPORTED, BAD_ARG, TOO_LARGE = 0, -1, -2, -3
F32 = np.float32


def _box(f, thin):
    """k_visible_faces' box of one face [9]: the cull box (vertex box +- r) for a thin face, else the vertex box."""
    if thin:
        return rs.boxes(np.asarray(f)[None], F32)[0]
    x, y = np.asarray(f, F32)[0::3], np.asarray(f, F32)[1::3]
    return np.array([x.min(), x.max(), y.min(), y.max()], F32)


def _crosses(f, S):
    thin = rs.thin_flag(f)
    xlo, xhi, ylo, yhi = _box(f, thin)
    return [rs.crosses_int32(xlo, S, -1), rs.crosses_int32(xhi, S, 1), rs.crosses_int32(ylo, S, -1),
            rs.crosses_int32(yhi, S, 1)]


def _inside64(f, S):
    """[S, S] (image rows from the top): pixel centres inside the triangle, closed, in float64."""
    c = rs.pixel_centre(np.arange(S), S, np.float64)
    xp, yp = np.meshgrid(c, c[::-1])
    x0, y0, _, x1, y1, _, x2, y2, _ = np.asarray(f, np.float64)
    det = x2 * (y0 - y1) + x0 * (y1 - y2) + x1 * (y2 - y0)
    w0 = ((y1 - y2) * xp + (x2 - x1) * yp + (x1 * y2 - x2 * y1)) / det
    w1 = ((y2 - y0) * xp + (x0 - x2) * yp + (x2 * y0 - x0 * y2)) / det
    return (w0 >= 0) & (w1 >= 0) & (1 - w0 - w1 >= 0)


def _depth32(f, w):
    """depth_of after clip_bary (raster_generic.cuh), in float32, at float32 barycentrics w [3, ...]."""
    lo, hi = F32(1e-5), F32(1 - 1e-5)
    k = [np.fmax(np.fmin(F32(v), hi), lo) for v in w]
    s = np.fmax(k[0] + k[1] + k[2], lo)
    k = [v / s for v in k]
    z = np.asarray(f, F32)[2::3]
    with np.errstate(divide="ignore"):
        return (F32(1) / (k[0] / z[0] + k[1] / z[1] + k[2] / z[2])).astype(F32)


def _bary32(f, xp, yp):
    """k_prep's barycentric inverse and the kernels' w = i0 x + i1 y + i2, in float32."""
    x0, y0, _, x1, y1, _, x2, y2, _ = np.asarray(f, F32)
    star = [y1 - y2, x2 - x1, x1 * y2 - x2 * y1, y2 - y0, x0 - x2, x2 * y0 - x0 * y2, y0 - y1, x1 - x0, x0 * y1 - x1 * y0]
    det = x2 * (y0 - y1) + x0 * (y1 - y2) + x1 * (y2 - y0)
    det = np.fmax(det, F32(1e-10)) if det > 0 else np.fmin(det, F32(-1e-10))
    inv = [F32(s / det) for s in star]
    return [(inv[3 * r] * xp + inv[3 * r + 1] * yp + inv[3 * r + 2]).astype(F32) for r in range(3)]


def test_far_off_boxes_cross_the_int32_index_range():
    """Factor 1/2 stays inside int32 at its S, factors 1, 2 and 1000 leave it; at S = 2048 the wide faces of factors
    1/2 and 1 take the tight vertex box (not thin) and the factor-1 one crosses: the tight-box path is covered too.
    (Past WIDE_DRAWN, where no wide face is drawn, k_prep's products overflow and may clear bit 4 again.)"""
    tight_crossing = 0
    for S in (64, 2048):
        fv, meta = rs.far_faces(S)
        for f, m in zip(fv[:, 0], meta):
            kind, axis, side, fac, X = m
            cr = _crosses(f, S)
            assert any(cr) == (fac >= 1), (S, m, cr)
            if kind == "thin":
                assert rs.thin_flag(f)
                k = 2 * axis + (side > 0)
                assert cr == [fac >= 1 and i == k for i in range(4)], (S, m, cr)   # one side only
            elif not rs.thin_flag(f) and X < rs.WIDE_DRAWN:   # past WIDE_DRAWN the face is not drawn at all
                assert S == 2048 and fac <= 1, (S, m)
                tight_crossing += fac == 1
    assert tight_crossing == 4


def test_far_off_faces_lie_over_pixel_centres():
    """In float64 every far face covers pixel centres: the wide ones all of them, the thin ones the band across the
    raster between y (or x) = -0.5 and 0.5."""
    for S in (64, 2048):
        fv, meta = rs.far_faces(S)
        for f, m in zip(fv[:, 0], meta):
            ins = _inside64(f, S)
            if m[0] == "wide":
                assert ins.all(), (S, m)
            else:
                assert 0 < ins.sum() < ins.size, (S, m)


def test_huge_faces():
    """1e20 overflows x y in float32 for the wide face (its inverse is not finite); the thin faces stay finite."""
    fv, meta = rs.huge_faces()
    for f, m in zip(fv[:, 0], meta):
        x0, y0, _, x1, y1, _, x2, y2, _ = f.astype(F32)
        with np.errstate(over="ignore", invalid="ignore"):
            prods = np.array([x1 * y2, x2 * y1, x2 * y0, x0 * y2, x0 * y1, x1 * y0], F32)
        assert np.isfinite(prods).all() == (m[0] == "thin" or m[1] == 1e15), m


def test_thin_switch_pairs_straddle_the_bit4_cut():
    """Bit 4 is set on the first sliver of each pair only (rs._sliver finds the two float heights either side of the
    cut); each sliver covers pixel centres within 3 % of its length of both ends of its box."""
    for S in (64, 65, 126, 1000):
        fv, thin = rs.thin_switch(S)
        assert [rs.thin_flag(f) for f in fv[0]] == thin.tolist()
        for f in fv[0]:
            ins = _inside64(f, S)
            cols = np.flatnonzero(ins.any(0)) if ins.any(1).sum() <= 1 else np.flatnonzero(ins.any(1))
            box = _box(f, rs.thin_flag(f))
            n = max(box[1] - box[0], box[3] - box[2]) * S / 2   # the box's length in pixels
            assert len(cols) and cols.max() - cols.min() >= 0.94 * n - 2, (S, cols.min(), cols.max(), n)


def test_zero_depth_pair():
    """Every covered pixel of the +0 face has depth +0, of the -0 face -0; both pass near = 0 (neither is < 0)."""
    fv = rs.zero_depths()
    S = 64
    c = rs.pixel_centre(np.arange(S), S, F32)
    xp, yp = np.meshgrid(c, c[::-1])
    for f, sign in ((fv[0, 0], 1), (fv[0, 1], -1)):
        ins = _inside64(f, S)
        w = _bary32(f, xp[ins], yp[ins])
        z = _depth32(f, w)
        assert ins.sum() > 100 and (z == 0).all() and (np.signbit(z) == (sign < 0)).all()
        assert not (z < F32(0)).any()
    assert fv[1, 0].tobytes() == fv[0, 1].tobytes() and fv[1, 1].tobytes() == fv[0, 0].tobytes()


def test_tie_scenes_have_equal_depths():
    """repeat: identical copies; edge: on the shared column / row the two halves have the same float32 depth and a
    barycentric exactly 0; depth cut: pixels of both faces on both sides of 1e7."""
    S = 64
    fv, names = rs.depth_order(S)
    r = fv[names.index("repeat")]
    assert r[1].tobytes() == r[2].tobytes() == r[4].tobytes() == r[5].tobytes()
    e = fv[names.index("edge")]
    c = rs.pixel_centre(np.arange(S), S, F32)
    for a, b, col in ((e[0], e[1], True), (e[2], e[3], False)):
        line = a[0] if col else a[1]
        idx = np.flatnonzero(c == line)
        assert len(idx) == 1
        o = c[(c > min(a[1::3].min(), b[1::3].min()) + 0.05) & (c < max(a[1::3].max(), b[1::3].max()) - 0.05)] if col else \
            c[(c > min(a[0::3].min(), b[0::3].min()) + 0.05) & (c < max(a[0::3].max(), b[0::3].max()) - 0.05)]
        xp, yp = (np.full_like(o, line), o) if col else (o, np.full_like(o, line))
        wa, wb = _bary32(a, xp, yp), _bary32(b, xp, yp)
        assert any((w == 0).all() for w in wa) and any((w == 0).all() for w in wb)
        assert np.array_equal(_depth32(a, wa), _depth32(b, wb))
    cut = rs.depth_cut()
    xp, yp = np.meshgrid(c, c[::-1])
    for f in cut[0, :2]:   # the rounding of clip_bary and depth_of puts both faces' pixels either side of 1e7
        ins = _inside64(f, S)
        z = _depth32(f, _bary32(f, xp[ins], yp[ins]))
        assert (z < F32(1e7)).any() and (z >= F32(1e7)).any(), np.unique(z)


def test_front_back_faces_alternate():
    fv = rs.front_back(seed=4)[0]
    for i, f in enumerate(fv):
        x0, y0, _, x1, y1, _, x2, y2, _ = f.astype(F32)
        front = (y2 - y0) * (x1 - x0) < (y1 - y0) * (x2 - x0)   # k_prep's bit 3
        assert front == (i % 2 == 0), i


def _params(B=1, F=4, isz=8, dist="euclidean"):
    return raster.make_params(B, F, 1, isz, False, (0.0, 0.0, 0.0), 1.0, 100.0, True, 1e-3, 1e-5, dist, 1e-4, 1e-4, "hard",
                              "prod", "surface")


def test_c_abi_refusals_without_gpu():
    """Argument checks return before any CUDA call."""
    lib = _lib.load()
    p = ctypes.c_void_p(256)
    ws = ctypes.c_void_p(512)
    call = lambda fv, aggrs, vis, prm, w: lib.umr_raster_visibility(fv, aggrs, vis, ctypes.byref(prm), w, None)  # noqa: E731
    assert call(None, p, p, _params(), ws) == BAD_ARG                         # no face_vertices
    assert call(p, None, None, _params(), ws) == BAD_ARG                      # neither output
    assert call(p, p, None, _params(), None) == BAD_ARG                       # no workspace
    assert call(p, None, p, _params(), ctypes.c_void_p(512 + 16)) == BAD_ARG  # workspace not 256-byte aligned
    assert call(p, p, p, _params(dist="barycentric"), ws) == UNSUPPORTED      # a generic mode
    assert call(p, p, p, _params(F=(1 << 24) + 1), ws) == TOO_LARGE           # F > UMR_RASTER_MAX_FACES
    assert call(p, p, p, _params(B=65536), ws) == TOO_LARGE
    assert call(p, p, p, _params(F=0), ws) == BAD_ARG
    assert lib.umr_raster_workspace_bytes(1, 1 << 24, 1, 0) > 0
