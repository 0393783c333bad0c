"""The NMR oracle (oracle/nmr.py) on the edge scenes of tests/nmr_scenes.py, its `window=`, `magnitude=` and `counts=`
options, and the host side of the umr_nmr_* entry points (refusals, workspace size) -- no GPU needed.

tests/test_nmr_range_gpu.py compares the kernels bit-exact with this oracle on the same scenes, so here the oracle's
per-face pixel regions are checked against its exhaustive walk (every face copy on every pixel) on each of them."""
import ctypes
import itertools

import numpy as np
import pytest

import nmr as oracle
import nmr_scenes as sc
from umr_b200 import _lib

f32 = np.float32
EYE = sc.EYE
UMR_ERR_BAD_ARG, UMR_ERR_TOO_LARGE = -2, -3
FAKE = ctypes.c_void_p(256)   # a non-null pointer that is never dereferenced: validation fails before any launch
N0 = ctypes.c_void_p(0)

SCENES = {
    "grid": lambda S: sc.grid(S, n=4, step=S // 8),
    "duplicates": lambda S: sc.duplicates(*sc.mesh(B=2, seed=1)),
    "zero_area": sc.zero_area,
    "thin": sc.thin,
    "invalid": lambda S: sc.invalid(B=2)[:2],
    "clipped": lambda S: sc.clipped(B=2),
}


@pytest.mark.parametrize("name", sorted(SCENES))
@pytest.mark.parametrize("aa", [False, True])
def test_pixel_regions_match_the_exhaustive_z_buffer(name, aa):
    IS = 24
    S = IS * (2 if aa else 1)
    v, f = SCENES[name](S)
    planes = [dict(), dict(near=4.5, far=9.0), dict(eye_z=-1.0, near=-3.0, far=6.0)] if name == "clipped" else [dict()]
    for kw in planes:
        for fill_back in (True, False):
            a = oracle.zbuffer(v, f, IS, aa, fill_back, **dict(dict(eye_z=EYE), **kw))
            b = oracle.zbuffer(v, f, IS, aa, fill_back, exhaustive=True, **dict(dict(eye_z=EYE), **kw))
            assert np.array_equal(a[0], b[0])
            assert np.array_equal(a[1].view(np.int32), b[1].view(np.int32))


def test_signed_zero_depths_follow_the_strict_walk():
    """eye_z = +0, near < 0: +0 and -0 depths meet; the lower face index wins either way, its own zero's sign kept."""
    v, f = sc.signed_zero()
    fidx, depth = oracle.zbuffer(v, f, 16, False, False, eye_z=0.0, near=-1.0, far=100.0, exhaustive=True)
    st = sc.pixel_stats(v, f, 16, False, False, eye_z=0.0, near=-1.0)
    assert st["zero"] > 0 and st["ties"] > 0
    assert set(np.unique(fidx)) == {-1, 0, 2}
    zero = depth == 0
    assert (zero & (fidx == 0)).any() and (zero & (fidx == 2)).any()
    assert not np.signbit(depth[zero & (fidx == 0)]).any() and np.signbit(depth[zero & (fidx == 2)]).all()


@pytest.mark.parametrize("aa", [False, True])
def test_window_equals_the_crop_of_the_full_z_buffer(aa):
    IS = 24
    S = IS * (2 if aa else 1)
    v, f = sc.thin(S)
    v2, f2 = sc.mesh(B=2, seed=2)
    for verts, faces in ((v, f), (v2, f2)):
        full = oracle.zbuffer(verts, faces, IS, aa, True, EYE)
        for win in ((0, S - 1, 0, S - 1), (3, 9, 5, 5), (0, 0, S - 1, S - 1), (S // 2, S - 1, 1, S // 3)):
            c0, c1, r0, r1 = win
            part = oracle.zbuffer(verts, faces, IS, aa, True, EYE, window=win)
            assert np.array_equal(part[0], full[0][:, r0:r1 + 1, c0:c1 + 1])
            assert np.array_equal(part[1], full[1][:, r0:r1 + 1, c0:c1 + 1])


def test_gradient_magnitude_and_counts_against_a_loop():
    B, IS, T = 2, 6, 3
    v, f = sc.mesh(B=B, seed=4, soup=3)
    rng = np.random.default_rng(9)
    g = rng.normal(size=(B, 3, IS, IS))
    g[:, :, ::3] = 0.0
    light = dict(Ia=0.4, Id=0.7, ca=(1, 0.5, 0.2), cd=(0.3, 1, 2), direction=(0.5, 1, -1))
    for aa, G in ((True, 1), (False, 2)):
        zb = oracle.zbuffer(v, f, IS, aa, True, EYE)
        shape = (B // G, f.shape[1], T, T, T, 3)
        out, mag, cnt = oracle.grad_textures(g, v, f, shape, zb, anti_aliasing=aa, fill_back=True, eye_z=EYE,
                                             shared_textures=G, magnitude=True, counts=True, **light)
        assert np.array_equal(out, oracle.grad_textures(g, v, f, shape, zb, anti_aliasing=aa, fill_back=True,
                                                        eye_z=EYE, shared_textures=G, **light))
        # brute force: one pixel and one corner at a time
        S = IS * (2 if aa else 1)
        F = f.shape[1]
        fv = oracle.face_copies(v, f, True)
        _, z, inv = oracle._records(fv, S, EYE)
        lit = oracle.lights(fv, **light).astype(np.float64)
        gr = oracle._raster_grad(g, S, aa)
        ref_s, ref_m, ref_n = np.zeros(shape), np.zeros(shape), np.zeros(shape[:-1], np.int64)
        for b, yi, xi in zip(*np.nonzero(zb[0] >= 0)):
            fc = int(zb[0][b, yi, xi])
            w, zp = oracle.bary(inv[b, fc], z[b, fc], f32(xi), f32(yi))
            tif = [min(max((w[k] * f32(T - 1)) * (zp / z[b, fc, k]), f32(0)), f32(T - 1) - f32(1e-3)) for k in range(3)]
            for pn in range(8):
                wt, ii = f32(1), []
                for k in range(3):
                    t0 = int(tif[k])
                    frac = tif[k] - f32(t0)
                    wt = wt * (frac if (pn >> k) & 1 else f32(1) - frac)
                    ii.append(t0 + ((pn >> k) & 1))
                i0, i1, i2 = ii[::-1] if fc >= F else ii
                at = (b // G, fc % F, i0, i1, i2)
                term = lit[b, fc] * float(wt) * gr[b, :, yi, xi]
                ref_s[at] += term
                ref_m[at] += np.abs(term)
                ref_n[at] += 1
        assert ref_n.sum() == 8 * (zb[0] >= 0).sum() and (zb[0] >= F).any()
        assert np.array_equal(cnt, ref_n)
        assert np.allclose(out, ref_s, rtol=1e-12, atol=1e-15) and np.allclose(mag, ref_m, rtol=1e-12, atol=1e-15)
        assert (mag > np.abs(out) * (1 + 1e-9)).any()   # mixed signs cancel somewhere


# ---------------------------------------------------------------------------------------------------------------------
# entry points: refusals and workspace
# ---------------------------------------------------------------------------------------------------------------------
def _params(B=2, V=10, F=4, T=3, IS=8, aa=1, fill_back=1, G=1):
    p = _lib.UmrNmrParams()
    p.batch_size, p.num_vertices, p.num_faces, p.texture_res = B, V, F, T
    p.image_size, p.anti_aliasing, p.fill_back, p.shared_textures = IS, aa, fill_back, G
    p.eye_z, p.near_plane, p.far_plane = EYE, 0.1, 100.0
    p.light_intensity_ambient, p.light_intensity_directional = 0.5, 0.5
    return p


def _fwd(p, tex=FAKE, ptrs=None, rgb=FAKE, ws=FAKE):
    v, f, fi, rd = ptrs or (FAKE,) * 4
    return _lib.load().umr_nmr_forward(v, f, tex, fi, rd, rgb, FAKE, FAKE, ctypes.byref(p), ws, None)


def _bwd(p, ptrs=None, gt=FAKE, ws=FAKE, det=False):
    lib = _lib.load()
    fn = lib.umr_nmr_backward_textures_deterministic if det else lib.umr_nmr_backward_textures
    v, f, fi, g = ptrs or (FAKE,) * 4
    return fn(v, f, fi, g, gt, ctypes.byref(p), ws, None)


SHAPE_REFUSALS = [
    (dict(B=0), UMR_ERR_BAD_ARG), (dict(B=65536), UMR_ERR_TOO_LARGE), (dict(V=0), UMR_ERR_BAD_ARG),
    (dict(F=0), UMR_ERR_BAD_ARG), (dict(IS=0), UMR_ERR_BAD_ARG), (dict(IS=8193), UMR_ERR_TOO_LARGE),
    (dict(IS=16385, aa=0), UMR_ERR_TOO_LARGE), (dict(T=1), UMR_ERR_BAD_ARG), (dict(T=102), UMR_ERR_TOO_LARGE),
    (dict(T=2 ** 31 - 1), UMR_ERR_TOO_LARGE), (dict(B=6, G=4), UMR_ERR_BAD_ARG),
    (dict(F=2 ** 29 + 1), UMR_ERR_TOO_LARGE), (dict(F=2 ** 30 + 1, fill_back=0), UMR_ERR_TOO_LARGE),
    (dict(F=2 ** 31 - 1), UMR_ERR_TOO_LARGE),
]


@pytest.mark.parametrize("kw,code", SHAPE_REFUSALS, ids=[",".join("%s=%s" % i for i in k.items()) for k, _ in SHAPE_REFUSALS])
def test_shapes_refused(kw, code):
    launches = _lib.load().umr_launch_count()
    p = _params(**kw)
    assert _fwd(p) == code
    assert _bwd(p) == code and _bwd(p, det=True) == code
    if "T" in kw:   # without textures the texture size is ignored: the shape passes, the NULL workspace is refused
        assert _fwd(p, tex=N0, rgb=N0, ws=N0) == UMR_ERR_BAD_ARG
    assert _lib.load().umr_launch_count() == launches   # a refused call launches nothing


def test_pointers_and_alignment_refused():
    launches = _lib.load().umr_launch_count()
    p = _params()
    for i in range(4):   # vertices, faces, face_index, raster_depth
        ptrs = [FAKE] * 4
        ptrs[i] = N0
        assert _fwd(p, ptrs=ptrs) == UMR_ERR_BAD_ARG
        for det in (False, True):   # vertices, faces, face_index, grad_rgb
            assert _bwd(p, ptrs=ptrs, det=det) == UMR_ERR_BAD_ARG
    assert _fwd(p, ws=N0) == UMR_ERR_BAD_ARG
    assert _fwd(p, tex=N0) == UMR_ERR_BAD_ARG                        # rgb without textures
    for off in (4, 16, 128):
        assert _fwd(p, ws=ctypes.c_void_p(256 + off)) == UMR_ERR_BAD_ARG   # workspace not 256-byte aligned
    for det in (False, True):
        assert _bwd(p, gt=N0, det=det) == UMR_ERR_BAD_ARG
        assert _bwd(p, ws=N0, det=det) == UMR_ERR_BAD_ARG
        assert _bwd(p, ws=ctypes.c_void_p(256 + 64), det=det) == UMR_ERR_BAD_ARG
        for off in (1, 2, 3):
            assert _bwd(p, gt=ctypes.c_void_p(256 + off), det=det) == UMR_ERR_BAD_ARG   # grad_textures not 4-byte aligned
    assert _lib.load().umr_nmr_forward(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None, FAKE, None) == UMR_ERR_BAD_ARG
    assert _lib.load().umr_launch_count() == launches


def _align256(x):
    return (x + 255) // 256 * 256


@pytest.mark.parametrize("B,F,fill_back", list(itertools.product([1, 3, 65535], [1, 7, 70000, 2 ** 29, 2 ** 30], [0, 1])))
def test_workspace_formula(B, F, fill_back):
    lib = _lib.load()
    Fc = F * (2 if fill_back else 1)
    expect = _align256(B * Fc * 128) + _align256(B * Fc * 16) if Fc <= 2 ** 30 else 0
    assert lib.umr_nmr_workspace_bytes(B, F, fill_back) == expect


def test_workspace_is_zero_for_refused_shapes():
    lib = _lib.load()
    for B, F, fb in ((0, 5, 1), (5, 0, 1), (-1, 5, 0), (65536, 5, 1), (1, 2 ** 29 + 1, 1), (1, 2 ** 31 - 1, 1),
                     (1, 2 ** 31 - 1, 0), (1, -5, 1)):
        assert lib.umr_nmr_workspace_bytes(B, F, fb) == 0, (B, F, fb)
