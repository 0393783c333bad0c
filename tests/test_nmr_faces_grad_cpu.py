"""The geometry-gradient oracle (tests/nmr_faces_oracle.py, DESIGN.md §14) against an independent brute-force
statement and hand-computed cases, and the host side of umr_nmr_backward_faces and of the functional API -- no GPU."""
import ctypes
import importlib

import numpy as np
import pytest
import torch

import nmr_faces_oracle as oracle
import nmr_scenes as sc
from umr_b200 import _lib
from umr_b200 import neural_renderer as nr

nr_mod = importlib.import_module("umr_b200.neural_renderer.rasterize")   # the module; nr.rasterize is the function

f32 = np.float32
UMR_ERR_UNSUPPORTED, UMR_ERR_BAD_ARG, UMR_ERR_TOO_LARGE = -1, -2, -3
FAKE = ctypes.c_void_p(256)   # a non-null pointer that is never dereferenced: validation fails before any launch


def brute_force(faces, fidx, I, g, eps):
    """The edge term stated pixel by pixel in float64: for every face, edge and pixel column (row), the pixels on the
    face's side of the edge and outside it are found by the sign of the edge's cross product, not by rounding the
    crossing; each pixel p whose colour would change if the edge moved onto it contributes (what the change costs) /
    (how far vertex a or b must move, found by intersecting the moved edge with the pixel's line)."""
    B, F = faces.shape[:2]
    S = fidx.shape[1]
    out = np.zeros((B, F, 3, 3))
    for b in range(B):
        for f in range(F):
            P = 0.5 * (faces[b, f, :, :2].astype(np.float64) * S + S - 1)
            x, y = faces[b, f, :, 0], faces[b, f, :, 1]
            if (y[2] - y[0]) * (x[1] - x[0]) < (y[1] - y[0]) * (x[2] - x[0]):
                continue
            for e in range(3):
                ka, kb, ko = e, (e + 1) % 3, (e + 2) % 3
                for axis in range(2):
                    u, v = (0, 1) if axis == 0 else (1, 0)
                    ua, ub = P[ka, u], P[kb, u]
                    if ua == ub:
                        continue
                    for d0 in range(S):
                        if not min(ua, ub) <= d0 <= max(ua, ub):
                            continue
                        t = (d0 - ua) / (ub - ua)
                        vc = P[ka, v] + t * (P[kb, v] - P[ka, v])
                        side_o = np.sign(P[ko, v] - (P[ka, v] + (P[ko, u] - ua) / (ub - ua) * (P[kb, v] - P[ka, v])))
                        # inner / outer pixels: the nearest centres on the third vertex's side and on the other side
                        inner = [d1 for d1 in range(S) if np.sign(d1 - vc) == side_o or d1 == vc]
                        outer = [d1 for d1 in range(S) if d1 not in inner]
                        if not inner or not outer:
                            continue
                        i_in = min(inner, key=lambda d1: abs(d1 - vc))
                        i_out = max(outer, key=lambda d1: -abs(d1 - vc))
                        if abs(i_in - i_out) != 1:
                            continue
                        at = lambda d1: (b, d1, d0) if axis == 0 else (b, d0, d1)  # noqa: E731

                        def add(d1, ref):
                            diff = float(np.dot(I[at(d1)] - I[at(ref)], g[at(d1)]))
                            if diff <= 0:
                                return
                            for k, lever in ((ka, (ub - ua) / (ub - d0) if ub != d0 else None),
                                             (kb, (ub - ua) / (d0 - ua) if ua != d0 else None)):
                                if lever is None:
                                    continue
                                dist = lever * (d1 - vc) * 2 / S
                                dist = dist + eps if dist > 0 else dist - eps
                                out[b, f, k, 1 if axis == 0 else 0] -= diff / dist
                        if fidx[at(i_in)] == f:
                            for d1 in outer:
                                add(d1, i_in)
                        for d1 in inner:
                            if fidx[at(d1)] == f:
                                add(d1, i_out)
    return out


def _scene(seed):
    rng = np.random.default_rng(seed)
    v, f = sc.mesh(B=1, subdiv=0, seed=seed, soup=3)
    faces = np.take_along_axis(v[:, None], f[..., None].astype(np.int64), axis=2).astype(f32)
    return faces + rng.uniform(-1e-3, 1e-3, size=faces.shape).astype(f32) * [1, 1, 0]


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("aa", [False, True])
def test_oracle_edge_term_matches_the_brute_force(seed, aa):
    """On a closed mesh every pixel a face's shrinking walk takes lies inside that face, so the walk's end is not
    visible here; the brute force takes the whole inner side and keeps the face's own pixels."""
    IS = 20
    S = IS * (2 if aa else 1)
    faces = _scene(seed)
    rng = np.random.default_rng(seed + 10)
    ga = rng.uniform(-1, 1, size=(1, IS, IS)).astype(f32)
    zb = oracle.zbuffer(faces, IS, aa)
    got = oracle.grad_faces(faces, grad_alpha=ga, image_size=IS, anti_aliasing=aa, zbuf=zb)
    A = (zb[0] >= 0).astype(np.float64)[..., None]
    G = oracle.raster_grad(ga, S, aa).astype(np.float64)[..., None]
    ref = brute_force(faces, zb[0], A, G, 1e-4)
    assert np.abs(ref).sum() > 0
    np.testing.assert_allclose(got, ref, rtol=2e-3, atol=1e-3 * np.abs(ref).max())


def test_half_plane_target_sign_and_magnitude():
    """One triangle; the alpha adjoint is -1 at one pixel just below its bottom edge (a target that wants the face to
    grow there) and 0 elsewhere.  Only the columns' growing walk sees it: the bottom edge's two vertices get a
    negative y gradient (descent moves them down), in proportion to the pixel's lever on each, and nothing else."""
    IS = 16
    c = lambda i: sc.centre(i, IS)  # noqa: E731
    y0 = 0.5 * (c(4) + c(5))        # bottom edge half-way between raster rows 4 and 5
    faces = np.array([[[[c(2), y0, 5.0], [c(12), y0, 5.0], [c(7), c(13), 5.0]]]], f32)
    ga = np.zeros((1, IS, IS), f32)
    col, row = 5, 3                  # raster pixel (x 5, y 3): two rows below the edge; output row IS-1-row
    ga[0, IS - 1 - row, col] = -1.0
    g = oracle.grad_faces(faces, grad_alpha=ga, image_size=IS, anti_aliasing=False)
    ua, ub = 2.0, 12.0
    vc = 4.5
    d_a = (ub - ua) / (ub - col) * (row - vc) * 2 / IS - 1e-4
    d_b = (ub - ua) / (col - ua) * (row - vc) * 2 / IS - 1e-4
    want = np.zeros((3, 3))
    want[0, 1] = -1.0 / d_a
    want[1, 1] = -1.0 / d_b
    np.testing.assert_allclose(g[0, 0], want, rtol=1e-5, atol=0)
    assert want[0, 1] > 0 and want[1, 1] > 0   # dL/dy > 0: gradient descent lowers y


def test_half_plane_target_x_gradient():
    """A triangle whose right edge is vertical; the alpha adjoint -1 one pixel to its right pulls both of that edge's
    vertices right (negative x gradient, descent increases x) through the rows' growing walk."""
    IS = 16
    c = lambda i: sc.centre(i, IS)  # noqa: E731
    x1 = 0.5 * (c(10) + c(11))
    faces = np.array([[[[c(2), c(2), 5.0], [x1, c(2), 5.0], [x1, c(13), 5.0]]]], f32)
    ga = np.zeros((1, IS, IS), f32)
    ga[0, IS - 1 - 7, 12] = -1.0     # raster pixel (x 12, y 7)
    g = oracle.grad_faces(faces, grad_alpha=ga, image_size=IS, anti_aliasing=False)
    # edge 1 -> 2 is vertical: on axis 1 (rows) it runs from y 2 to y 13; lever (13-2)/(13-7) on vertex 1, /(7-2) on 2
    d1 = (13.0 - 2.0) / (13.0 - 7.0) * (12 - 10.5) * 2 / IS + 1e-4
    d2 = (13.0 - 2.0) / (7.0 - 2.0) * (12 - 10.5) * 2 / IS + 1e-4
    want = np.zeros((3, 3))
    want[1, 0] = -1.0 / d1
    want[2, 0] = -1.0 / d2
    np.testing.assert_allclose(g[0, 0], want, rtol=1e-5, atol=0)


def test_depth_term_is_the_derivative_of_the_depth_plane():
    """The depth term against central differences of the oracle's own depth plane, at pixels well inside faces."""
    faces = _scene(3)
    IS = 24
    rng = np.random.default_rng(0)
    gd = rng.uniform(-1, 1, size=(1, IS, IS)).astype(f32)
    g = oracle.grad_faces(faces, grad_depth=gd, image_size=IS, anti_aliasing=False)
    fidx = oracle.zbuffer(faces, IS, False)[0]

    def loss(fc):
        r = oracle.render(fc.astype(f32), image_size=IS, anti_aliasing=False)
        same = r["face_index"] == fidx
        return float((r["depth"].astype(np.float64) * gd * same[:, ::-1]).sum()), same.all()
    checked = 0
    for f in np.unique(fidx[fidx >= 0])[:4]:
        for k in range(3):
            for comp in range(3):
                h = 1e-3
                fp, fm = faces.astype(np.float64).copy(), faces.astype(np.float64).copy()
                fp[0, f, k, comp] += h
                fm[0, f, k, comp] -= h
                lp, okp = loss(fp)
                lm, okm = loss(fm)
                if not (okp and okm):
                    continue
                np.testing.assert_allclose(g[0, f, k, comp], (lp - lm) / (2 * h), rtol=2e-2, atol=2e-2)
                checked += 1
    assert checked > 6


def test_oracle_magnitude_and_counts():
    faces = _scene(2)
    rng = np.random.default_rng(1)
    IS = 16
    tex = rng.uniform(0, 1, size=faces.shape[:2] + (2, 2, 2, 3)).astype(f32)
    gr = rng.uniform(-1, 1, size=(1, 3, IS, IS)).astype(f32)
    ga = rng.uniform(-1, 1, size=(1, IS, IS)).astype(f32)
    gd = rng.uniform(-1, 1, size=(1, IS, IS)).astype(f32)
    g, mag, cnt = oracle.grad_faces(faces, tex, gr, ga, gd, image_size=IS, magnitude=True)
    assert (mag >= np.abs(g)).all() and (cnt > 0).any() and (mag[cnt == 0] == 0).all()
    assert np.array_equal(oracle.grad_faces(faces, tex, gr, ga, gd, image_size=IS), g)


# ---------------------------------------------------------------------------------------------------------------
# the C entry point without a GPU
# ---------------------------------------------------------------------------------------------------------------
def _params(**kw):
    p = nr_mod._params(2, 10, 3, 32, True, 0.1, 100.0, [0, 0, 0])
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _call(p, vertices=FAKE, faces=FAKE, face_index=FAKE, textures=FAKE, grad_rgb=FAKE, grad_alpha=FAKE,
          grad_depth=FAKE, grad=FAKE, eps=1e-4, workspace=FAKE):
    lib = _lib.load()
    return lib.umr_nmr_backward_faces(vertices, faces, face_index, textures, grad_rgb, grad_alpha, grad_depth, grad,
                                      ctypes.byref(p) if p is not None else None, eps, workspace, None)


def test_backward_faces_refusals():
    N0 = None
    assert _call(None) == UMR_ERR_BAD_ARG
    for field, val in (("batch_size", 0), ("num_vertices", 0), ("num_faces", 0), ("image_size", 0),
                       ("texture_res", 1)):
        assert _call(_params(**{field: val})) == UMR_ERR_BAD_ARG, field
    assert _call(_params(batch_size=65536)) == UMR_ERR_TOO_LARGE
    assert _call(_params(image_size=8193)) == UMR_ERR_TOO_LARGE
    assert _call(_params(texture_res=102)) == UMR_ERR_TOO_LARGE
    assert _call(_params(num_faces=2 ** 30 + 1)) == UMR_ERR_TOO_LARGE
    for arg in ("vertices", "faces", "face_index", "grad", "workspace"):
        assert _call(_params(), **{arg: N0}) == UMR_ERR_BAD_ARG, arg
    assert _call(_params(texture_res=0), textures=N0) == UMR_ERR_BAD_ARG            # grad_rgb without textures
    assert _call(_params(), workspace=ctypes.c_void_p(256 + 128)) == UMR_ERR_BAD_ARG
    assert _call(_params(), grad=ctypes.c_void_p(258)) == UMR_ERR_BAD_ARG
    for eps in (-1e-4, float("inf"), float("nan")):
        assert _call(_params(), eps=eps) == UMR_ERR_BAD_ARG, eps
    assert _call(_params(fill_back=1)) == UMR_ERR_UNSUPPORTED
    assert _call(_params(light_intensity_directional=0.5)) == UMR_ERR_UNSUPPORTED


@pytest.mark.parametrize("B,F,IS,aa", [(1, 1, 1, 0), (2, 10, 32, 1), (16, 1280, 256, 1), (3, 7, 65, 0)])
def test_backward_faces_workspace_formula(B, F, IS, aa):
    lib = _lib.load()
    a = lambda x: (x + 255) // 256 * 256  # noqa: E731
    S = IS * (2 if aa else 1)
    assert lib.umr_nmr_backward_faces_workspace_bytes(B, F, IS, aa) == a(128 * B * F) + a(16 * B * F) + a(12 * B * S * S)


def test_backward_faces_workspace_refused_sizes():
    lib = _lib.load()
    for args in ((0, 1, 1, 0), (1, 0, 1, 0), (1, 1, 0, 0), (65536, 1, 1, 0), (1, 2 ** 30 + 1, 1, 0), (1, 1, 8193, 1),
                 (1, 1, 16385, 0)):
        assert lib.umr_nmr_backward_faces_workspace_bytes(*args) == 0, args


# ---------------------------------------------------------------------------------------------------------------
# the Python API without a GPU
# ---------------------------------------------------------------------------------------------------------------
def test_api_defaults_and_names():
    assert (nr.DEFAULT_NEAR, nr.DEFAULT_FAR, nr.DEFAULT_EPS) == (0.1, 100, 1e-4)
    assert nr.DEFAULT_IMAGE_SIZE == 256 and nr.DEFAULT_ANTI_ALIASING is True
    assert tuple(nr.DEFAULT_BACKGROUND_COLOR) == (0, 0, 0)
    for name in ("rasterize_rgbad", "rasterize", "rasterize_silhouettes", "rasterize_depth", "vertices_to_faces",
                 "Renderer"):
        assert name in nr.__all__ and callable(getattr(nr, name))


def test_api_argument_validation():
    faces = torch.zeros(2, 4, 3, 3)
    tex = torch.zeros(2, 4, 2, 2, 2, 3)
    with pytest.raises(TypeError):
        nr.rasterize_rgbad(faces, tex)                       # CPU tensors
    with pytest.raises(TypeError):
        nr.rasterize_silhouettes(faces)
    with pytest.raises(TypeError):
        nr.rasterize_depth(faces.double())
    with pytest.raises(ValueError):
        nr.rasterize_rgbad(torch.zeros(2, 4, 3))             # not [B,F,3,3]
    with pytest.raises(ValueError):
        nr.rasterize_rgbad(torch.zeros(2, 4, 3, 3, dtype=torch.int32), tex)
    with pytest.raises(ValueError):
        nr.rasterize_rgbad(faces)                             # rgb without textures
    with pytest.raises(ValueError):
        nr.rasterize_rgbad(faces, torch.zeros(2, 4, 2, 2, 3, 3))
    with pytest.raises(ValueError):
        nr.rasterize_rgbad(faces, torch.zeros(2, 5, 2, 2, 2, 3))
    with pytest.raises(NotImplementedError):
        nr.rasterize_rgbad(faces, torch.zeros(2, 4, 1, 1, 1, 3))
    with pytest.raises(ValueError):
        nr.rasterize_rgbad(faces, tex, image_size=0)
    with pytest.raises(ValueError):
        nr.rasterize_rgbad(faces, tex, eps=-1.0)
    with pytest.raises(ValueError):
        nr.rasterize_rgbad(faces, tex, background_color=[0, 0])
    with pytest.raises(ValueError):
        nr.rasterize_rgbad(faces, tex, return_rgb=False, return_alpha=False, return_depth=False)


def test_vertices_to_faces_is_a_differentiable_gather():
    rng = np.random.default_rng(0)
    v = torch.from_numpy(rng.normal(size=(2, 5, 3))).requires_grad_(True)
    f = torch.tensor([[[0, 1, 2], [2, 3, 4]], [[4, 0, 1], [1, 1, 3]]], dtype=torch.int32)
    fv = nr.vertices_to_faces(v, f)
    assert fv.shape == (2, 2, 3, 3)
    for b in range(2):
        assert torch.equal(fv[b], v[b][f[b].long()])
    fv.sum().backward()
    assert torch.equal(v.grad[1, 1], torch.full((3,), 3.0, dtype=torch.float64))
    with pytest.raises(ValueError):
        nr.vertices_to_faces(v, f.float())
    with pytest.raises(ValueError):
        nr.vertices_to_faces(v, f + 5)
    with pytest.raises(ValueError):
        nr.vertices_to_faces(v[:, :, :2], f)
