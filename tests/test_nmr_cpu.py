"""The NMR render contract's CPU oracle (oracle/nmr.py) on hand-computed cases, its texture adjoint, and the host side of
umr_b200.neural_renderer (registration, construction, refusals) -- no GPU needed."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import nmr as oracle
from umr_b200 import synth

f32 = np.float32
EYE = -2.732


def tri(*xy, z=5.0):
    """One face [1,3,3] vertices + [1,1,3] faces."""
    v = np.array([[[x, y, z] for x, y in xy]], f32)
    return v, np.array([[[0, 1, 2]]], np.int32)


def test_single_triangle_covers_exactly_the_pixel_centres_its_edge_tests_admit():
    S = 16
    v, f = tri((-0.6, -0.5), (0.7, -0.4), (0.1, 0.8))
    out = oracle.render(v, f, None, image_size=S, anti_aliasing=False, fill_back=False, eye_z=EYE)
    P = [(Fraction(float(a)), Fraction(float(b))) for a, b in v[0, :, :2]]
    cov = np.zeros((S, S), bool)
    for yi in range(S):
        for xi in range(S):
            xp, yp = Fraction(2 * xi + 1 - S, S), Fraction(2 * yi + 1 - S, S)
            cov[yi, xi] = all((yp - P[k][1]) * (P[(k + 1) % 3][0] - P[k][0]) >= (xp - P[k][0]) * (P[(k + 1) % 3][1] - P[k][1])
                              for k in range(3))
    assert 20 < cov.sum() < S * S
    assert np.array_equal(out["face_index"][0] == 0, cov)
    assert np.array_equal(out["face_index"][0] == -1, ~cov)
    assert np.allclose(out["raster_depth"][0][cov], f32(5.0) - f32(EYE), rtol=1e-6)  # 1/sum(w/z) rounds
    assert np.all(out["raster_depth"][0][~cov] == f32(100.0))
    # no anti-aliasing: the output planes are the flipped raster planes
    assert np.array_equal(out["alpha"][0], cov[::-1].astype(f32))


def test_vertical_flip_puts_a_face_with_positive_y_in_the_top_rows():
    v, f = tri((-0.5, 0.2), (0.5, 0.2), (0.0, 0.9))
    out = oracle.render(v, f, None, image_size=16, anti_aliasing=True, fill_back=False, eye_z=EYE)
    S = 32
    rows = np.nonzero((out["face_index"][0] >= 0).any(1))[0]
    assert rows.min() >= S // 2                      # raster rows run bottom-up (yi = 0 is y = -1)
    a = out["alpha"][0]
    assert a[:8].sum() > 0 and a[8:].sum() == 0      # output rows run top-down
    assert set(np.unique(a)) <= {0.0, 0.25, 0.5, 0.75, 1.0}


def _vertex_pixel_scene():
    """A triangle whose vertex 0 sits exactly on the centre of pixel (xi, yi) = (2, 2) of an 8x8 raster, in the plane
    z = 5 (normal along z); `front` picks the vertex order."""
    S = 8
    c = lambda i: (2 * i + 1 - S) / S  # noqa: E731
    return S, (c(2), c(2)), (c(6), c(3)), (c(3), c(6))


@pytest.mark.parametrize("fill_back", [False, True])
def test_back_facing_triangle_and_fill_back(fill_back):
    S, p0, p1, p2 = _vertex_pixel_scene()
    v, f = tri(p0, p2, p1)  # clockwise: back-facing
    rng = np.random.default_rng(0)
    T = 3
    tex = rng.uniform(0.1, 1.0, size=(1, 1, T, T, T, 3)).astype(f32)
    light = dict(light_intensity_ambient=0.25, light_intensity_directional=0.5, light_direction=(0.0, 0.0, -1.0))
    out = oracle.render(v, f, tex, image_size=S, anti_aliasing=False, fill_back=fill_back, eye_z=EYE, **light)
    if not fill_back:
        assert (out["face_index"] == -1).all() and (out["rgb"] == 0).all()
        return
    assert set(np.unique(out["face_index"])) == {-1, 1}  # only the reversed copy (index F + 0) is drawn
    # the copy's light: its normal is -n of the original triangle
    fv = oracle.face_copies(v, f, True)
    lit = oracle.lights(fv, 0.25, 0.5, (1, 1, 1), (1, 1, 1), (0, 0, -1))
    n = np.cross((fv[0, 0, 0] - fv[0, 0, 1]).astype(np.float64), (fv[0, 0, 2] - fv[0, 0, 1]).astype(np.float64))
    n /= np.linalg.norm(n)
    assert abs(n[2]) == pytest.approx(1.0)
    assert np.allclose(lit[0, 0], 0.25 + 0.5 * max(-n[2], 0.0), atol=1e-7)
    assert np.allclose(lit[0, 1], 0.25 + 0.5 * max(n[2], 0.0), atol=1e-7)
    assert not np.allclose(lit[0, 0], lit[0, 1])
    # at original vertex 0 the back copy samples the corner of axis 0 of the ORIGINAL cube (its own axis 2, transposed)
    assert out["face_index"][0, 2, 2] == 1
    frac = f32(T - 1) - f32(1e-3) - f32(T - 2)
    expect = lit[0, 1] * ((f32(1) - frac) * tex[0, 0, T - 2, 0, 0] + frac * tex[0, 0, T - 1, 0, 0])
    got = out["rgb"][0, :, S - 1 - 2, 2]
    assert np.allclose(got, expect, rtol=1e-5), (got, expect)


def test_a_pixel_at_a_vertex_samples_that_vertex_corner_texel():
    S, p0, p1, p2 = _vertex_pixel_scene()
    T = 4
    tex = np.random.default_rng(1).uniform(0.1, 1.0, size=(1, 1, T, T, T, 3)).astype(f32)
    frac = f32(T - 1) - f32(1e-3) - f32(T - 2)
    for k, order in enumerate([(p0, p1, p2), (p2, p0, p1), (p1, p2, p0)]):  # the pixel's vertex in slot k
        v, f = tri(*order)
        out = oracle.render(v, f, tex, image_size=S, anti_aliasing=False, fill_back=False, eye_z=EYE,
                            light_intensity_ambient=1.0, light_intensity_directional=0.0)
        assert out["face_index"][0, 2, 2] == 0
        lo, hi = [0, 0, 0], [0, 0, 0]
        lo[k], hi[k] = T - 2, T - 1
        expect = (f32(1) - frac) * tex[0, 0][tuple(lo)] + frac * tex[0, 0][tuple(hi)]
        assert np.allclose(out["rgb"][0, :, S - 1 - 2, 2], expect, rtol=1e-5)


def test_two_sided_light_matches_its_closed_form():
    rng = np.random.default_rng(2)
    v = rng.normal(size=(2, 30, 3)).astype(f32)
    f = np.stack([rng.permutation(30)[:3] for _ in range(40)])[None].repeat(2, 0).astype(np.int32)
    d = np.array([0.3, 1.0, -1.0], f32)
    Ia, Id = f32(0.8), f32(0.4)
    ca, cd = np.array([1.0, 0.9, 0.8], f32), np.array([0.7, 1.0, 0.5], f32)
    lit = oracle.lights(oracle.face_copies(v, f, True), Ia, Id, ca, cd, d)
    fv = v[np.arange(2)[:, None, None], f].astype(np.float64)
    n = np.cross(fv[:, :, 0] - fv[:, :, 1], fv[:, :, 2] - fv[:, :, 1])
    n /= np.maximum(np.linalg.norm(n, axis=-1, keepdims=True), 1e-5)
    cos = n @ d.astype(np.float64)
    front = Ia * ca + Id * cd * np.maximum(cos, 0)[..., None]
    back = Ia * ca + Id * cd * np.maximum(-cos, 0)[..., None]
    assert np.allclose(lit[:, :40], front, atol=2e-6) and np.allclose(lit[:, 40:], back, atol=2e-6)
    # the reversed copy's normal is exactly -n, so its light is bit-exactly the closed form on the same float32 dot
    lit1 = oracle.lights(oracle.face_copies(v, f, False), Ia, Id, ca, cd, -d)
    assert np.array_equal(lit[:, 40:], lit1)


def _scene(B=2, subdiv=1, seed=0, soup=0):
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(subdiv)
    verts = synth.bird_like(v, rng, B).astype(np.float64) * 0.8
    verts[..., 2] += 5.0
    verts[..., 1] *= -1
    faces = np.repeat(f[None], B, 0)
    if soup:  # open triangles in both orientations: the fill_back copies are drawn
        sv = rng.uniform(-0.9, 0.9, size=(B, 3 * soup, 3))
        sv[..., 2] = rng.uniform(3.5, 4.5, size=(B, 3 * soup))
        verts = np.concatenate([verts, sv], 1)
        sf = (v.shape[0] + np.arange(3 * soup).reshape(soup, 3))[None].repeat(B, 0)
        faces = np.concatenate([faces, sf], 1)
    return verts.astype(f32), faces.astype(np.int32)


def test_bounding_regions_match_the_exhaustive_z_buffer():
    v, f = _scene(B=1, subdiv=1, soup=6)
    # add a sliver and a degenerate face
    v = np.concatenate([v, np.array([[[-0.9, 0.1, 4.0], [0.9, 0.1001, 4.0], [0.95, 0.1002, 4.0],
                                      [-0.5, -0.5, 4.0], [0.5, -0.5, 4.0], [0.0, -0.5, 4.0]]], f32)], 1)
    n = v.shape[1]
    f = np.concatenate([f, np.array([[[n - 6, n - 5, n - 4], [n - 3, n - 2, n - 1]]], np.int32)], 1)
    for aa in (False, True):
        a = oracle.zbuffer(v, f, 24, aa, True, EYE)
        b = oracle.zbuffer(v, f, 24, aa, True, EYE, exhaustive=True)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        assert (a[0] >= f.shape[1]).any()  # back copies win somewhere


@pytest.mark.parametrize("aa,fill_back,G", [(True, True, 1), (False, True, 2), (True, False, 1)])
def test_texture_gradient_is_the_adjoint_of_the_render(aa, fill_back, G):
    B, T, IS = 2, 3, 16
    v, f = _scene(B=B, subdiv=1, soup=5)
    rng = np.random.default_rng(3)
    tex = rng.uniform(0, 1, size=(B // G, f.shape[1], T, T, T, 3))
    dt = rng.normal(size=tex.shape)
    g = rng.normal(size=(B, 3, IS, IS))
    light = dict(Ia=0.6, Id=0.5, ca=(1, 0.9, 0.8), cd=(0.5, 1, 1), direction=(0.2, 1, -1))
    zb = oracle.zbuffer(v, f, IS, aa, fill_back, EYE)
    kw = dict(anti_aliasing=aa, fill_back=fill_back, eye_z=EYE, shared_textures=G, **light)
    grad = oracle.grad_textures(g, v, f, tex.shape, zb, **kw)
    lhs = np.sum(grad * dt)
    d = oracle.render_rgb_linear(tex + dt, v, f, IS, zb, **kw) - oracle.render_rgb_linear(tex, v, f, IS, zb, **kw)
    rhs = np.sum(g * d)
    assert abs(lhs) > 1.0
    assert lhs == pytest.approx(rhs, rel=1e-12, abs=1e-12)
    if fill_back:
        F = f.shape[1]
        assert (zb[0] >= F).any()
    # the float32 render is the same linear map plus the background, up to float32 rounding
    out = oracle.render(v, f, tex.astype(f32), IS, aa, fill_back, EYE, near=0.1, far=100.0,
                        light_intensity_ambient=0.6, light_intensity_directional=0.5, light_color_ambient=(1, 0.9, 0.8),
                        light_color_directional=(0.5, 1, 1), light_direction=(0.2, 1, -1), background_color=(0, 0, 0),
                        shared_textures=G, zbuf=zb)
    lin = oracle.render_rgb_linear(tex.astype(f32), v, f, IS, zb, **kw)
    assert np.allclose(out["rgb"], lin, atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------------
# host side of umr_b200.neural_renderer
# ---------------------------------------------------------------------------------------------------------------------
def _nmr_pytorch_renderer():
    """nnutils/nmr_pytorch.py:42 (NMR.__init__ as NeuralRenderer calls it, :92) and the attribute writes of
    :95 (eye), :98 (ambient), :105-108 (ambient_light_only), :110-111 (set_bgcolor), :113-117 (set_light_dir)."""
    from umr_b200 import compat
    compat.install()
    import neural_renderer
    r = neural_renderer.Renderer(image_size=64, anti_aliasing=True, camera_mode="look_at", perspective=False,
                                 background_color=[0, 0, 0])
    r.eye = [0, 0, -2.732]
    r.light_intensity_ambient = 0.8
    r.light_intensity_ambient = 1
    r.light_intensity_directional = 0
    r.background_color = [1, 1, 1]
    r.light_direction = [0, 1, -1]
    r.light_intensity_directional = 0.4
    r.light_intensity_ambient = 0.8
    return r


def test_compat_install_registers_our_neural_renderer():
    import sys
    from umr_b200 import neural_renderer as ours
    r = _nmr_pytorch_renderer()
    assert sys.modules["neural_renderer"] is ours and isinstance(r, ours.Renderer)
    p = r._params(2, 10, 4, 6, 1)
    assert (p.eye_z, p.light_intensity_ambient, p.light_intensity_directional) == (f32(-2.732), f32(0.8), f32(0.4))
    assert list(p.light_direction) == [0, 1, -1] and list(p.background_color) == [1, 1, 1]
    # NMR's look_at default eye
    d = ours.Renderer(camera_mode="look_at", perspective=False)
    assert d.eye[:2] == [0, 0] and d.eye[2] == pytest.approx(-(1 / np.tan(np.radians(30)) + 1))


def test_install_without_neural_renderer_registers_nothing(monkeypatch):
    import sys
    from umr_b200 import compat
    monkeypatch.delitem(sys.modules, "neural_renderer", raising=False)
    compat.install(stub_neural_renderer=False)
    assert "neural_renderer" not in sys.modules


def test_refusals():
    from umr_b200.neural_renderer import Renderer
    with pytest.raises(NotImplementedError, match="camera_mode"):
        Renderer()
    with pytest.raises(NotImplementedError, match="perspective"):
        Renderer(camera_mode="look_at")
    r = Renderer(image_size=8, camera_mode="look_at", perspective=False)
    v = torch.zeros(1, 3, 3)
    f = torch.tensor([[[0, 1, 2]]], dtype=torch.int32)
    r.eye = [0.1, 0, -2.7]
    with pytest.raises(NotImplementedError, match="eye"):
        r.render_silhouettes(v, f)
    r.eye = [0, 0, -2.7]
    r.perspective = True
    with pytest.raises(NotImplementedError, match="perspective"):
        r.render_silhouettes(v, f)
    r.perspective = False
    with pytest.raises(NotImplementedError, match="T >= 2"):
        r.render_rgb(v, f, torch.zeros(1, 1, 1, 1, 1, 3))
    vg = torch.zeros(1, 3, 3, requires_grad=True)
    with pytest.raises(NotImplementedError, match="vertex / camera gradient.*train_s2.py:246"):
        r.render_silhouettes(vg, f)
    with pytest.raises(TypeError, match="cuda"):   # no CPU path
        r.render_silhouettes(v, f)
    with pytest.raises(TypeError, match="cuda"):
        with torch.no_grad():
            r.render_rgb(vg, f, torch.zeros(1, 1, 2, 2, 2, 3))


def test_multi_texture_loss_builds_the_nmr_renderer():
    from umr_b200.neural_renderer import Renderer
    from umr_b200.nnutils import loss_utils
    m = loss_utils.MultiTextureLoss(image_size=32, texture_loss_type="l1", renderer="nmr")
    r = m.renderer.renderer
    assert isinstance(r, Renderer) and r.image_size == 32 and r.anti_aliasing
    assert (r.light_intensity_ambient, r.light_intensity_directional) == (1, 0) and r.eye == [0, 0, -2.732]
    assert isinstance(loss_utils.MultiTextureLoss(texture_loss_type="l1").renderer, loss_utils.SoftRenderer)
