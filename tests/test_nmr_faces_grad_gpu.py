"""The functional NMR rasterisers on the GPU (DESIGN.md §14): the geometry gradient against the oracle
(tests/nmr_faces_oracle.py) within the float32 summation bound, forward planes bitwise `Renderer`'s, the texture
gradient `Renderer`'s, reproducibility, autograd from vertices, and silhouette / depth fitting."""
import ctypes
import importlib

import numpy as np
import pytest
import torch

import nmr_faces_oracle as oracle
import nmr_scenes as sc
from umr_b200 import _lib, synth
from umr_b200 import neural_renderer as nr

nr_mod = importlib.import_module("umr_b200.neural_renderer.rasterize")   # the module; nr.rasterize is the function
from umr_b200.raster import _ptr, _stream_ptr

pytestmark = pytest.mark.gpu
f32 = np.float32
DEV = "cuda"
GUARD = 12345.0


def gamma(n):
    u = 2.0 ** -24
    return n * u / (1 - n * u)


def scene_faces(B=2, seed=0, soup=4, subdiv=1):
    """A lumpy closed sphere plus open triangles of both orientations, as face coordinates [B,F,3,3]."""
    v, f = sc.mesh(B=B, subdiv=subdiv, seed=seed, soup=soup)
    return np.take_along_axis(v[:, None], f[..., None].astype(np.int64), axis=2).astype(f32)


def special_faces(S):
    """Vertical and horizontal edges, vertices on pixel centres, a back-facing face, faces cut by near / far."""
    c = lambda i: sc.centre(i, S)  # noqa: E731
    return np.array([
        [[c(1), c(1), 5.0], [c(S // 2), c(1), 5.0], [c(1), c(S // 2), 5.0]],              # axis-aligned, on centres
        [[c(S - 2), c(S - 2), 4.0], [c(S // 3), c(S - 2), 4.5], [c(S - 2), c(S // 3), 5.0]],  # back-facing (CW)
        [[-0.7, 0.1, 0.05], [0.3, 0.2, 0.3], [-0.2, 0.9, 0.2]],                           # cut by near = 0.1
        [[0.1, -0.8, 90.0], [0.9, -0.7, 120.0], [0.5, -0.1, 95.0]],                       # cut by far = 100
        [[-0.95, -0.9, 3.0], [-0.3, -0.9, 3.5], [-0.6, -0.35, 3.2]],
    ], f32)


def textures_for(B, F, T=3, seed=1):
    return np.random.default_rng(seed).uniform(0.05, 1.0, size=(B, F, T, T, T, 3)).astype(f32)


def call_backward(faces, tex, grads, IS, aa, eps=1e-4, near=0.1, far=100.0, bg=(0, 0, 0)):
    """Forward + umr_nmr_backward_faces through the C ABI, output prefilled with a guard value."""
    lib = _lib.load()
    B, F = faces.shape[:2]
    T = 0 if tex is None else tex.shape[2]
    fv = torch.from_numpy(faces).to(DEV)
    tx = None if tex is None else torch.from_numpy(tex).to(DEV)
    p = nr_mod._params(B, F, T, IS, aa, near, far, list(bg))
    S = IS * (2 if aa else 1)
    verts = fv.reshape(B, 3 * F, 3).contiguous()
    index = torch.arange(3 * F, device=DEV, dtype=torch.int32).reshape(1, F, 3).expand(B, F, 3).contiguous()
    ws = torch.empty(lib.umr_nmr_workspace_bytes(B, F, 0), device=DEV, dtype=torch.uint8)
    fidx = torch.empty(B, S, S, device=DEV, dtype=torch.int32)
    rdepth = torch.empty(B, S, S, device=DEV, dtype=torch.float32)
    _lib.check(lib.umr_nmr_forward(_ptr(verts), _ptr(index), _ptr(tx), _ptr(fidx), _ptr(rdepth), None, None, None,
                                   ctypes.byref(p), _ptr(ws), _stream_ptr(fv.device)), "forward")
    g = [None if a is None else torch.from_numpy(np.ascontiguousarray(a, f32)).to(DEV) for a in grads]
    out = torch.full((B, F, 3, 3), GUARD, device=DEV)
    ws2 = torch.empty(lib.umr_nmr_backward_faces_workspace_bytes(B, F, IS, int(aa)), device=DEV, dtype=torch.uint8)
    _lib.check(lib.umr_nmr_backward_faces(_ptr(verts), _ptr(index), _ptr(fidx), _ptr(tx), _ptr(g[0]), _ptr(g[1]),
                                          _ptr(g[2]), _ptr(out), ctypes.byref(p), eps, _ptr(ws2),
                                          _stream_ptr(fv.device)), "backward_faces")
    torch.cuda.synchronize()
    return out.cpu().numpy(), fidx.cpu().numpy(), rdepth.cpu().numpy()


def check_against_oracle(faces, tex, grads, IS, aa, eps=1e-4, near=0.1, far=100.0, bg=(0, 0, 0)):
    got, fidx, rdepth = call_backward(faces, tex, grads, IS, aa, eps, near, far, bg)
    zb = oracle.zbuffer(faces, IS, aa, near, far)
    assert np.array_equal(fidx, zb[0])
    ref, mag, cnt = oracle.grad_faces(faces, tex, *grads, image_size=IS, anti_aliasing=aa, near=near, far=far,
                                      eps=eps, background_color=bg, zbuf=zb, magnitude=True)
    assert not (got == GUARD).any(), "unwritten gradient elements"
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(got), fin)
    assert np.array_equal(got[~fin], ref[~fin].astype(f32), equal_nan=True)
    bound = np.vectorize(gamma)(cnt + 1) * mag
    err = np.abs(got.astype(np.float64) - ref)
    assert (err[fin] <= bound[fin]).all(), "max excess %g" % (err - bound)[fin].max()
    return got, ref, cnt


def adjoints(rng, B, IS, which, kind="mixed"):
    def plane(*shape):
        if kind == "zero":
            return np.zeros(shape, f32)
        return rng.uniform(-1, 1, size=shape).astype(f32)
    return (plane(B, 3, IS, IS) if "rgb" in which else None, plane(B, IS, IS) if "alpha" in which else None,
            plane(B, IS, IS) if "depth" in which else None)


WHICH = {"rgb": ("rgb",), "alpha": ("alpha",), "depth": ("depth",), "all": ("rgb", "alpha", "depth")}


@pytest.mark.parametrize("which", sorted(WHICH))
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("IS", [1, 2, 63, 65])
def test_grad_faces_matches_the_oracle(which, aa, IS):
    rng = np.random.default_rng(IS * 7 + aa)
    S = IS * (2 if aa else 1)
    faces = np.concatenate([scene_faces(B=2, subdiv=0), np.repeat(special_faces(max(S, 4))[None], 2, 0)], 1)
    tex = textures_for(2, faces.shape[1])
    got, ref, cnt = check_against_oracle(faces, tex, adjoints(rng, 2, IS, WHICH[which]), IS, aa, bg=(0.2, 0.5, 0.9))
    if IS >= 63:
        assert cnt.sum() > 0 and np.abs(ref).sum() > 0


@pytest.mark.parametrize("which", sorted(WHICH))
def test_grad_faces_at_256(which):
    rng = np.random.default_rng(5)
    faces = scene_faces(B=1, subdiv=0, soup=2)
    check_against_oracle(faces, textures_for(1, faces.shape[1]), adjoints(rng, 1, 256, WHICH[which]), 256, True)


@pytest.mark.parametrize("kind", ["zero", "mixed"])
def test_grad_faces_zero_and_mixed_sign_adjoints(kind):
    rng = np.random.default_rng(3)
    faces = scene_faces(B=2, subdiv=1)
    got, ref, _ = check_against_oracle(faces, textures_for(2, faces.shape[1]),
                                       adjoints(rng, 2, 32, WHICH["all"], kind), 32, True)
    if kind == "zero":
        assert (got == 0).all()


def test_grad_faces_huge_and_non_finite_coordinates():
    faces = np.repeat(special_faces(64)[None], 2, 0)
    faces[0, 0, 0, 0] = 1e6
    faces[0, 4, 1, 1] = -1e6
    faces[1, 0, 2, 0] = np.nan
    faces[1, 4, 0, 2] = np.inf
    faces[1, 2, 1, 1] = -np.inf
    rng = np.random.default_rng(4)
    got, ref, _ = check_against_oracle(faces, textures_for(2, 5), adjoints(rng, 2, 32, WHICH["all"]), 32, True)
    assert (got[1, 0] == 0).all() and (got[1, 2] == 0).all()   # hidden: no edge term, never wins a pixel


def test_forward_planes_are_renderers():
    """rasterize_rgbad == Renderer.render bit for bit on equivalent inputs: fill_back off, ambient light 1, and the
    face z already translated by -eye_z in float32."""
    rng = np.random.default_rng(0)
    v, f = sc.mesh(B=2, subdiv=2, seed=2)
    T = 4
    tex = torch.from_numpy(rng.uniform(0, 1, size=(2, f.shape[1], T, T, T, 3)).astype(f32)).to(DEV)
    verts, fcs = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)
    for aa, IS in ((True, 64), (False, 65)):
        r = nr.Renderer(image_size=IS, anti_aliasing=aa, background_color=[0.1, 0.2, 0.3], fill_back=False,
                        camera_mode="look_at", perspective=False, light_intensity_ambient=1.0,
                        light_intensity_directional=0.0)
        rgb, depth, alpha = r.render(verts, fcs, tex)
        fv = nr.vertices_to_faces(verts, fcs).clone()
        fv[..., 2] = fv[..., 2] - torch.tensor(r.eye[2], dtype=torch.float32)
        out = nr.rasterize_rgbad(fv, tex, IS, aa, background_color=[0.1, 0.2, 0.3])
        for a, b in ((out["rgb"], rgb), (out["alpha"], alpha), (out["depth"], depth)):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        assert torch.equal(nr.rasterize(fv, tex, IS, aa, background_color=[0.1, 0.2, 0.3]), rgb)
        assert torch.equal(nr.rasterize_silhouettes(fv, IS, aa), alpha)
        assert torch.equal(nr.rasterize_depth(fv, IS, aa), depth)


@pytest.mark.parametrize("det", [False, True])
def test_texture_gradient_is_renderers(det):
    rng = np.random.default_rng(1)
    v, f = sc.mesh(B=2, subdiv=1, seed=3)
    T, IS = 3, 48
    tex0 = rng.uniform(0, 1, size=(2, f.shape[1], T, T, T, 3)).astype(f32)
    gr = torch.from_numpy(rng.uniform(-1, 1, size=(2, 3, IS, IS)).astype(f32)).to(DEV)
    verts, fcs = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)
    r = nr.Renderer(image_size=IS, fill_back=False, camera_mode="look_at", perspective=False,
                    light_intensity_ambient=1.0, light_intensity_directional=0.0)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        t1 = torch.from_numpy(tex0).to(DEV).requires_grad_(True)
        (r.render_rgb(verts, fcs, t1) * gr).sum().backward()
        fv = nr.vertices_to_faces(verts, fcs).clone()
        fv[..., 2] = fv[..., 2] - torch.tensor(r.eye[2], dtype=torch.float32)
        t2 = torch.from_numpy(tex0).to(DEV).requires_grad_(True)
        (nr.rasterize(fv, t2, IS) * gr).sum().backward()
    finally:
        torch.use_deterministic_algorithms(prev)
    if det:
        assert torch.equal(t1.grad, t2.grad)
    else:
        torch.testing.assert_close(t2.grad, t1.grad, rtol=1e-5, atol=1e-6)


def test_grad_faces_is_bitwise_reproducible():
    rng = np.random.default_rng(6)
    faces = scene_faces(B=2, subdiv=2)
    fv = torch.from_numpy(faces).to(DEV)
    tex = torch.from_numpy(textures_for(2, faces.shape[1])).to(DEV)
    ga = [torch.from_numpy(a).to(DEV) for a in adjoints(rng, 2, 64, WHICH["all"])]
    grads = []
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        for det in (False, True, False, True):
            torch.use_deterministic_algorithms(det)
            x = fv.clone().requires_grad_(True)
            out = nr.rasterize_rgbad(x, tex, 64)
            torch.autograd.backward([out["rgb"], out["alpha"], out["depth"]], ga)
            grads.append(x.grad)
    finally:
        torch.use_deterministic_algorithms(prev)
    for g in grads[1:]:
        assert torch.equal(g, grads[0])


def test_autograd_from_vertices_matches_the_oracle():
    """vertices_to_faces -> rasterize_rgbad -> loss: the vertex gradient is the face gradient gathered back, in the
    input dtype (float64 renders in float32)."""
    rng = np.random.default_rng(8)
    v, f = sc.mesh(B=2, subdiv=1, seed=4)
    IS = 32
    tex = textures_for(2, f.shape[1])
    gr, ga, gd = adjoints(rng, 2, IS, WHICH["all"])
    for dtype in (torch.float32, torch.float64):
        verts = torch.from_numpy(v).to(DEV, dtype).requires_grad_(True)
        t = torch.from_numpy(tex).to(DEV, dtype).requires_grad_(True)
        fv = nr.vertices_to_faces(verts, torch.from_numpy(f).to(DEV))
        out = nr.rasterize_rgbad(fv, t, IS)
        loss = (out["rgb"] * torch.from_numpy(gr).to(DEV, dtype)).sum() + \
            (out["alpha"] * torch.from_numpy(ga).to(DEV, dtype)).sum() + (out["depth"] * torch.from_numpy(gd).to(DEV, dtype)).sum()
        loss.backward()
        assert verts.grad.dtype == dtype and t.grad.dtype == dtype
        faces = np.take_along_axis(v[:, None], f[..., None].astype(np.int64), axis=2).astype(f32)
        ref, mag, cnt = oracle.grad_faces(faces, tex, gr, ga, gd, image_size=IS, magnitude=True)
        want = np.zeros(v.shape)
        bound = np.zeros(v.shape)
        for b in range(2):
            np.add.at(want[b], f[b], ref[b])
            np.add.at(bound[b], f[b], (np.vectorize(gamma)(cnt[b] + 4) * mag[b]))
        err = np.abs(verts.grad.double().cpu().numpy() - want)
        assert (err <= bound + 1e-30).all()


def test_grad_faces_launches():
    lib = _lib.load()
    faces = scene_faces(B=1, subdiv=1)
    rng = np.random.default_rng(2)
    n0 = lib.umr_launch_count()
    call_backward(faces, textures_for(1, faces.shape[1]), adjoints(rng, 1, 32, WHICH["all"]), 32, True)
    assert lib.umr_launch_count() - n0 == 2 + 3   # forward: prep, zbuf; backward: prep, shade_raster, grad_faces
    n0 = lib.umr_launch_count()
    call_backward(faces, None, adjoints(rng, 1, 32, ("alpha",)), 32, True)
    assert lib.umr_launch_count() - n0 == 2 + 2


def _iou(a, b):
    inter = (a * b).sum()
    return float(inter / (a + b - a * b).sum())


def _sphere(dev, subdiv=2, scale=0.5, z=5.0):
    v, f = synth.icosphere(subdiv)
    v = torch.from_numpy(v.astype(f32)).to(dev) * scale
    v[:, 2] += z
    return v[None], torch.from_numpy(f.astype(np.int64)).to(dev)[None]


def test_silhouette_fitting_lowers_one_minus_iou():
    """100 Adam steps on an icosphere's vertices against an ellipse-like target silhouette."""
    torch.manual_seed(0)
    IS = 64
    v0, f = _sphere(DEV)
    target_v = v0.clone()
    target_v[..., 0] *= 1.5
    target_v[..., 1] *= 0.8
    target = nr.rasterize_silhouettes(nr.vertices_to_faces(target_v, f), IS).detach()
    verts = v0.clone().requires_grad_(True)
    opt = torch.optim.Adam([verts], lr=0.005)
    hist = []
    for _ in range(100):
        opt.zero_grad()
        a = nr.rasterize_silhouettes(nr.vertices_to_faces(verts, f), IS)
        loss = 1 - (a * target).sum() / (a + target - a * target).sum()
        hist.append(float(loss.detach()))
        loss.backward()
        opt.step()
    final = 1 - _iou(nr.rasterize_silhouettes(nr.vertices_to_faces(verts, f), IS).detach(), target)
    assert np.mean(hist[:10]) > np.mean(hist[45:55]) > np.mean(hist[-10:])
    assert hist[0] > 0.1 and final < 0.05, (hist[0], final)


def test_depth_fitting_lowers_the_depth_error():
    """100 Adam steps on the icosphere's vertex depths against a target depth map (the sphere moved 0.3 nearer and
    flattened).  Only z is fitted: the depth map has no gradient where no face is drawn, so x / y steps that uncover
    a pixel could not be undone through it."""
    torch.manual_seed(0)
    IS = 64
    v0, f = _sphere(DEV)
    target_v = v0.clone()
    target_v[..., 2] = (target_v[..., 2] - 5.0) * 0.6 + 4.7
    target = nr.rasterize_depth(nr.vertices_to_faces(target_v, f), IS).detach()
    mask = nr.rasterize_silhouettes(nr.vertices_to_faces(target_v, f), IS).detach() == 1
    z = v0[..., 2:].clone().requires_grad_(True)
    opt = torch.optim.Adam([z], lr=0.005)
    hist = []
    for _ in range(100):
        opt.zero_grad()
        d = nr.rasterize_depth(nr.vertices_to_faces(torch.cat([v0[..., :2], z], -1), f), IS)
        loss = ((d - target)[mask] ** 2).mean()
        hist.append(float(loss.detach()))
        loss.backward()
        opt.step()
    assert np.mean(hist[:10]) > np.mean(hist[45:55]) > np.mean(hist[-10:])
    assert hist[-1] < 0.05 * hist[0], (hist[0], hist[-1])
