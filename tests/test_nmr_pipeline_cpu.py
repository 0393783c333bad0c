"""neural_renderer's camera, lighting and OBJ functions without a GPU (DESIGN.md §15): the cameras against float64
closed forms, the OBJ round trip, `lighting`'s argument validation, dtype rules, C entry-point refusals and workspace
formula, and the numpy oracle (tests/nmr_light_oracle.py) against torch autograd of the upstream formula."""
import ctypes
import importlib
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as tF

import nmr_light_oracle as oracle
from umr_b200 import _lib
from umr_b200 import neural_renderer as nr

lt = importlib.import_module("umr_b200.neural_renderer.lighting")   # the module; nr.lighting is the function


def test_exports():
    for name in ("look_at", "look", "perspective", "projection", "get_points_from_angles", "lighting", "load_obj",
                 "save_obj"):
        assert name in nr.__all__ and callable(getattr(nr, name))


# ----------------------------------------------------------------------------------------------------------------
# cameras
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("eye,at,up", [((0.3, 1.2, -2.5), (0, 0, 0), (0, 1, 0)), ((4.0, -1.0, 0.5), (0.2, 0.1, -0.3),
                                                                                     (0.1, 1.0, 0.2))])
def test_look_at_frame(eye, at, up):
    eye_, at_ = np.asarray(eye, np.float64), np.asarray(at, np.float64)
    pts = torch.tensor(np.stack([eye_, at_, eye_ + [1, 0, 0], eye_ + [0, 1, 0], eye_ + [0, 0, 1]])[None])
    out = nr.look_at(pts, eye, at, up)[0].numpy()
    assert np.abs(out[0]).max() < 1e-12                                   # eye -> origin
    assert np.allclose(out[1], [0, 0, np.linalg.norm(at_ - eye_)], atol=1e-12)   # at on +z
    R = out[2:5].T                                                        # columns: images of the unit axes
    assert np.allclose(R @ R.T, np.eye(3), atol=1e-12) and np.isclose(np.linalg.det(R), 1.0)
    # the camera's x axis is perpendicular to up
    assert abs(R[0] @ np.asarray(up, np.float64)) < 1e-12


def test_look_defaults_and_identity():
    v = torch.randn(2, 7, 3, dtype=torch.float64)
    got = nr.look(v, (0.0, 0.0, -3.0), direction=(0, 0, 1))
    assert torch.allclose(got, v - torch.tensor([0.0, 0.0, -3.0], dtype=torch.float64), atol=1e-12)
    assert torch.equal(nr.look(v, (1, 2, 3), (0.3, 0.2, 1.0), None), nr.look(v, (1, 2, 3), (0.3, 0.2, 1.0), (0, 1, 0)))


def test_look_at_gradient_reaches_eye():
    v = torch.randn(2, 5, 3, dtype=torch.float64, requires_grad=True)
    eye = torch.tensor([[0.3, 0.4, -2.0], [1.0, 0.5, 2.0]], dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda a, e: nr.look_at(a, e), (v, eye))


@pytest.mark.parametrize("angle", [30.0, 15.0, 60])
def test_perspective(angle):
    rng = np.random.default_rng(int(angle))
    v = rng.uniform(-1, 1, (2, 9, 3)) + [0, 0, 4]
    got = nr.perspective(torch.tensor(v), angle).numpy()
    w = math.tan(math.radians(angle))
    ref = np.stack([v[..., 0] / v[..., 2] / w, v[..., 1] / v[..., 2] / w, v[..., 2]], -1)
    assert np.allclose(got, ref, rtol=1e-6)                               # the tangent is a float32's
    # NMR's definition, bit for bit: x / z / tan(float32(angle in radians))
    w32 = torch.tan(torch.tensor(angle / 180 * math.pi, dtype=torch.float32))
    v32 = torch.tensor(v, dtype=torch.float32)
    assert torch.equal(nr.perspective(v32, angle)[..., 0], v32[..., 0] / v32[..., 2] / w32)
    # soft_renderer keeps its own (double-precision tangent)
    from umr_b200.soft_renderer.functional import geometry
    assert torch.equal(geometry.perspective(v32, angle)[..., 1], v32[..., 1] / v32[..., 2] / math.tan(math.radians(angle)))


def _projection_ref(v, K, R, t, dist, orig_size, eps=1e-9):
    c = np.einsum("bij,bvj->bvi", R, v) + t
    x, y, z = c[..., 0], c[..., 1], c[..., 2]
    xn, yn = x / (z + eps), y / (z + eps)
    k1, k2, p1, p2, k3 = (dist[:, i, None] for i in range(5))
    r2 = xn ** 2 + yn ** 2
    rad = 1 + k1 * r2 + k2 * r2 ** 2 + k3 * r2 ** 3
    xd = xn * rad + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn ** 2)
    yd = yn * rad + p1 * (r2 + 2 * yn ** 2) + 2 * p2 * xn * yn
    uvw = np.einsum("bij,bvj->bvi", K, np.stack([xd, yd, np.ones_like(z)], -1))
    u, vv = uvw[..., 0], orig_size - uvw[..., 1]
    return np.stack([2 * (u - orig_size / 2) / orig_size, 2 * (vv - orig_size / 2) / orig_size, z], -1)


def _camera(B, rng):
    K = np.zeros((B, 3, 3))
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = 500, 480, 128, 120, 1
    ang = rng.uniform(-0.3, 0.3, (B, 3))
    R = np.stack([_rot(a) for a in ang])
    t = rng.uniform(-0.2, 0.2, (B, 1, 3)) + [0, 0, 5]
    dist = np.tile([0.1, -0.05, 0.01, -0.02, 0.003], (B, 1)) * rng.uniform(0.5, 1.5, (B, 1))
    return K, R, t, dist


def _rot(a):
    cx, sx, cy, sy, cz, sz = math.cos(a[0]), math.sin(a[0]), math.cos(a[1]), math.sin(a[1]), math.cos(a[2]), math.sin(a[2])
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def test_projection_with_distortion():
    rng = np.random.default_rng(4)
    B = 3
    v = rng.uniform(-1, 1, (B, 11, 3))
    K, R, t, dist = _camera(B, rng)
    got = nr.projection(*(torch.tensor(a) for a in (v, K, R, t, dist)), 256).numpy()
    assert np.allclose(got, _projection_ref(v, K, R, t, dist, 256), rtol=1e-12, atol=1e-12)
    assert np.abs(dist).min() > 0


def test_projection_gradients_reach_K_R_t():
    rng = np.random.default_rng(5)
    v = torch.tensor(rng.uniform(-1, 1, (2, 4, 3)), requires_grad=True)
    K, R, t, dist = (torch.tensor(a, requires_grad=True) for a in _camera(2, rng))
    assert torch.autograd.gradcheck(lambda *a: nr.projection(*a, 256), (v, K, R, t, dist))


def test_get_points_from_angles():
    d, el, az = 2.732, 30.0, 45.0
    x, y, z = nr.get_points_from_angles(d, el, az)
    e, a = math.radians(el), math.radians(az)
    assert np.allclose([x, y, z], [d * math.cos(e) * math.sin(a), d * math.sin(e), -d * math.cos(e) * math.cos(a)])
    assert np.allclose(nr.get_points_from_angles(d, e, a, degrees=False), [x, y, z])
    D = torch.tensor([2.0, 3.0], dtype=torch.float64)
    E_ = torch.tensor([10.0, -20.0], dtype=torch.float64)
    A = torch.tensor([0.0, 135.0], dtype=torch.float64)
    got = nr.get_points_from_angles(D, E_, A).numpy()
    er, ar = np.radians(E_.numpy()), np.radians(A.numpy())
    Dn = D.numpy()
    ref = np.stack([Dn * np.cos(er) * np.sin(ar), Dn * np.sin(er), -Dn * np.cos(er) * np.cos(ar)], 1)
    assert got.shape == (2, 3) and np.allclose(got, ref, atol=1e-12)
    assert np.allclose(np.linalg.norm(got, axis=1), D.numpy())


# ----------------------------------------------------------------------------------------------------------------
# OBJ
# ----------------------------------------------------------------------------------------------------------------
@pytest.fixture
def cpu_cuda(monkeypatch):
    """load_obj puts its tensors on the GPU; here they stay on the CPU."""
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)


OBJ = """# quad, pentagon and a triangle in every index form
v 0 0 0
v 2 0 0
v 2 1 0
v 0 1 0
v 1 2 3
v -1 0.5 1
vt 0 0
vt 1 0
vn 0 0 1
f 1 2 3 4
f 1/1 2/2 5/1 6/2 4/1
f 2//1 3//1 5//1
f 3/1/1 4/2/1 6/1/1
"""


def test_load_obj_fan_and_index_forms(tmp_path, cpu_cuda):
    fn = tmp_path / "m.obj"
    fn.write_text(OBJ)
    v, f = nr.load_obj(str(fn), normalization=False)
    assert v.dtype == torch.float32 and f.dtype == torch.int32
    assert v.shape == (6, 3) and f.tolist() == [[0, 1, 2], [0, 2, 3], [0, 1, 4], [0, 4, 5], [0, 5, 3], [1, 2, 4],
                                                [2, 3, 5]]


def test_load_obj_normalization(tmp_path, cpu_cuda):
    fn = tmp_path / "m.obj"
    fn.write_text(OBJ)
    raw, _ = nr.load_obj(str(fn), normalization=False)
    v, _ = nr.load_obj(str(fn))                                          # normalization=True is the default
    r = raw.double().numpy()
    ref = r - r.min(0)
    ref = ref / np.abs(ref).max() * 2
    ref = ref - ref.max(0) / 2
    assert np.allclose(v.numpy(), ref, atol=1e-6)
    ext = v.max(0)[0] - v.min(0)[0]
    assert abs(float(ext.max()) - 2.0) < 1e-6                              # longest side spans [-1, 1]
    assert torch.allclose(v.max(0)[0], -v.min(0)[0], atol=1e-6)           # centred
    assert float(v.abs().max()) <= 1.0 + 1e-6


def test_save_load_round_trip(tmp_path, cpu_cuda):
    rng = np.random.default_rng(0)
    v = torch.tensor(rng.uniform(-1, 1, (9, 3)), dtype=torch.float32)
    f = torch.tensor(rng.integers(0, 9, (12, 3)), dtype=torch.int32)
    fn = str(tmp_path / "out.obj")
    nr.save_obj(fn, v, f)
    v2, f2 = nr.load_obj(fn, normalization=False)
    assert torch.equal(f2, f) and torch.allclose(v2, v, atol=1e-7)


def test_obj_texture_settings_are_refused(tmp_path):
    with pytest.raises(NotImplementedError, match="load_texture"):
        nr.load_obj(str(tmp_path / "x.obj"), load_texture=True)
    with pytest.raises(NotImplementedError, match="textures"):
        nr.save_obj(str(tmp_path / "x.obj"), torch.zeros(3, 3), torch.zeros(1, 3, dtype=torch.int32),
                    textures=torch.zeros(1, 2, 2, 2, 3))


# ----------------------------------------------------------------------------------------------------------------
# lighting: validation, dtypes, C ABI
# ----------------------------------------------------------------------------------------------------------------
def _args(B=2, F=3, T=2, dtype=torch.float32):
    return torch.zeros(B, F, 3, 3, dtype=dtype), torch.zeros(B, F, T, T, T, 3, dtype=dtype)


@pytest.mark.parametrize("bad", [
    dict(faces=torch.zeros(2, 3, 3)), dict(faces=torch.zeros(2, 3, 3, 2)), dict(faces=torch.zeros(2, 3, 3, 3,
                                                                                                  dtype=torch.int32)),
    dict(textures=torch.zeros(2, 3, 2, 2, 2)), dict(textures=torch.zeros(2, 4, 2, 2, 2, 3)),
    dict(textures=torch.zeros(2, 3, 2, 3, 2, 3)), dict(textures=torch.zeros(2, 3, 2, 2, 2, 4)),
    dict(color_ambient=(1, 1)), dict(color_directional=torch.ones(3, 3)), dict(direction=np.ones((2, 2))),
])
def test_lighting_argument_validation(bad):
    faces, tex = _args()
    kw = dict(faces=faces, textures=tex)
    kw.update(bad)
    with pytest.raises(ValueError):
        nr.lighting(**kw)


def test_lighting_refusals():
    faces, tex = _args()
    with pytest.raises(TypeError, match="cuda"):
        nr.lighting(faces, tex)
    with pytest.raises(NotImplementedError, match="intensity_ambient"):
        nr.lighting(faces, tex, intensity_ambient=torch.tensor(0.5, requires_grad=True))
    with pytest.raises(TypeError):
        nr.lighting(faces, tex, direction="up")


def test_lighting_dtype_rules():
    f32, f64, f16 = torch.float32, torch.float64, torch.float16
    cases = [((f32, f32), {}, f32), ((f16, f16), {}, f32), ((f64, f32), {}, f64), ((f32, f64), {}, f64),
             ((f32, f32), dict(color_ambient=torch.ones(3, dtype=f64)), f64),
             ((f32, f32), dict(direction=np.array([0.0, 1.0, 0.0])), f32),     # ndarrays become float32, as upstream
             ((f16, f32), dict(color_directional=torch.ones(2, 3, dtype=f16)), f32)]
    for (fd, td), kw, want in cases:
        faces, _ = _args(dtype=fd)
        _, tex = _args(dtype=td)
        ca, cd, d, p, dtype = lt._prepare(faces, tex, kw.pop("Ia", 0.5), 0.5, kw.get("color_ambient", (1, 1, 1)),
                                          kw.get("color_directional", (1, 1, 1)), kw.get("direction", (0, 1, 0)))
        assert dtype == want and p.dtype == (1 if want == f64 else 0)
    faces, tex = _args()
    _, _, _, p, _ = lt._prepare(faces, tex, 0.3, 0.7, torch.ones(2, 3), (1, 1, 1), torch.ones(2, 3))
    assert (p.color_ambient_bstride, p.color_directional_bstride, p.direction_bstride) == (3, 0, 3)
    assert (p.batch_size, p.num_faces, p.texture_res, p.reserved) == (2, 3, 2, 0)
    assert (p.intensity_ambient, p.intensity_directional) == (0.3, 0.7)


def test_lighting_int32_limit():
    faces = torch.zeros(1, 1, 3, 3).expand(2 ** 16, 1, 3, 3)
    tex = torch.zeros(1, 1, 1, 1, 1, 3).expand(2 ** 16, 1, 32, 32, 32, 3)
    with pytest.raises(ValueError, match="int32"):
        lt._prepare(faces, tex, 0.5, 0.5, (1, 1, 1), (1, 1, 1), (0, 1, 0))


def test_workspace_formula():
    lib = _lib.load()
    for B, F, dt, es in [(1, 1, 0, 4), (16, 1280, 0, 4), (3, 65537, 1, 8), (7, 33, 1, 8)]:
        n = 9 * B * F * es
        assert lib.umr_nmr_lighting_workspace_bytes(B, F, dt) == (n + 255) // 256 * 256
    for args in [(0, 5, 0), (5, 0, 0), (-1, 5, 0), (2, 5, 2), (2, 5, -1), (65536, 4096, 0)]:
        assert lib.umr_nmr_lighting_workspace_bytes(*args) == 0
    assert lib.umr_sizeof_nmr_light_params() == ctypes.sizeof(_lib.UmrNmrLightParams)


def _p(**kw):
    p = _lib.UmrNmrLightParams()
    p.batch_size, p.num_faces, p.texture_res, p.dtype = 2, 3, 2, 0
    p.intensity_ambient, p.intensity_directional = 0.5, 0.5
    for k, v in kw.items():
        setattr(p, k, v)
    return p


BAD, TOO_LARGE = -2, -3
A = 4096  # a fake device address: every call below is refused before it touches memory


@pytest.mark.parametrize("kw,code", [
    (dict(batch_size=0), BAD), (dict(num_faces=0), BAD), (dict(texture_res=0), BAD), (dict(dtype=2), BAD),
    (dict(reserved=1), BAD), (dict(color_ambient_bstride=1), BAD), (dict(direction_bstride=6), BAD),
    (dict(texture_res=1025), TOO_LARGE), (dict(batch_size=65536, num_faces=4096), TOO_LARGE),
    (dict(batch_size=2 ** 20, num_faces=2 ** 10, texture_res=1), TOO_LARGE),
])
def test_entry_point_refusals(kw, code):
    lib = _lib.load()
    launches = lib.umr_launch_count()
    p = _p(**kw)
    assert lib.umr_nmr_lighting_forward(A, A, A, A, A, A, ctypes.byref(p), None) == code
    assert lib.umr_nmr_lighting_backward(A, A, A, A, A, A, A, A, A, ctypes.byref(p), A * 2, None) == code
    assert lib.umr_launch_count() == launches   # a refused call launches nothing


def test_entry_point_buffer_refusals():
    lib = _lib.load()
    p = _p()
    fwd, bwd = lib.umr_nmr_lighting_forward, lib.umr_nmr_lighting_backward
    assert fwd(None, A, A, A, A, A, None, None) == BAD                   # NULL params
    for i in range(6):
        ptrs = [A] * 6
        ptrs[i] = 0
        assert fwd(*ptrs, ctypes.byref(p), None) == BAD                  # NULL buffer
        ptrs[i] = A + 2
        assert fwd(*ptrs, ctypes.byref(p), None) == BAD                  # not aligned to the element size
    p64 = _p(dtype=1)
    assert fwd(A + 4, A, A, A, A, A, ctypes.byref(p64), None) == BAD    # float64 wants 8-byte alignment
    for i in range(6):
        ptrs = [A] * 9
        ptrs[i] = 0
        assert bwd(*ptrs, ctypes.byref(p), A, None) == BAD
    assert bwd(A, A, A, A, A, A, None, None, None, ctypes.byref(p), A, None) == BAD    # no output
    assert bwd(A, A, A, A, A, A, A + 2, None, None, ctypes.byref(p), A, None) == BAD   # misaligned output
    assert bwd(A, A, A, A, A, A, None, None, A, ctypes.byref(p), None, None) == BAD    # grad_light, no workspace
    assert bwd(A, A, A, A, A, A, None, None, A, ctypes.byref(p), A + 16, None) == BAD  # misaligned workspace


# ----------------------------------------------------------------------------------------------------------------
# the oracle
# ----------------------------------------------------------------------------------------------------------------
def _torch_lighting(faces, tex, Ia, Id, ca, cd, d):
    """Upstream's formula, out of place, in torch float64."""
    B, F = faces.shape[:2]
    light = torch.zeros(B, F, 3, dtype=torch.float64)
    if Ia != 0:
        light = light + Ia * (ca if ca.dim() == 2 else ca[None])[:, None, :]
    if Id != 0:
        fv = faces.reshape(B * F, 3, 3)
        n = tF.normalize(torch.cross(fv[:, 0] - fv[:, 1], fv[:, 2] - fv[:, 1], dim=-1), eps=1e-5).reshape(B, F, 3)
        dd = (d if d.dim() == 2 else d[None])[:, None, :]
        cos = tF.relu((n * dd).sum(2))
        light = light + Id * ((cd if cd.dim() == 2 else cd[None])[:, None, :] * cos[:, :, None])
    return tex * light[:, :, None, None, None, :]


def random_scene(rng, B, F, T):
    faces = rng.uniform(-1, 1, (B, F, 3, 3))
    tex = rng.uniform(0, 1, (B, F, T, T, T, 3))
    return faces, tex


@pytest.mark.parametrize("Ia,Id,batched", [(0.5, 0.5, False), (0.3, 0.8, True), (0.0, 0.7, True), (0.6, 0.0, False)])
def test_oracle_matches_torch_autograd(Ia, Id, batched):
    rng = np.random.default_rng(7)
    B, F, T = 3, 17, 3
    faces, tex = random_scene(rng, B, F, T)
    faces[0, 0] = [[0, 0, 0], [0, 0, 0], [1, 1, 1]]                       # zero area: the eps branch
    faces[1, 1] = [[0, 0, 0], [1e-4, 0, 0], [0, 1e-4, 0]]                  # |cross| = 1e-8 < eps
    sh = (B, 3) if batched else (3,)
    ca, cd, d = rng.uniform(0.2, 1.0, sh), rng.uniform(0.2, 1.0, sh), rng.uniform(-1, 1, sh) + [0, 0.5, 0]
    g = rng.uniform(-1, 1, tex.shape)
    ts = [torch.tensor(a, requires_grad=True) for a in (faces, tex, ca, cd, d)]
    out = _torch_lighting(ts[0], ts[1], Ia, Id, *ts[2:])
    out.backward(torch.tensor(g))
    lit, _ = oracle.forward(faces, tex, Ia, Id, ca, cd, d, u=oracle.U64)
    assert np.allclose(lit.v, out.detach().numpy(), rtol=1e-13, atol=1e-15)
    gb = oracle.backward(faces, tex, g, Ia, Id, ca, cd, d, u=oracle.U64)
    # an input the formula does not reach (faces with Id = 0) has no .grad: its gradient is zero
    grad = lambda t: np.zeros(t.shape) if t.grad is None else t.grad.numpy()  # noqa: E731
    for key, t in (("grad_faces", ts[0]), ("grad_textures", ts[1])):
        assert np.allclose(gb[key].v, grad(t), rtol=1e-11, atol=1e-13), key
    for key, t in (("grad_ca", ts[2]), ("grad_cd", ts[3]), ("grad_dir", ts[4])):
        ref = gb[key] if batched else oracle.batch_sum(gb[key])
        assert np.allclose(ref.v, grad(t), rtol=1e-11, atol=1e-13), key
    if Id == 0:
        assert (gb["grad_faces"].v == 0).all()


def test_oracle_bound_covers_float32_rounding():
    """A float32 numpy restatement of the kernel's op order stays within the oracle's float32 bound."""
    rng = np.random.default_rng(8)
    faces, tex = random_scene(rng, 2, 64, 2)
    faces, tex = faces.astype(np.float32), tex.astype(np.float32)
    d = np.array([0.3, 0.9, -0.4], np.float32)
    lit, L = oracle.forward(faces, tex, 0.4, 0.6, (1, 1, 1), (0.9, 0.8, 0.7), d)
    assert not L["ambiguous"].any()
    f = faces
    a = f[:, :, 0] - f[:, :, 1]
    b = f[:, :, 2] - f[:, :, 1]
    c = np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                  a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)
    nrm = np.sqrt((c[..., 0] * c[..., 0] + c[..., 1] * c[..., 1]) + c[..., 2] * c[..., 2])
    n = c / np.maximum(nrm, np.float32(1e-5))[..., None]
    cs = np.maximum((n[..., 0] * d[0] + n[..., 1] * d[1]) + n[..., 2] * d[2], np.float32(0))
    cd = np.array([0.9, 0.8, 0.7], np.float32)
    light = np.float32(0.4) * np.float32(1) + np.float32(0.6) * (cd * cs[..., None])
    got = tex * light[:, :, None, None, None, :]
    assert got.dtype == np.float32
    assert (np.abs(got.astype(np.float64) - lit.v) <= lit.e).all()
