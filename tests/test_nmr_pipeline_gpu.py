"""neural_renderer's lighting kernels and functional pipeline on the GPU (DESIGN.md §15): values and every gradient
against the float64 oracle (tests/nmr_light_oracle.py) within its per-coordinate error bound, with guard bands round
every buffer; gradcheck; reproducibility and launch counts; the composed pipeline against `Renderer`; and two
NMR-example-shaped optimisations on synthetic meshes."""
import ctypes
import numpy as np
import pytest
import torch

import nmr_light_oracle as oracle
from umr_b200 import _lib, synth
from umr_b200 import neural_renderer as nr
from umr_b200.raster import _ptr, _stream_ptr

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 12345.0
PAD = 64   # guard elements either side (keeps 16-byte alignment; PAD + 1 skews it)

TD = {0: (torch.float32, np.float32, oracle.U32), 1: (torch.float64, np.float64, oracle.U64)}


def guarded(shape, dtype, skew=0, fill=GUARD):
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * PAD + 1,), fill, dtype=dtype, device=DEV)
    return buf, buf[PAD + skew:PAD + skew + n].view(shape)


def guards_intact(buf, n, skew=0):
    head, tail = buf[:PAD + skew], buf[PAD + skew + n:]
    return bool((head == GUARD).all()) and bool((tail == GUARD).all())


def call(faces, tex, g, Ia, Id, ca, cd, d, dt=0, skew=0, outputs=("faces", "tex", "light")):
    """Forward and backward through the C ABI with every buffer between guard bands."""
    lib = _lib.load()
    tdt, ndt, _ = TD[dt]
    B, F = faces.shape[:2]
    T = tex.shape[2]
    ins = {}
    bufs = []
    for name, a in (("faces", faces), ("tex", tex), ("ca", ca), ("cd", cd), ("d", d), ("g", g)):
        b, v = guarded(a.shape, tdt)
        v.copy_(torch.from_numpy(np.ascontiguousarray(a, ndt)))
        ins[name] = v
        bufs.append((b, v.numel(), 0))
    p = lib_params(B, F, T, dt, Ia, Id, ca, cd, d)
    lbuf, lit = guarded(tex.shape, tdt, skew)
    stream = _stream_ptr(torch.device(DEV))
    _lib.check(lib.umr_nmr_lighting_forward(_ptr(ins["faces"]), _ptr(ins["tex"]), _ptr(ins["ca"]), _ptr(ins["cd"]),
                                            _ptr(ins["d"]), _ptr(lit), ctypes.byref(p), stream), "forward")
    gf = gt = gl = ws = None
    outs = {}
    if "faces" in outputs:
        outs["faces"] = guarded(faces.shape, tdt, skew)
        gf = outs["faces"][1]
    if "tex" in outputs:
        outs["tex"] = guarded(tex.shape, tdt, skew)
        gt = outs["tex"][1]
    if "light" in outputs:
        outs["light"] = guarded((B, 9), tdt, skew)
        gl = outs["light"][1]
        ws = torch.full((lib.umr_nmr_lighting_workspace_bytes(B, F, dt),), 0x7f, dtype=torch.uint8, device=DEV)
    _lib.check(lib.umr_nmr_lighting_backward(_ptr(ins["faces"]), _ptr(ins["tex"]), _ptr(ins["ca"]), _ptr(ins["cd"]),
                                             _ptr(ins["d"]), _ptr(ins["g"]), _ptr(gf), _ptr(gt), _ptr(gl),
                                             ctypes.byref(p), _ptr(ws), stream), "backward")
    torch.cuda.synchronize()
    for b, n, s in bufs:
        assert guards_intact(b, n, s), "an input's guard band changed"
    assert guards_intact(lbuf, lit.numel(), skew), "write outside lit_textures"
    res = {"lit": lit.cpu().numpy()}
    for k, (b, v) in outs.items():
        assert guards_intact(b, v.numel(), skew), "write outside grad %s" % k
        res[k] = v.cpu().numpy()
    return res


def lib_params(B, F, T, dt, Ia, Id, ca, cd, d):
    p = _lib.UmrNmrLightParams()
    p.batch_size, p.num_faces, p.texture_res, p.dtype = B, F, T, dt
    p.intensity_ambient, p.intensity_directional = Ia, Id
    p.color_ambient_bstride, p.color_directional_bstride, p.direction_bstride = (3 if np.ndim(x) == 2 else 0
                                                                                 for x in (ca, cd, d))
    return p


def assert_within(got, ref, what):
    """Non-finite elements equal, finite ones within twice the oracle's first-order bound; no guard value left."""
    assert not (got == GUARD).any(), "%s: unwritten elements" % what
    fin = np.isfinite(ref.v)
    assert np.array_equal(np.isfinite(got), fin), "%s: non-finite pattern differs" % what
    assert np.array_equal(got[~fin], ref.v[~fin], equal_nan=True), "%s: non-finite values differ" % what
    err = np.abs(got.astype(np.float64) - ref.v)[fin]
    bound = 2 * ref.e[fin]
    bound[np.isnan(bound)] = np.inf     # a finite result computed from non-finite intermediates: not bounded
    assert (err <= bound).all(), "%s: max excess %g (err %g)" % (what, (err - bound).max(), err.max())


def check(faces, tex, g, Ia, Id, ca, cd, d, dt=0, skew=0, random=True):
    """`random`: no face of the scene may sit within the error bound of the relu or eps branch point, where the
    oracle and the kernel could take different branches (the special-face scene builds its branch cases exactly)."""
    u = TD[dt][2]
    lit, _ = oracle.forward(faces, tex, Ia, Id, ca, cd, d, u=u)
    ref = oracle.backward(faces, tex, g, Ia, Id, ca, cd, d, u=u)
    if random:
        assert not ref["ambiguous"].any(), "the scene has faces on a branch point: change its seed"
    got = call(faces, tex, g, Ia, Id, ca, cd, d, dt, skew)
    assert_within(got["lit"], lit, "lit")
    assert_within(got["tex"], ref["grad_textures"], "grad_textures")
    assert_within(got["faces"], ref["grad_faces"], "grad_faces")
    for i, k in enumerate(("grad_ca", "grad_cd", "grad_dir")):
        assert_within(got["light"][:, 3 * i:3 * i + 3], ref[k], k)
    if Id == 0:
        assert (got["faces"] == 0).all() and not np.signbit(got["faces"]).any()
    return got, ref


def scene(rng, B, F, T, batched, dt=0):
    nd = TD[dt][1]
    faces = rng.uniform(-1, 1, (B, F, 3, 3)).astype(nd)
    tex = rng.uniform(0, 1, (B, F, T, T, T, 3)).astype(nd)
    g = rng.uniform(-1, 1, tex.shape).astype(nd)
    sh = (B, 3) if batched else (3,)
    ca = rng.uniform(0.1, 1.0, sh).astype(nd)
    cd = rng.uniform(0.1, 1.0, sh).astype(nd)
    d = (rng.uniform(-1, 1, sh) + [0.2, 0.6, -0.3]).astype(nd)
    return faces, tex, g, ca, cd, d


SIZES = [(1, 1, 2), (1, 31, 3), (3, 32, 4), (3, 33, 6), (16, 1, 3), (16, 31, 2), (16, 1280, 6), (16, 1280, 2),
         (1, 65537, 2), (3, 65537, 3)]


@pytest.mark.parametrize("B,F,T", SIZES)
@pytest.mark.parametrize("batched", [False, True])
def test_float32_against_oracle(B, F, T, batched):
    rng = np.random.default_rng(B * 1000 + F + T)
    faces, tex, g, ca, cd, d = scene(rng, B, F, T, batched)
    check(faces, tex, g, 0.5, 0.5, ca, cd, d)


@pytest.mark.parametrize("B,F,T", [(1, 1, 2), (3, 33, 3), (16, 1280, 4), (1, 65537, 2)])
@pytest.mark.parametrize("batched", [False, True])
def test_float64_against_oracle(B, F, T, batched):
    rng = np.random.default_rng(B * 7 + F + T)
    faces, tex, g, ca, cd, d = scene(rng, B, F, T, batched, dt=1)
    check(faces, tex, g, 0.4, 0.7, ca, cd, d, dt=1)


@pytest.mark.parametrize("dt", [0, 1])
@pytest.mark.parametrize("Ia,Id", [(0.0, 0.8), (0.7, 0.0), (0.0, 0.0), (1.3, -0.4)])
def test_zero_and_signed_intensities(dt, Ia, Id):
    rng = np.random.default_rng(11)
    faces, tex, g, ca, cd, d = scene(rng, 3, 33, 3, True, dt)
    got, _ = check(faces, tex, g, Ia, Id, ca, cd, d, dt)
    if Ia == 0 and Id == 0:
        assert (got["lit"] == 0).all() and (got["tex"] == 0).all()


@pytest.mark.parametrize("dt", [0, 1])
@pytest.mark.parametrize("skew", [0, 1])
def test_special_faces(dt, skew):
    """Zero-area faces (the eps branch), n.d exactly 0, tiny faces, and NaN / +-inf coordinates, beside ordinary
    faces whose results must not change."""
    rng = np.random.default_rng(12)
    nd = TD[dt][1]
    faces, tex, g, ca, cd, d = scene(rng, 2, 40, 3, False, dt)
    d = np.array([0.0, 1.0, 0.0], nd)
    faces[0, 0] = [[0, 0, 0], [0, 0, 0], [0.5, 0.2, 0.1]]          # two equal vertices: cross exactly 0
    faces[0, 1] = [[0, 0, 0], [1, 1, 1], [2, 2, 2]]                # collinear, exactly
    faces[0, 2] = [[0, 0, 0.5], [0.5, 0, 0.5], [0, 0.5, 0.5]]      # in a z plane: n = (0,0,1), n.d exactly 0
    faces[0, 3] = [[0, 0, 0.5], [0, 0.5, 0.5], [0.5, 0, 0.5]]      # the same, reversed
    faces[0, 4] = [[0.1, 0.2, 0.3], [0.1 + 1e-4, 0.2, 0.3], [0.1, 0.2, 0.3 + 1e-4]]   # |cross| ~ 1e-8 < eps
    faces[1, 0, 0, 0] = np.nan
    faces[1, 1, 1, 2] = np.inf
    faces[1, 2, 2, 1] = -np.inf
    faces[1, 3] = [[np.inf, 0, 0], [0, 0, 0], [0, 1, 0]]
    got, ref = check(faces, tex, g, 0.5, 0.5, ca, cd, d, dt, skew, random=False)
    assert np.isfinite(got["lit"][0]).all() and np.isfinite(got["faces"][0]).all()
    assert (got["faces"][0, 2:4] == 0).all()                        # relu at exactly 0: no gradient
    assert not np.isfinite(got["faces"][1, 0]).all()


def test_launch_counts_and_reproducibility():
    lib = _lib.load()
    rng = np.random.default_rng(13)
    faces, tex, g, ca, cd, d = scene(rng, 16, 1280, 6, True)
    ft = torch.from_numpy(faces).to(DEV).requires_grad_(True)
    tt = torch.from_numpy(tex).to(DEV).requires_grad_(True)
    cat = torch.from_numpy(ca).to(DEV).requires_grad_(True)
    gt = torch.from_numpy(g).to(DEV)
    results = []
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        for det in (False, True, False, True):
            torch.use_deterministic_algorithms(det)
            for x in (ft, tt, cat):
                x.grad = None
            n0 = lib.umr_launch_count()
            out = nr.lighting(ft, tt, 0.5, 0.5, cat, cd, d)
            assert lib.umr_launch_count() - n0 == 1
            n0 = lib.umr_launch_count()
            out.backward(gt)
            assert lib.umr_launch_count() - n0 == 2          # backward + the light-parameter reduction
            results.append([t.detach().clone() for t in (out, ft.grad, tt.grad, cat.grad)])
        ft.grad = None
        out = nr.lighting(ft, tt.detach(), 0.5, 0.5, ca, cd, d)
        n0 = lib.umr_launch_count()
        out.backward(gt)
        assert lib.umr_launch_count() - n0 == 1              # no light parameter wants a gradient
    finally:
        torch.use_deterministic_algorithms(prev)
    for r in results[1:]:
        for a, b in zip(results[0], r):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_autograd_api_dtypes_and_out_of_place():
    rng = np.random.default_rng(14)
    faces, tex, g, ca, cd, d = scene(rng, 2, 5, 2, False)
    ft = torch.from_numpy(faces).to(DEV).half().requires_grad_(True)
    tt = torch.from_numpy(tex).to(DEV).requires_grad_(True)
    dd = torch.from_numpy(d).to(DEV).double().requires_grad_(True)
    out = nr.lighting(ft, tt, 0.5, 0.5, list(ca), cd, dd)
    assert out.dtype == torch.float64                            # a float64 direction: double compute
    out.sum().backward()
    assert ft.grad.dtype == torch.float16 and tt.grad.dtype == torch.float32 and dd.grad.dtype == torch.float64
    tex0 = tt.detach().clone()
    out = nr.lighting(ft.detach().float(), tt)
    assert out.dtype == torch.float32 and torch.equal(tt.detach(), tex0)   # textures untouched
    assert out.data_ptr() != tt.data_ptr()
    # [3] arguments: their gradient is the per-image gradient summed over the batch
    cdt = torch.from_numpy(cd).to(DEV).requires_grad_(True)
    cdb = cdt.detach()[None].repeat(2, 1).requires_grad_(True)
    gg = torch.from_numpy(g).to(DEV)
    nr.lighting(ft.detach().float(), tt.detach(), 0.5, 0.5, ca, cdt, d).backward(gg)
    nr.lighting(ft.detach().float(), tt.detach(), 0.5, 0.5, ca, cdb, d).backward(gg)
    assert torch.equal(cdt.grad, cdb.grad.sum(0))


def test_double_backward_raises():
    rng = np.random.default_rng(16)
    faces, tex, _, ca, cd, d = scene(rng, 1, 3, 2, False)
    ft = torch.from_numpy(faces).to(DEV).requires_grad_(True)
    tt = torch.from_numpy(tex).to(DEV).requires_grad_(True)
    out = nr.lighting(ft, tt, 0.5, 0.5, ca, cd, d)
    v = torch.ones_like(out, requires_grad=True)          # a graph through the first backward, as gradgradcheck builds
    (gf,) = torch.autograd.grad(out, ft, grad_outputs=v, create_graph=True)
    with pytest.raises(RuntimeError, match="once_differentiable"):
        gf.sum().backward()


def test_gradcheck_float64():
    rng = np.random.default_rng(15)
    faces, tex, g, ca, cd, d = scene(rng, 2, 4, 2, True, dt=1)
    args = [torch.from_numpy(a).to(DEV).requires_grad_(True) for a in (faces, tex, ca, cd, d)]
    fn = lambda f, t, a, c, dd: nr.lighting(f, t, 0.6, 0.7, a, c, dd)   # noqa: E731
    assert torch.autograd.gradcheck(fn, args)
    args[2] = torch.from_numpy(ca[0]).to(DEV).requires_grad_(True)     # a [3] colour
    assert torch.autograd.gradcheck(fn, args)


# ----------------------------------------------------------------------------------------------------------------
# the composed pipeline
# ----------------------------------------------------------------------------------------------------------------
def _mesh(B, subdiv, seed):
    v, f = synth.icosphere(subdiv)
    rng = np.random.default_rng(seed)
    v = (v * rng.uniform(0.6, 0.9, (B, 1, 3)) + rng.uniform(-0.1, 0.1, (B, 1, 3))).astype(np.float32)
    return torch.from_numpy(v).to(DEV), torch.from_numpy(np.repeat(f[None].astype(np.int32), B, 0)).to(DEV)


@pytest.mark.parametrize("aa,IS", [(True, 64), (False, 65)])
def test_composition_is_renderers(aa, IS):
    """Fill-back concatenation, lighting on the world-space faces, look_at(eye=(0,0,e)), vertices_to_faces and
    rasterize_rgbad reproduce Renderer.render: alpha and depth bit for bit, rgb within the rounding of lighting the texel
    before the blend."""
    verts, fcs = _mesh(2, 2, 1)
    B, F = fcs.shape[:2]
    T = 3
    rng = np.random.default_rng(2)
    tex = torch.from_numpy(rng.uniform(0, 1, (B, F, T, T, T, 3)).astype(np.float32)).to(DEV)
    kw = dict(light_intensity_ambient=0.4, light_intensity_directional=0.7, light_color_ambient=[1.0, 0.9, 0.8],
              light_color_directional=[0.7, 0.8, 1.0], light_direction=[0.3, 1.0, -0.5])
    r = nr.Renderer(image_size=IS, anti_aliasing=aa, background_color=[0.1, 0.2, 0.3], fill_back=True,
                    camera_mode="look_at", perspective=False, **kw)
    rgb, depth, alpha = r.render(verts, fcs, tex)
    faces_all = torch.cat([fcs, fcs[:, :, [2, 1, 0]]], 1)
    tex_all = torch.cat([tex, tex.permute(0, 1, 4, 3, 2, 5)], 1)
    lit = nr.lighting(nr.vertices_to_faces(verts, faces_all), tex_all, kw["light_intensity_ambient"],
                      kw["light_intensity_directional"], kw["light_color_ambient"], kw["light_color_directional"],
                      kw["light_direction"])
    cam = nr.look_at(verts, r.eye)
    out = nr.rasterize_rgbad(nr.vertices_to_faces(cam, faces_all), lit, IS, aa, r.near, r.far,
                             background_color=[0.1, 0.2, 0.3])
    assert torch.equal(out["alpha"].view(torch.int32), alpha.view(torch.int32))
    assert torch.equal(out["depth"].view(torch.int32), depth.view(torch.int32))
    assert alpha.sum() > 0
    # each texel is rounded once more when lit first: 8 blend terms + the pool, each off by <= u * |term|
    tol = 16 * 2.0 ** -24 * rgb.abs().max()
    assert float((out["rgb"] - rgb).abs().max()) <= tol


def _views(verts, eyes):
    """[B,V,3] world vertices, eyes [n,3] -> [B*n,V,3] perspective NDC vertices."""
    B, n = verts.shape[0], eyes.shape[0]
    vv = verts.repeat_interleave(n, 0)
    e = eyes.repeat(B, 1)
    return nr.perspective(nr.look_at(vv, e), 30.0)


def _iou_loss(a, b):
    inter = (a * b).sum((1, 2))
    union = (a + b - a * b).sum((1, 2))
    return (1 - inter / union).mean()


def test_silhouette_fitting_from_three_views():
    """NMR's example 2: fit an icosphere's vertices to the silhouettes of a deformed target seen from three
    get_points_from_angles + look_at + perspective views."""
    v, f = synth.icosphere(2)
    f = np.concatenate([f, f[:, [2, 1, 0]]])                   # both orientations: no culling surprises
    base = torch.from_numpy(v.astype(np.float32)).to(DEV)[None]
    faces = torch.from_numpy(f.astype(np.int32)).to(DEV)[None]
    target_v = base * torch.tensor([1.2, 0.75, 0.9], device=DEV) + 0.15 * torch.sin(3 * base[..., [1, 2, 0]])
    eyes = torch.tensor([nr.get_points_from_angles(4.0, 20.0, az) for az in (0.0, 120.0, 240.0)], device=DEV)
    IS = 64

    def render(vert):
        fv = nr.vertices_to_faces(_views(vert, eyes), faces.repeat(eyes.shape[0], 1, 1))
        return nr.rasterize_silhouettes(fv, IS, True)
    with torch.no_grad():
        target = render(target_v)
    disp = torch.zeros_like(base, requires_grad=True)
    opt = torch.optim.Adam([disp], lr=0.01)
    losses = []
    for _ in range(150):
        opt.zero_grad()
        loss = _iou_loss(render(base + disp), target)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[0] > 0.1
    assert np.mean(losses[-10:]) < 0.5 * np.mean(losses[:10])
    assert losses[-1] < 0.1


def test_eye_recovery_through_look_at():
    """Recover a perturbed eye position from a lit, textured target image; the gradient reaches the eye through
    look_at and perspective."""
    v, f = synth.icosphere(3)
    f = np.concatenate([f, f[:, [2, 1, 0]]])
    verts = torch.from_numpy(v.astype(np.float32)).to(DEV)[None] * torch.tensor([1.0, 0.7, 0.8], device=DEV)
    faces = torch.from_numpy(f.astype(np.int32)).to(DEV)[None]
    F, T = faces.shape[1], 2
    fv_world = nr.vertices_to_faces(verts, faces)
    centre = fv_world.mean(2)                                    # colour varies smoothly over the surface
    tex = (0.5 + 0.5 * torch.sin(3 * centre + torch.tensor([0.0, 2.0, 4.0], device=DEV)))[:, :, None, None, None, :]
    tex = tex.expand(1, F, T, T, T, 3).contiguous()
    lit = nr.lighting(fv_world, tex, 0.4, 0.6, direction=(0.3, 0.8, -0.5))
    eye0 = torch.tensor([nr.get_points_from_angles(3.5, 20.0, 40.0)], device=DEV)
    IS = 96

    def render(eye):
        out = nr.rasterize_rgbad(nr.vertices_to_faces(_views(verts, eye), faces), lit, IS, True, return_depth=False)
        return out["rgb"], out["alpha"]
    with torch.no_grad():
        trgb, talpha = render(eye0)
    eye = (eye0 + torch.tensor([[0.35, -0.25, 0.3]], device=DEV)).requires_grad_(True)
    opt = torch.optim.Adam([eye], lr=0.02)
    errs = [float((eye - eye0).norm())]
    for _ in range(120):
        opt.zero_grad()
        rgb, alpha = render(eye)
        loss = ((rgb - trgb) ** 2).mean() + ((alpha - talpha) ** 2).mean()
        loss.backward()
        opt.step()
        errs.append(float((eye - eye0).norm()))
    assert eye.grad is not None and torch.isfinite(eye.grad).all()
    assert errs[-1] < 0.7 * errs[0], errs[::10]
