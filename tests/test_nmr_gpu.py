"""umr_nmr_* kernels (csrc/nmr.cu) against the CPU oracle of the NMR render contract (oracle/nmr.py), on seeded synthetic
scenes from umr_b200.synth: forward planes, texture gradient, the nmr_pytorch.NeuralRenderer call pattern, agreement with
the SoftRas hard z-buffer, MultiTextureLoss(renderer="nmr") and the launch count.

Forward planes (face index, raster depth, rgb, alpha, depth) are compared BIT-EXACT: the kernels keep the contract's
operation order, including the 2x2 pool's summation order, so no ulp tolerance is needed."""
import ctypes

import numpy as np
import pytest
import torch

import losses as oracle_losses
import nmr as oracle
from umr_b200 import _lib, synth
from umr_b200.nnutils import geom_utils, loss_utils
from umr_b200.raster import _ptr, _stream_ptr

pytestmark = pytest.mark.gpu
EYE = -2.732
AMBIENT = dict(Ia=1.0, Id=0.0)                               # nmr_pytorch.py:105-108 ambient_light_only
VISUAL = dict(Ia=0.8, Id=0.4, direction=(0.0, 1.0, -1.0))   # train_s2.py:111-113, demo.py:64-67
DEFAULT = dict(Ia=0.5, Id=0.5, direction=(0.0, 1.0, 0.0))   # NMR's defaults


def nmr_inputs(B, subdiv, seed=0, soup=0):
    """Renderer input as nmr_pytorch.Render hands it over: orthographic_proj_withz(..., offset_z=5) with y negated
    (nmr_pytorch.py:76-77,123).  `soup` adds open triangles of both orientations, so fill_back copies are drawn."""
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(subdiv)
    verts = torch.from_numpy(synth.bird_like(v, rng, B))
    cams = torch.from_numpy(synth.cameras(rng, B))
    proj = geom_utils.orthographic_proj_withz(verts, cams, offset_z=5.0)
    proj[:, :, 1] *= -1
    proj = proj.numpy()
    faces = np.repeat(f[None], B, 0)
    if soup:
        sv = rng.uniform(-0.9, 0.9, size=(B, 3 * soup, 3)).astype(np.float32)
        sv[..., 2] = rng.uniform(3.0, 4.0, size=(B, 3 * soup))
        proj = np.concatenate([proj, sv], 1)
        faces = np.concatenate([faces, (v.shape[0] + np.arange(3 * soup).reshape(soup, 3))[None].repeat(B, 0)], 1)
    return proj.astype(np.float32), faces.astype(np.int32)


def params(B, V, F, T, IS, aa=True, fill_back=True, G=1, Ia=0.5, Id=0.5, ca=(1, 1, 1), cd=(1, 1, 1),
           direction=(0, 1, 0), bg=(0, 0, 0)):
    p = _lib.UmrNmrParams()
    p.batch_size, p.num_vertices, p.num_faces, p.texture_res = B, V, F, T
    p.image_size, p.anti_aliasing, p.fill_back, p.shared_textures = IS, int(aa), int(fill_back), G
    p.eye_z, p.near_plane, p.far_plane = EYE, 0.1, 100.0
    p.light_intensity_ambient, p.light_intensity_directional = Ia, Id
    p.light_color_ambient[:], p.light_color_directional[:], p.light_direction[:] = ca, cd, direction
    p.background_color[:] = bg
    return p


def abi_forward(verts, faces, tex, IS, **kw):
    lib = _lib.load()
    dev = torch.device("cuda:0")
    B, V = verts.shape[:2]
    F = faces.shape[1]
    T = 0 if tex is None else tex.shape[2]
    G = 1 if tex is None else B // tex.shape[0]
    p = params(B, V, F, T, IS, G=G, **kw)
    S = IS * (2 if p.anti_aliasing else 1)
    v = torch.from_numpy(verts).to(dev)
    f = torch.from_numpy(faces).to(dev)
    t = None if tex is None else torch.from_numpy(np.ascontiguousarray(tex)).to(dev)
    ws = torch.empty(lib.umr_nmr_workspace_bytes(B, F, p.fill_back), device=dev, dtype=torch.uint8)
    fidx = torch.empty(B, S, S, device=dev, dtype=torch.int32)
    rdepth = torch.empty(B, S, S, device=dev)
    rgb = None if tex is None else torch.empty(B, 3, IS, IS, device=dev)
    alpha, depth = torch.empty(B, IS, IS, device=dev), torch.empty(B, IS, IS, device=dev)
    _lib.check(lib.umr_nmr_forward(_ptr(v), _ptr(f), _ptr(t), _ptr(fidx), _ptr(rdepth), _ptr(rgb), _ptr(alpha),
                                   _ptr(depth), ctypes.byref(p), _ptr(ws), _stream_ptr(dev)), "umr_nmr_forward")
    out = {"face_index": fidx, "raster_depth": rdepth, "alpha": alpha, "depth": depth}
    if rgb is not None:
        out["rgb"] = rgb

    def backward(grad_rgb):
        g = torch.from_numpy(grad_rgb.astype(np.float32)).to(dev)
        gt = torch.full(t.shape, float("nan"), device=dev)   # the call zero-fills it
        _lib.check(lib.umr_nmr_backward_textures(_ptr(v), _ptr(f), _ptr(fidx), _ptr(g), _ptr(gt), ctypes.byref(p),
                                                 _ptr(ws), _stream_ptr(dev)), "umr_nmr_backward_textures")
        return gt.cpu().numpy()
    return {k: x.cpu().numpy() for k, x in out.items()}, backward


def oracle_kw(IS, aa=True, fill_back=True, Ia=0.5, Id=0.5, ca=(1, 1, 1), cd=(1, 1, 1), direction=(0, 1, 0),
              bg=(0, 0, 0), G=1):
    return dict(image_size=IS, anti_aliasing=aa, fill_back=fill_back, eye_z=EYE, light_intensity_ambient=Ia,
                light_intensity_directional=Id, light_color_ambient=ca, light_color_directional=cd,
                light_direction=direction, background_color=bg, shared_textures=G)


def assert_planes_equal(got, ref, names=("face_index", "raster_depth", "rgb", "alpha", "depth")):
    for n in names:
        if n not in ref:
            continue
        a, b = got[n], ref[n]
        assert a.shape == b.shape, (n, a.shape, b.shape)
        bad = ~((a == b) | (np.isnan(a) & np.isnan(b)) if a.dtype.kind == "f" else (a == b))
        assert not bad.any(), "%s differs at %d of %d elements, first %s: got %r, oracle %r" % (
            n, bad.sum(), bad.size, np.argwhere(bad)[0], a[tuple(np.argwhere(bad)[0])], b[tuple(np.argwhere(bad)[0])])


_ZB = {}


def zbuf(key, verts, faces, IS, aa=True, fill_back=True):
    if key not in _ZB:
        _ZB[key] = oracle.zbuffer(verts, faces, IS, aa, fill_back, EYE)
    return _ZB[key]


SMALL = dict(B=2, subdiv=2, seed=1, soup=8)


@pytest.mark.parametrize("fill_back,bg,light", [
    (True, (0, 0, 0), AMBIENT), (True, (1, 1, 1), VISUAL), (False, (0, 0, 0), VISUAL), (False, (1, 1, 1), DEFAULT)])
def test_forward_matches_oracle_64(fill_back, bg, light):
    verts, faces = nmr_inputs(**SMALL)
    tex = np.random.default_rng(2).uniform(0, 1, size=(2, faces.shape[1], 4, 4, 4, 3)).astype(np.float32)
    got, _ = abi_forward(verts, faces, tex, 64, fill_back=fill_back, bg=bg, **light)
    zb = zbuf(("small", fill_back), verts, faces, 64, True, fill_back)
    ref = oracle.render(verts, faces, tex, zbuf=zb, **oracle_kw(64, fill_back=fill_back, bg=bg, **light))
    assert_planes_equal(got, ref)
    assert 0.05 < ref["alpha"].mean() < 0.9
    if fill_back:
        assert (ref["face_index"] >= faces.shape[1]).any()   # the reversed copies are exercised


@pytest.mark.parametrize("aa", [True, False])
def test_silhouettes_and_depth_without_texture(aa):
    verts, faces = nmr_inputs(**SMALL)
    got, _ = abi_forward(verts, faces, None, 64, aa=aa)
    ref = oracle.render(verts, faces, None, zbuf=zbuf(("small", True, aa), verts, faces, 64, aa, True),
                        **oracle_kw(64, aa=aa))
    assert "rgb" not in got
    assert_planes_equal(got, ref)


def test_forward_at_the_training_visual_shape():
    """train_s2.py:322-324: batch 16, 256^2, 1280 faces, the [B,F,6,6,3] texture repeated along the cube's last axis."""
    B, T = 16, 6
    verts, faces = nmr_inputs(B, 3, seed=3)
    assert faces.shape[1] == 1280
    tex = np.random.default_rng(4).uniform(0, 1, size=(B, 1280, T, T, 3)).astype(np.float32)
    cube = np.repeat(tex[:, :, :, :, None], T, axis=4)
    zb = zbuf("train", verts, faces, 256)
    for bg in ((0, 0, 0), (1, 1, 1)):
        got, _ = abi_forward(verts, faces, cube, 256, bg=bg, **VISUAL)
        assert_planes_equal(got, oracle.render(verts, faces, cube, zbuf=zb, **oracle_kw(256, bg=bg, **VISUAL)))


@pytest.mark.parametrize("fill_back,G,aa", [(True, 1, True), (False, 1, True), (True, 2, False)])
def test_texture_gradient_matches_the_oracle_adjoint(fill_back, G, aa):
    verts, faces = nmr_inputs(**SMALL)
    B, F = faces.shape[:2]
    rng = np.random.default_rng(5)
    tex = rng.uniform(0, 1, size=(B // G, F, 3, 3, 3, 3)).astype(np.float32)
    light = dict(Ia=0.6, Id=0.5, ca=(1, 0.9, 0.8), cd=(0.5, 1, 1), direction=(0.2, 1, -1))
    got, backward = abi_forward(verts, faces, tex, 64, aa=aa, fill_back=fill_back, **light)
    g = rng.uniform(0.5, 1.5, size=got["rgb"].shape)   # one sign: no cancellation in the float32 accumulation
    gk = backward(g)
    zb = (got["face_index"], got["raster_depth"])
    gr = oracle.grad_textures(g, verts, faces, tex.shape, zb, anti_aliasing=aa, fill_back=fill_back, eye_z=EYE,
                              shared_textures=G, Ia=light["Ia"], Id=light["Id"], ca=light["ca"], cd=light["cd"],
                              direction=light["direction"])
    assert np.abs(gr).max() > 0
    err = np.abs(gk - gr)
    assert (err <= 1e-5 * np.maximum(np.abs(gk), np.abs(gr)) + 1e-7).all(), err.max()
    if fill_back:
        back = np.unique(zb[0][zb[0] >= F]) - F
        assert back.size and np.abs(gr[:, back]).max() > 0


def _nmr_pytorch(img_size):
    """nnutils/nmr_pytorch.py restated (the reference tree is not importable here): NMR.__init__ :42-43,
    NeuralRenderer.__init__ :89-103, ambient_light_only :105-108, set_light_dir :113-117 (as train_s2.py:111-113 calls
    them), Render.forward :73-86, NeuralRenderer.forward :123-128."""
    from umr_b200 import compat
    compat.install()
    import neural_renderer
    r = neural_renderer.Renderer(image_size=img_size, anti_aliasing=True, camera_mode="look_at", perspective=False,
                                 background_color=[0, 0, 0])
    r.eye = [0, 0, -2.732]
    r.light_intensity_ambient = 0.8
    r.light_intensity_ambient, r.light_intensity_directional = 1, 0       # ambient_light_only()
    r.light_direction, r.light_intensity_directional, r.light_intensity_ambient = [0, 1, -1], 0.4, 0.8  # set_light_dir

    def forward(vertices, faces, cams, textures=None):
        faces = faces.int()
        vs = geom_utils.orthographic_proj_withz(vertices, cams, offset_z=5.)
        vs[:, :, 1] *= -1
        if textures is None:
            return r.render_silhouettes(vs, faces)
        return r.render_rgb(vs, faces, textures)
    return r, forward


def test_neural_renderer_call_pattern():
    B, IS, T = 4, 64, 6
    rng = np.random.default_rng(6)
    v, f = synth.icosphere(3)
    dev = torch.device("cuda:0")
    verts = torch.from_numpy(synth.bird_like(v, rng, B)).to(dev)
    faces = torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1).to(dev)
    cams = torch.from_numpy(synth.cameras(rng, B)).to(dev)
    tex = torch.rand(B, f.shape[0], T, T, 3, device=dev)
    cube = tex.view(B, f.shape[0], T, T, 3).unsqueeze(4).repeat(1, 1, 1, 1, T, 1)   # train_s2.py:322
    _, vis = _nmr_pytorch(IS)
    with torch.no_grad():
        image_pred = vis(verts, faces, cams, cube)                 # train_s2.py:323
        mask_pred = vis(verts, faces, cams).unsqueeze(1)           # train_s2.py:324
        vs = geom_utils.orthographic_proj_withz(verts, cams, offset_z=5.)
        vs[:, :, 1] *= -1
    assert image_pred.shape == (B, 3, IS, IS) and mask_pred.shape == (B, 1, IS, IS)
    vs, fs = vs.cpu().numpy(), faces.int().cpu().numpy()
    ref = oracle.render(vs, fs, cube.cpu().numpy(), **oracle_kw(IS, **VISUAL))
    assert np.array_equal(image_pred.cpu().numpy(), ref["rgb"])
    assert np.array_equal(mask_pred[:, 0].cpu().numpy(), ref["alpha"])
    # the texture gets its gradient through autograd (the geometry is detached, as at every UMR call site)
    r, vis = _nmr_pytorch(IS)
    cube_g = cube.detach().requires_grad_(True)
    vis(verts, faces, cams, cube_g).sum().backward()
    assert torch.isfinite(cube_g.grad).all() and cube_g.grad.abs().sum() > 0
    with pytest.raises(NotImplementedError, match="vertex / camera gradient"):
        vis(verts.detach().requires_grad_(True), faces, cams, cube)


def test_coverage_agrees_with_the_softras_hard_z_buffer():
    """Same mesh and camera: NMR's coverage and smr.SoftRenderer("hard")'s visibility plane differ only within one pixel
    of a silhouette edge (a flip or pixel-centre error between the two images UMR shows side by side fails this)."""
    B, IS = 4, 64
    rng = np.random.default_rng(7)
    v, f = synth.icosphere(3)
    dev = torch.device("cuda:0")
    verts = torch.from_numpy(synth.bird_like(v, rng, B)).to(dev)
    faces = torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1).to(dev)
    cams = torch.from_numpy(synth.cameras(rng, B)).to(dev)
    _, aggrs = loss_utils.SoftRenderer(IS, "hard").visibility(verts, faces, cams)
    soft = aggrs[:, 1].cpu().numpy() >= 0                      # rows top-down
    vs = geom_utils.orthographic_proj_withz(verts, cams, offset_z=5.)
    vs[:, :, 1] *= -1
    got, _ = abi_forward(vs.cpu().numpy(), faces.int().cpu().numpy(), None, IS, **VISUAL)
    hard = got["face_index"][:, ::-1] >= 0                     # raster rows bottom-up -> top-down
    assert hard.shape == soft.shape and 0.05 < hard.mean() < 0.9
    pad = np.pad(hard, ((0, 0), (1, 1), (1, 1)), mode="edge")
    S = hard.shape[1]
    nb = np.stack([pad[:, 1 + dy:1 + dy + S, 1 + dx:1 + dx + S] for dy in (-1, 0, 1) for dx in (-1, 0, 1)])
    edge = nb.any(0) != nb.all(0)
    diff = hard != soft
    assert not (diff & ~edge).any(), "coverage differs away from the silhouette at %d pixels" % (diff & ~edge).sum()
    assert diff.sum() < 0.1 * edge.sum()


def test_multi_texture_loss_nmr_matches_the_oracle_composition():
    B, H, IS = 2, 8, 64
    rng = np.random.default_rng(8)
    v, f = synth.icosphere(2)
    F = f.shape[0]
    dev = torch.device("cuda:0")
    vs = torch.from_numpy(synth.bird_like(v, rng, B)).to(dev)
    fs = torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1).to(dev)
    cams = torch.from_numpy(synth.cameras(rng, B * H)).to(dev).view(B, H, 7)
    cam_probs = torch.softmax(torch.from_numpy(rng.normal(size=(B, H)).astype(np.float32)), 1).to(dev)
    proj_cam = cams[:, 0].contiguous()
    rgbs = torch.from_numpy(synth.smooth_images(rng, B, IS)).to(dev)
    masks = torch.from_numpy(synth.ellipse_masks(rng, B, IS)).to(dev)
    masks_pred = torch.from_numpy(rng.uniform(0, 1, size=(B * H, IS, IS)).astype(np.float32)).to(dev)
    tx = torch.from_numpy(rng.uniform(0, 1, size=(B, F, 36, 3)).astype(np.float32)).to(dev).requires_grad_(True)
    flow = torch.from_numpy(synth.texture_flow(rng, B, F)).to(dev)
    dts = torch.from_numpy(np.stack([synth.dt_barrier(mk) for mk in masks.cpu().numpy()])).to(dev).unsqueeze(1)
    m = loss_utils.MultiTextureLoss(samples_per_gpu=B, num_hypo_cams=H, image_size=IS, texture_loss_type="l1",
                                    renderer="nmr")
    tex_loss, _, _, texture_pred = m(vs, fs, cams, cam_probs, proj_cam, rgbs, masks, masks_pred, tx, flow, dts)
    tex_loss.backward()
    assert texture_pred.shape == (B * H, 3, IS, IS)
    # CPU composition: oracle render of the same renderer input + oracle/losses.py
    with torch.no_grad():
        vr = geom_utils.orthographic_proj_withz(loss_utils.tile_hypotheses(vs, H), cams.view(-1, 7), offset_z=5.)
        vr[:, :, 1] *= -1
    vr, fr = vr.cpu().numpy(), np.repeat(f[None], B * H, 0).astype(np.int32)
    cube = np.repeat(tx.detach().cpu().numpy().reshape(B, F, 6, 6, 3)[:, :, None], 6, axis=2)
    kw = oracle_kw(IS, G=H, **AMBIENT)
    ref = oracle.render(vr, fr, cube, **kw)
    assert np.array_equal(texture_pred.detach().cpu().numpy(), ref["rgb"])
    rgb_t = torch.from_numpy(ref["rgb"]).requires_grad_(True)
    per = oracle_losses.texture_loss_masks(rgb_t, loss_utils.tile_hypotheses(rgbs, H).cpu(),
                                           loss_utils.tile_hypotheses(masks, H).cpu(), masks_pred.cpu(), avg=False)
    loss_ref = (per.view(B, -1) * cam_probs.cpu()).sum(1).mean()
    loss_ref.backward()
    assert float(tex_loss.detach()) == pytest.approx(float(loss_ref.detach()), rel=1e-5)
    g = oracle.grad_textures(rgb_t.grad.numpy(), vr, fr, cube.shape, (ref["face_index"], ref["raster_depth"]),
                             anti_aliasing=True, fill_back=True, eye_z=EYE, shared_textures=H, Ia=1.0, Id=0.0)
    g = g.sum(axis=2).reshape(B, F, 36, 3)
    got = tx.grad.cpu().numpy()
    assert np.abs(g).max() > 0
    assert np.allclose(got, g, rtol=1e-4, atol=1e-6 * np.abs(g).max()), np.abs(got - g).max()


def test_render_rgb_launch_count():
    lib = _lib.load()
    r, _ = _nmr_pytorch(64)
    verts, faces = nmr_inputs(**SMALL)
    v, f = torch.from_numpy(verts).cuda(), torch.from_numpy(faces).cuda()
    tex = torch.rand(2, faces.shape[1], 3, 3, 3, 3, device="cuda", requires_grad=True)
    r.render_rgb(v, f, tex)   # warm-up
    torch.cuda.synchronize()
    n0 = lib.umr_launch_count()
    img = r.render_rgb(v, f, tex)
    assert lib.umr_launch_count() - n0 == 3   # prep, z-buffer, shading
    n0 = lib.umr_launch_count()
    img.sum().backward()
    assert lib.umr_launch_count() - n0 == 2   # prep, texture gradient
