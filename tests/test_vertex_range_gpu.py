"""The fused vertex kernels (umr_b200/csrc/vertex.cu) against the float64 reference (oracle/vertex_ref.py) across
their accepted input range: vertex counts on both sides of the 256-vertex CTA of `k_project_backward` (the camera
gradient is summed across CTAs), face counts on both sides of the 256-face CTA, 1 to 8 camera hypotheses and up to
65535 renders, every face layout with a different face order per mesh, the light off / default / coloured with an
unnormalised direction, viewing_scale 1 and 0.75, flip_y off, the eps branch of the normal, partial gradients, and
`k_corr_fwd` / `k_corr_bwd` / `k_corr_gather` at target counts around a warp, more than 256 selected vertices,
exact distance ties, shared vertices, zero weights and 128 renders.

Tolerances are error bounds, not tuned rtols.  u = 2^-24 and gamma_n = n u / (1 - n u).
* Every compared quantity except the light is a polynomial of the float32 inputs that the kernel evaluates with
  one rounding per operation (-fmad=false), so |kernel - exact| <= gamma_D * M, where M is the magnitude
  evaluation (`vertex_ref`, `magnitude=True`; for gradients autograd through it with |upstream|) and D the longest
  chain of roundings.  One more rounding in D covers the float64 reference's own error.  D, counted in vertex.cu:
  - face vertices: 11 (8 in the two quaternion products, scale, translate / offset, look_at or orthogonal).
  - corner gradients: 1 (the viewing-scale product), 28 with the light; the scatter adds one rounding per
    corner that lands on a vertex (`valence`, the largest count of corners on one vertex).
  - vertex gradients: corner depth + valence + 8 (closed-form rotation backward) + H (hypothesis atomics).
  - camera gradients: corner depth + valence + 11 (per-vertex terms) + 5 (warp tree) + 8 (CTA's warps) +
    ceil(V / 256) (one atomic per CTA).
  - corr: vert2d 10; loss 14 (expanded distance) + 1 (weight) + ceil(NS / 8) (a warp's running sum) + 8 (the
    CTA's warps) + 1 (mean); gradients 26 per selected vertex + ceil(NS / 256) + 13 for the cameras, + the
    largest number of selections of one vertex (+ B when one mesh serves every render) for the vertices.
* The light is not polynomial; `vertex_ref.light_error_bound` and `light_grad_magnitude` give first-order
  bounds from the conditioning kappa = |n_abs| / max(|n|, 1e-6) of each face's normal (their docstrings derive them).
* Faces whose cosine lies within its bound of the relu kink (n . d = 0) get a zero light gradient upstream: there
  the kernel and the exact relu may disagree on the branch.  They are rare (a handful of ~10^5).
* A nearest-target index that differs from the float64 argmin must be a near-tie (the two float64 distances differ
  by no more than both distances' rounding bound, as in test_losses_gpu.py::test_chamfer); the reference then uses
  the kernel's index for the loss and the gradients.
Each check prints the largest ratio of observed error to its bound (`pytest -s`).
"""
import math

import numpy as np
import pytest
import torch

import vertex_ref as R
from umr_b200 import ops, raster
from umr_b200 import soft_renderer as sr
from umr_b200.nnutils import geom_utils, loss_utils, smr
from umr_b200.vertex import project_faces
from vertex_ref import gamma

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EYE_Z = float(np.float32(-2.732))   # what the kernel receives
DEFAULT_LIGHT = (0.8, (1.0, 1.0, 1.0), 0.5, (1.0, 1.0, 1.0), (0.0, 1.0, 0.0))
COLOUR_LIGHT = (0.375, (0.9, 0.5, 0.25), 0.625, (0.5, 1.0, 0.75), (0.3, 1.1, -0.4))   # |d| != 1
LIGHTS = {"off": None, "default": DEFAULT_LIGHT, "colour": COLOUR_LIGHT}


def _f32(light):
    """The light parameters as the kernel sees them (float32)."""
    if light is None:
        return None
    ia, ca, idr, cd, d = light
    r = lambda x: float(np.float32(x))   # noqa: E731
    return r(ia), tuple(map(r, ca)), r(idr), tuple(map(r, cd)), tuple(map(r, d))


def _check(name, got, ref, mag, D):
    """|got - ref| <= gamma_D * mag everywhere; prints the largest error / bound ratio."""
    got = got.detach().double().cpu()
    ref = ref.detach().double().cpu()
    bound = gamma(D + 1) * mag.detach().double().cpu()
    err = (got - ref).abs()
    ratio = float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0
    print("%-44s D=%-5d max err/bound = %.3e" % (name, D, ratio))
    bad = err > bound
    assert not bad.any(), "%s: %d values outside the bound, worst ratio %.3g at %s (got %r ref %r)" % (
        name, int(bad.sum()), ratio, tuple(np.argwhere(bad.numpy())[0]), float(got[bad][0]), float(ref[bad][0]))
    return ratio


def _check_bound(name, got, ref, bound):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    err = (got - ref).abs()
    ratio = float((err / bound.clamp_min(1e-300)).max())
    print("%-44s          max err/bound = %.3e" % (name, ratio))
    assert (err <= bound).all(), "%s: worst ratio %.3g" % (name, ratio)


def _random_cams(g, n):
    q = torch.nn.functional.normalize(torch.randn(n, 4, generator=g, dtype=torch.float64), dim=1)
    s = 0.55 + 0.3 * torch.rand(n, 1, generator=g, dtype=torch.float64)
    t = 0.2 * torch.rand(n, 2, generator=g, dtype=torch.float64) - 0.1
    return torch.cat([s, t, q], 1).float()


def _case(V, F, Bv, H, layout, seed):
    """float32 vertices [Bv,V,3] in [-0.7, 0.7]^3, cams [Bv*H,7], faces of random distinct corners in the layout
    '2d' [F,3], '1' [1,F,3] or 'per_mesh' [Bv,F,3] (mesh k's face list is a different permutation of mesh 0's)."""
    g = torch.Generator().manual_seed(seed)
    verts = (1.4 * torch.rand(Bv, V, 3, generator=g, dtype=torch.float64) - 0.7).float()
    cams = _random_cams(g, Bv * H)
    base = torch.stack([torch.randperm(V, generator=g)[:3] for _ in range(F)]).int()
    if layout == "2d":
        faces = base
    elif layout == "1":
        faces = base[None]
    else:
        faces = torch.stack([base] + [base[torch.randperm(F, generator=g)] for _ in range(Bv - 1)])
    return verts, cams, faces


def _valence(faces, V):
    f = faces.reshape(-1, faces.shape[-2] * 3) if faces.dim() == 3 else faces.reshape(1, -1)
    return int(max(torch.bincount(row.long(), minlength=V).max() for row in f))


def _kink_faces(verts, cams, faces, flip_y, light):
    """[B,F] faces whose cosine is within its float32 bound of 0 (vertex_ref.light_error_bound)."""
    n, N, kappa, _ = R.normal_conditioning(verts.double(), cams.double(), faces, 5.0, flip_y)
    d = torch.tensor(light[4], dtype=torch.float64)
    cos = ((n / N[..., None]) * d).sum(2)
    return cos.abs() <= gamma(24) * (2 * kappa + 1) * d.norm()


def _compare_projection(tag, verts, cams, faces, vs, flip_y, light, g_fv, g_lt, got_fv, got_lt, got_gv, got_gc,
                        vert_batch=None, exact_corners=False):
    """got_* from the kernel, g_* the upstream gradients used; checks everything against the float64 reference."""
    V, B = verts.shape[1], cams.shape[0]
    H = B // verts.shape[0]
    vd = verts.double().requires_grad_(True)
    cd = cams.double().requires_grad_(True)
    fv, lt = R.project_faces_ref(vd, cd, faces, 5.0, EYE_Z, vs, flip_y, light)
    s = (fv * g_fv.double().cpu()).sum()
    if lt is not None:
        s = s + (lt * g_lt.double().cpu()).sum()
    gv, gc = torch.autograd.grad(s, (vd, cd))
    fv_m, _ = R.project_faces_ref(verts.double().abs(), cams.double().abs(), faces, 5.0, EYE_Z, vs, flip_y, None,
                                  magnitude=True)
    _check(tag + " face vertices", got_fv, fv, fv_m, 11)
    m_pre, corner = None, 1
    if light is not None:
        if got_lt is not None:
            _check_bound(tag + " light", got_lt, lt, R.light_error_bound(verts.double(), cams.double(), faces, 5.0,
                                                                         flip_y, light, exact_corners))
        m_pre, corner = R.light_grad_magnitude(verts.double(), cams.double(), faces, 5.0, flip_y, light,
                                               g_lt.double().cpu(), exact_corners), 28
    mv, mc = R.project_grad_magnitude(verts.double(), cams.double(), faces, 5.0, EYE_Z, vs, g_fv.double().cpu(), m_pre)
    val = _valence(faces, V)
    if got_gv is not None:
        if vert_batch is not None:     # vertices were an expanded view of one mesh: autograd summed the Bv copies
            gv, mv = gv.sum(0, keepdim=True), mv.sum(0, keepdim=True)
        _check(tag + " grad vertices", got_gv, gv, mv, corner + val + 8 + H + (verts.shape[0] if vert_batch else 0))
    if got_gc is not None:
        _check(tag + " grad cams", got_gc, gc, mc, corner + val + 24 + math.ceil(V / 256))


def _upstream(B, F, light, kink, seed):
    g = torch.Generator().manual_seed(seed + 1000)
    g_fv = torch.randn(B, F, 3, 3, generator=g)
    g_lt = None
    if light is not None:
        g_lt = torch.randn(B, F, 3, generator=g)
        g_lt[kink] = 0.0
    return g_fv, g_lt


# (V, F, Bv, H, face layout, light, viewing_scale, flip_y)
PROJ_CASES = [
    (3, 1, 1, 1, "2d", "off", 1.0, True),
    (255, 255, 2, 1, "per_mesh", "default", 1.0, True),
    (256, 256, 2, 2, "1", "colour", 0.75, True),
    (257, 257, 4, 2, "per_mesh", "default", 1.0, True),
    (642, 1280, 16, 8, "per_mesh", "colour", 0.75, True),
    (2562, 1280, 2, 8, "2d", "default", 1.0, True),
    (642, 1280, 128, 1, "per_mesh", "off", 1.0, True),
    (3, 257, 3, 2, "per_mesh", "colour", 0.75, False),
    (2562, 255, 1, 8, "1", "off", 0.75, False),
    (257, 1, 8, 8, "per_mesh", "default", 1.0, True),
]


@pytest.mark.parametrize("V,F,Bv,H,layout,light,vs,flip_y", PROJ_CASES)
def test_project_faces_matches_float64(V, F, Bv, H, layout, light, vs, flip_y):
    seed = V * 7 + F * 3 + Bv + H
    verts, cams, faces = _case(V, F, Bv, H, layout, seed)
    lc = _f32(LIGHTS[light])
    B = Bv * H
    kink = _kink_faces(verts, cams, faces, flip_y, lc) if lc is not None else None
    g_fv, g_lt = _upstream(B, F, lc, kink, seed)
    v = verts.to(DEV).requires_grad_(True)
    c = cams.to(DEV).requires_grad_(True)
    fv, lt = project_faces(v, c, faces.to(DEV), offset_z=5.0, eye_z=EYE_Z, viewing_scale=vs, flip_y=flip_y, light=lc)
    outs, grads = [fv], [g_fv.to(DEV)]
    if lt is not None:
        outs.append(lt)
        grads.append(g_lt.to(DEV))
    torch.autograd.backward(outs, grads)
    tag = "V%d F%d Bv%d H%d %s %s vs%g%s" % (V, F, Bv, H, layout, light, vs, "" if flip_y else " noflip")
    _compare_projection(tag, verts, cams, faces, vs, flip_y, lc, g_fv, g_lt, fv, lt, v.grad, c.grad)
    # the forward stays bit-identical to the drop-in's generic float32 torch chain
    X = v.detach().repeat_interleave(H, 0)
    p = geom_utils.orthographic_proj_withz(X, c.detach(), offset_z=5.0)
    if flip_y:
        p[:, :, 1] *= -1
    p = sr.functional.orthogonal(sr.functional.look_at(p, [0, 0, EYE_Z]), vs)
    fi = faces.to(DEV)
    fi = (fi[None] if fi.dim() == 2 else fi)
    fi = fi.expand(B, -1, -1) if fi.shape[0] == 1 else fi.repeat_interleave(H, 0)
    assert torch.equal(fv.detach(), sr.functional.face_vertices(p, fi)), "fused projection is not bit-identical"


@pytest.mark.parametrize("which", ["vertices", "cams", "expanded_vertices"])
def test_project_faces_partial_gradients(which):
    V, F, Bv, H = 300, 257, 4, 2
    verts, cams, faces = _case(V, F, Bv, H, "per_mesh", 5)
    lc = _f32(COLOUR_LIGHT)
    if which == "expanded_vertices":
        verts = verts[:1].expand(Bv, -1, -1)
    kink = _kink_faces(verts, cams, faces, True, lc)
    g_fv, g_lt = _upstream(Bv * H, F, lc, kink, 5)
    base = (verts[:1] if which == "expanded_vertices" else verts).to(DEV).requires_grad_(which != "cams")
    v = base.expand(Bv, -1, -1) if which == "expanded_vertices" else base
    c = cams.to(DEV).requires_grad_(which == "cams")
    fv, lt = project_faces(v, c, faces.to(DEV), offset_z=5.0, eye_z=EYE_Z, viewing_scale=1.0, flip_y=True, light=lc)
    torch.autograd.backward([fv, lt], [g_fv.to(DEV), g_lt.to(DEV)])
    assert (base.grad is None) == (which == "cams") and (c.grad is None) == (which != "cams")
    _compare_projection("partial " + which, verts, cams, faces, 1.0, True, lc, g_fv, g_lt, fv, lt, base.grad, c.grad,
                        vert_batch=Bv if which == "expanded_vertices" else None)


def test_project_faces_near_zero_normal_branch():
    """An identity camera and dyadic coordinates make the float32 projection exact, so only the light stage rounds.
    Face 0 has legs of 2^-10: |n| = 2^-20 < 1e-6, so the forward divides by the eps and the backward must take the
    plain G / eps branch (F.normalize's clamp has no gradient).  Face 1 is an ordinary lit face.  The light bounds
    use the exact corners (`exact_corners`), so they measure the light stage alone."""
    verts = torch.tensor([[[0.25, 0.5, 0.125], [0.25 + 2 ** -10, 0.5, 0.125], [0.25, 0.5 + 2 ** -10, 0.125],
                           [-0.5, 0.25, 0.375], [0.5, 0.375, -0.25]]])
    cams = torch.tensor([[1.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]])
    faces = torch.tensor([[0, 1, 2], [0, 3, 4]], dtype=torch.int32)
    lc = _f32((0.5, (1.0, 0.5, 0.25), 0.75, (0.25, 0.5, 1.0), (0.2, -0.3, -1.0)))
    n, N, _, _ = R.normal_conditioning(verts.double(), cams.double(), faces, 5.0, True)
    d = torch.tensor(lc[4], dtype=torch.float64)
    assert float(n[0, 0].norm()) < 1e-6 and float(n[0, 1].norm()) > 1e-6
    assert bool((((n / N[..., None]) * d).sum(2) > 1e-3).all()), "both faces must be lit"
    g_fv = torch.zeros(1, 2, 3, 3)
    g_lt = torch.tensor([[[1.0, -0.5, 0.75], [0.5, 1.0, -1.0]]])
    v = verts.to(DEV).requires_grad_(True)
    c = cams.to(DEV).requires_grad_(True)
    fv, lt = project_faces(v, c, faces.to(DEV), offset_z=5.0, eye_z=EYE_Z, viewing_scale=1.0, flip_y=True, light=lc)
    torch.autograd.backward([fv, lt], [g_fv.to(DEV), g_lt.to(DEV)])
    _compare_projection("near-zero normal", verts, cams, faces, 1.0, True, lc, g_fv, g_lt, fv, lt, v.grad, c.grad,
                        exact_corners=True)


def test_project_faces_65535_renders_and_the_limit():
    verts = torch.tensor([[[0.5, -0.25, 0.125], [-0.375, 0.5, 0.25], [0.125, 0.25, -0.5]]])
    faces = torch.tensor([[0, 1, 2]], dtype=torch.int32)
    g = torch.Generator().manual_seed(11)
    cams = _random_cams(g, 65535)
    lc = _f32(DEFAULT_LIGHT)
    kink = _kink_faces(verts, cams, faces, True, lc)
    g_fv, g_lt = _upstream(65535, 1, lc, kink, 11)
    v = verts.to(DEV).requires_grad_(True)
    c = cams.to(DEV).requires_grad_(True)
    fv, lt = project_faces(v, c, faces.to(DEV), offset_z=5.0, eye_z=EYE_Z, light=lc)
    torch.autograd.backward([fv, lt], [g_fv.to(DEV), g_lt.to(DEV)])
    _compare_projection("65535 renders", verts, cams, faces, 1.0, True, lc, g_fv, g_lt, fv, lt, v.grad, c.grad)
    with pytest.raises(RuntimeError, match="umr_project_faces_forward failed: size exceeds a compiled limit"):
        project_faces(v.detach(), torch.cat([c.detach(), c.detach()[:1]]), faces.to(DEV), light=lc)


class _Spy:
    """Keeps the (face_vertices, textures) our glue hands to the rasteriser, still attached to the graph."""

    def __enter__(self):
        self.calls, self.orig = [], raster.SoftRasterizeFunction.apply
        outer = self

        def spy(fv, tex, *a):
            outer.calls.append((fv, tex))
            return outer.orig(fv, tex, *a)
        raster.SoftRasterizeFunction.apply = staticmethod(spy)
        return self

    def __exit__(self, *exc):
        raster.SoftRasterizeFunction.apply = self.orig


# (V, F, Bv, H, face layout, light, viewing_scale, textures)
SMR_CASES = [
    (642, 1280, 2, 8, "per_mesh", "default", 1.0, True),
    (257, 257, 3, 2, "1", "colour", 0.75, False),
    (2562, 1280, 2, 1, "2d", "colour", 1.0, True),
    (300, 255, 4, 2, "per_mesh", "off", 0.75, True),
]


@pytest.mark.parametrize("V,F,Bv,H,layout,light,vs,with_tex", SMR_CASES)
def test_soft_renderer_fused_and_generic_match_float64(V, F, Bv, H, layout, light, vs, with_tex):
    """smr.SoftRenderer on the fused path and on the generic torch path (what runs under
    torch.use_deterministic_algorithms(True)), with the light set through sr.Lighting.  The loss is a random linear
    function of the face vertices and lit textures handed to the rasteriser, so the vertex and camera gradients are
    those of the vertex stage alone; the generic path is held to the kernel's bounds."""
    seed = V + F + Bv + H
    verts, cams, faces = _case(V, F, Bv, H, layout, seed)
    B = Bv * H
    g = torch.Generator().manual_seed(seed)
    tex = torch.rand(Bv, F, 4, 3, generator=g) if with_tex else None
    lc = _f32(LIGHTS[light])
    kink = _kink_faces(verts, cams, faces, True, lc) if lc is not None else torch.zeros(B, F, dtype=torch.bool)
    w1 = torch.randn(B, F, 3, 3, generator=g)
    w2 = torch.randn(B, F, 4 if with_tex else 1, 3, generator=g)
    w2[kink] = 0.0      # their light gradient depends on the relu branch
    t64 = tex.double().repeat_interleave(H, 0) if with_tex else torch.ones(B, F, 1, 3, dtype=torch.float64)
    if lc is not None:
        _, lt64 = R.project_faces_ref(verts.double(), cams.double(), faces, 5.0, EYE_Z, vs, True, lc)
        tex64 = t64 * lt64[:, :, None, :]
        tex_bound = t64.abs() * R.light_error_bound(verts.double(), cams.double(), faces, 5.0, True, lc)[:, :, None, :] \
            + gamma(1) * tex64.abs()
    else:
        tex64, tex_bound = t64, torch.zeros_like(t64)      # ambient_light_only: textures * 1
    g_lt = (t64 * w2.double()).sum(2).float()
    fvs = []
    for fused in (True, False):
        r = smr.SoftRenderer(16, "softmax")
        r.fuse_vertex_pipeline = fused
        if lc is None:
            r.ambient_light_only()
        elif light != "default":
            ia, ca, idr, cd, d = lc
            r.renderer.lighting = sr.Lighting(intensity_ambient=ia, color_ambient=ca, intensity_directionals=idr,
                                              color_directionals=cd, directions=d)
        r.renderer.transform.transformer.viewing_scale = vs
        v = verts.to(DEV).requires_grad_(True)
        c = cams.to(DEV).requires_grad_(True)
        with _Spy() as spy:
            r(v, faces.to(DEV), c, None if tex is None else tex.to(DEV))
        assert len(spy.calls) == 1
        fv, tx = spy.calls[0]
        fv = fv.reshape(B, F, 3, 3)
        # textures the hypotheses share reach the rasteriser once per mesh (or once for all), as the raster takes them
        tx = tx.expand(B, F, -1, 3) if tx.shape[0] == 1 else tx.repeat_interleave(B // tx.shape[0], 0)
        ((fv * w1.to(DEV)).sum() + (tx * w2.to(DEV)).sum()).backward()
        tag = "smr %s V%d F%d Bv%d H%d %s %s vs%g%s" % ("fused" if fused else "generic", V, F, Bv, H, layout, light,
                                                       vs, " tex" if with_tex else "")
        _check_bound(tag + " lit textures", tx, tex64, tex_bound)
        _compare_projection(tag, verts, cams, faces, vs, True, lc, w1, g_lt if lc is not None else None, fv, None,
                            v.grad, c.grad)
        fvs.append(fv.detach())
    assert torch.equal(fvs[0], fvs[1]), "fused projection is not bit-identical to the generic path"


def _corr_case(B, sizes, counts, mode, seed, V=642):
    """Part selections over V vertices (drawn with replacement across parts, so vertices repeat between parts),
    targets [B,m_g,2] and verts [1,V,3] ('shared'), an expanded stride-0 view ('expanded') or [B,V,3]."""
    g = torch.Generator().manual_seed(seed)
    parts = [torch.randint(0, V, (n,), generator=g) for n in sizes]
    targets = [(torch.rand(B, m, 2, generator=g) - 0.5).float() for m in counts]
    nv = 1 if mode != "per_render" else B
    verts = (1.4 * torch.rand(nv, V, 3, generator=g, dtype=torch.float64) - 0.7).float()
    cams = _random_cams(g, B)
    return parts, targets, verts, cams


def _corr_against_float64(tag, parts, targets, weights, verts, cams, loss, vert2d, nn, gl, gv2, got_gv, got_gc,
                          summed_renders=0):
    B, NS = cams.shape[0], vert2d.shape[1]
    vd, cd = verts.double().requires_grad_(True), cams.double().requires_grad_(True)
    t64 = [t.double() for t in targets]
    _, q64, idx64 = R.corr_chamfer_ref(vd, cd, parts, t64, weights)
    nn = nn.long().cpu()
    # an index that differs from the float64 argmin must be a near-tie (test_losses_gpu.py::test_chamfer)
    with torch.no_grad():
        qm = R.project_vertices(verts.double().abs()[:, torch.cat(parts)].expand(B, -1, -1), cams.double().abs())[..., :2]
        start = 0
        for p, t in zip(parts, t64):
            n = len(p)
            sl = slice(start, start + n)
            d = ((q64[:, sl, None, :] - t[:, None, :, :]) ** 2).sum(-1)
            dm = ((qm[:, sl, None, :] + t.abs()[:, None, :, :]) ** 2).sum(-1)   # magnitude of the expanded form
            pick = lambda x, i: torch.gather(x, 2, i[:, sl, None])[..., 0]   # noqa: E731
            tol = gamma(15) * (pick(dm, nn) + pick(dm, idx64))
            assert bool(((pick(d, nn) - pick(d, idx64)).abs() <= tol).all()), tag + ": nearest differs beyond a near-tie"
            start += n
    loss64, q64, _ = R.corr_chamfer_ref(vd, cd, parts, t64, weights, nearest=nn)
    gv, gc = torch.autograd.grad((loss64 * gl.double()).sum() + (q64 * gv2.double()).sum(), (vd, cd))
    va, ca = verts.double().abs().requires_grad_(True), cams.double().abs().requires_grad_(True)
    lm, qm, _ = R.corr_chamfer_ref(va, ca, parts, [t.abs() for t in t64], weights, nearest=nn, magnitude=True)
    mv, mc = torch.autograd.grad((lm * gl.double().abs()).sum() + (qm * gv2.double().abs()).sum(), (va, ca))
    _check(tag + " vert2d", vert2d, q64, qm, 10)
    _check(tag + " loss", loss, loss64, lm, 24 + math.ceil(NS / 8))
    mult = int(torch.bincount(torch.cat(parts)).max())
    if got_gv is not None:
        _check(tag + " grad vertices", got_gv, gv, mv, 26 + mult + summed_renders)
    if got_gc is not None:
        _check(tag + " grad cams", got_gc, gc, mc, 39 + math.ceil(NS / 256))


# (B, part sizes, target counts, weights, vertex mode, deterministic)
CORR_CASES = [
    (1, (1, 0, 0, 0), (1, 1, 1, 1), (1, 1, 0, 0), "per_render", False),
    (4, (100, 57, 60, 40), (31, 32, 33, 1), (1, 0, 0.5, 2), "shared", False),
    (128, (300, 200, 100, 100), (700, 33, 32, 31), (1, 1, 0, 0), "expanded", False),
    (8, (250, 250, 100, 100), (1, 31, 32, 33), (0, 1, 2, 0.25), "per_render", True),
    (3, (100, 57, 60, 40), (33, 700, 1, 32), (1, 1, 0, 0), "shared", True),
    (2, (0, 257, 0, 0), (5, 32, 5, 5), (1, 1, 1, 1), "expanded", True),
]


@pytest.mark.parametrize("B,sizes,counts,weights,mode,det", CORR_CASES)
def test_corr_chamfer_matches_float64(B, sizes, counts, weights, mode, det):
    parts, targets, verts, cams = _corr_case(B, sizes, counts, mode, seed=B + sum(sizes) + sum(counts))
    NS = sum(sizes)
    g = torch.Generator().manual_seed(NS)
    gl, gv2 = torch.randn(B, generator=g), torch.randn(B, NS, 2, generator=g)
    base = verts.to(DEV).requires_grad_(True)
    v = base.expand(B, -1, -1) if mode == "expanded" else base
    c = cams.to(DEV).requires_grad_(True)
    sel = torch.cat(parts).to(DEV)
    ends = np.cumsum(sizes).tolist()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        loss, vert2d = ops.corr_chamfer(v, c, sel, [t.to(DEV) for t in targets], ends, weights)
        nn = loss.grad_fn.saved_tensors[4]
        torch.autograd.backward([loss, vert2d], [gl.to(DEV), gv2.to(DEV)])
    finally:
        torch.use_deterministic_algorithms(prev)
    tag = "corr B%d NS%d m%s w%s %s%s" % (B, NS, counts, weights, mode, " det" if det else "")
    _corr_against_float64(tag, parts, targets, weights, verts, cams, loss, vert2d, nn, gl, gv2, base.grad, c.grad,
                          summed_renders=B if mode != "per_render" else 0)


@pytest.mark.parametrize("avg", [True, False])
def test_corr_loss_module_matches_float64(avg):
    B, sizes, counts = 5, (40, 80, 40, 80), (10, 30, 10, 30)
    parts, targets, verts, cams = _corr_case(B, sizes, counts, "per_render", seed=21)
    m = loss_utils.CorrLossChamfer(None, 64, part_vertices=parts)
    v = verts.to(DEV).requires_grad_(True)
    c = cams.to(DEV).requires_grad_(True)
    out = m(*[t.to(DEV) for t in targets], v, c, avg=avg)
    loss = out[0] if avg else out
    loss64, _, _ = R.corr_chamfer_ref(verts.double(), cams.double(), parts, [t.double() for t in targets])
    lm, _, _ = R.corr_chamfer_ref(verts.double().abs(), cams.double().abs(), parts, [t.double().abs() for t in targets],
                                  magnitude=True)
    D = 24 + math.ceil(sum(sizes) / 8)
    if avg:
        _check("CorrLossChamfer avg", loss.reshape(1), loss64.mean().reshape(1), lm.mean().reshape(1), D + B)
    else:
        _check("CorrLossChamfer per render", loss, loss64, lm, D)


@pytest.mark.parametrize("det", [False, True])
def test_corr_exact_ties_take_the_lowest_index(det):
    """Identity camera, dyadic coordinates: every projection and distance is exact in float32, so targets 1 and 2
    (lanes 1 and 2 of the warp) and targets 5 and 37 (both in lane 5) are exactly as near as each other.  torch.min
    returns the lowest index; so must the kernel, or the gradient goes to the wrong target."""
    B, V = 2, 4
    verts = torch.tensor([[[0.25, 0.5, 0.125], [-0.5, 0.25, 0.0], [0.125, -0.25, 0.5], [0.0, 0.0, 0.0]]]).expand(B, -1, -1)
    cams = torch.tensor([[1.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]]).repeat(B, 1)
    t0 = torch.full((B, 40, 2), 4.0)
    t0[:, 1] = torch.tensor([0.25 + 0.125, 0.5])       # vertex 0 at (0.25, 0.5): targets 1 and 2 at distance 1/8
    t0[:, 2] = torch.tensor([0.25, 0.5 - 0.125])
    t0[:, 0] = torch.tensor([0.25, 0.5 + 0.25])        # target 0 farther
    t0[:, 5] = torch.tensor([-0.5 - 0.25, 0.25])       # vertex 1 at (-0.5, 0.25): targets 5 and 37 at distance 1/4
    t0[:, 37] = torch.tensor([-0.5, 0.25 + 0.25])
    others = [torch.rand(B, 3, 2) for _ in range(3)]
    parts = [torch.tensor([0, 1]), torch.tensor([2]), torch.tensor([3]), torch.tensor([0])]
    v = verts.contiguous().to(DEV).requires_grad_(True)
    c = cams.to(DEV).requires_grad_(True)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        loss, vert2d = ops.corr_chamfer(v, c, torch.cat(parts).to(DEV), [t.to(DEV) for t in [t0] + others], [2, 3, 4, 5],
                                        (1, 1, 1, 1))
        nn = loss.grad_fn.saved_tensors[4].cpu()
        loss.sum().backward()
    finally:
        torch.use_deterministic_algorithms(prev)
    assert nn[:, 0].tolist() == [1] * B and nn[:, 1].tolist() == [5] * B, nn
    _, _, idx64 = R.corr_chamfer_ref(verts.double(), cams.double(), parts, [t.double() for t in [t0] + others],
                                     (1, 1, 1, 1))
    assert torch.equal(nn.long(), idx64)
    _corr_against_float64("corr exact ties" + (" det" if det else ""), parts, [t0] + others, (1, 1, 1, 1),
                          verts.contiguous(), cams, loss, vert2d, nn, torch.ones(B), torch.zeros(B, 5, 2), v.grad,
                          c.grad)
