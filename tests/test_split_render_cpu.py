"""Host-side contract of the split raster backward (no GPU): the entry points are exported and refuse what they do not
cover before touching the device, `soft_rasterize_split` refuses float64 and the generic modes, `SoftRenderer.render_split`
takes one projection and one split raster in the fused configuration and two ordinary renders elsewhere, and
`MultiMaskTextureLoss` builds with train_s2's arguments."""
import ctypes

import pytest
import torch

from umr_b200 import _lib, raster
from umr_b200.nnutils import loss_utils, smr

ENTRY_POINTS = ("umr_raster_backward_split", "umr_raster_backward_split_deterministic")
UMR_OK, UMR_ERR_UNSUPPORTED, UMR_ERR_BAD_ARG = 0, -1, -2


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def test_symbols_exported(lib):
    for name in ENTRY_POINTS:
        assert name in _lib.EXPORTS
        assert getattr(lib, name) is not None
    assert lib.umr_version() == 204


def test_error_codes_match_header():
    with open(_lib.os.path.join(_lib.os.path.dirname(_lib._PKG), "include", "umr_b200.h")) as fh:
        text = fh.read()
    assert "#define UMR_ERR_BAD_ARG (%d)" % UMR_ERR_BAD_ARG in text
    assert "#define UMR_ERR_UNSUPPORTED (%d)" % UMR_ERR_UNSUPPORTED in text


def _params(**kw):
    cfg = dict(B=2, F=4, T2=4, image_size=8, anti_aliasing=False, background_color=(0, 0, 0), near=1, far=100,
               fill_back=True, eps=1e-3, sigma_val=1e-5, dist_func="euclidean", dist_eps=1e-4, gamma_val=1e-4,
               aggr_func_rgb="softmax", aggr_func_alpha="prod", texture_type="surface")
    cfg.update(kw)
    return raster.make_params(**cfg)


FAKE = ctypes.c_void_p(256)   # a non-NULL pointer: every case below is refused before a buffer is touched


def _call(lib, name, p, grad_faces=FAKE, grad_tex=FAKE):
    return getattr(lib, name)(FAKE, FAKE, FAKE, FAKE, FAKE, grad_faces, grad_tex, ctypes.byref(p), FAKE, None)


@pytest.mark.parametrize("name", ENTRY_POINTS)
def test_both_outputs_are_required(lib, name):
    p = _params()
    assert _call(lib, name, p, grad_faces=None) == UMR_ERR_BAD_ARG
    assert _call(lib, name, p, grad_tex=None) == UMR_ERR_BAD_ARG
    assert _call(lib, name, p, grad_faces=None, grad_tex=None) == UMR_ERR_BAD_ARG


@pytest.mark.parametrize("name", ENTRY_POINTS)
@pytest.mark.parametrize("mode", [dict(dist_func="barycentric"), dict(dist_func="hard"), dict(aggr_func_alpha="sum"),
                                  dict(aggr_func_alpha="hard"), dict(texture_type="vertex", T2=3)])
def test_generic_modes_are_refused(lib, name, mode):
    assert _call(lib, name, _params(**mode)) == UMR_ERR_BAD_ARG


@pytest.mark.parametrize("name", ENTRY_POINTS)
def test_four_channels_are_refused(lib, name):
    p = _params()
    p.color_channels = 4
    assert _call(lib, name, p) == UMR_ERR_BAD_ARG


@pytest.mark.parametrize("name", ENTRY_POINTS)
def test_params_are_checked_first(lib, name):
    assert getattr(lib, name)(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None, FAKE, None) == UMR_ERR_BAD_ARG
    p = _params()
    p.batch_size = 0
    assert _call(lib, name, p) == UMR_ERR_BAD_ARG
    p = _params()
    p.func_id_rgb = 7
    assert _call(lib, name, p) == UMR_ERR_UNSUPPORTED


def test_kernel_mode_resolves_the_split_symbols():
    assert raster.KernelMode(False).symbol("umr_raster_backward_split", True)[1] == "umr_raster_backward_split"
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        assert raster.KernelMode(False).symbol("umr_raster_backward_split", True)[1] == \
            "umr_raster_backward_split_deterministic"
    finally:
        torch.use_deterministic_algorithms(prev)


@pytest.mark.parametrize("kw,dtype,nc", [({}, torch.float64, 3), (dict(dist_func="barycentric"), torch.float32, 3),
                                         (dict(aggr_func_alpha="sum"), torch.float32, 3),
                                         (dict(texture_type="vertex"), torch.float32, 3), ({}, torch.float32, 4)])
def test_split_function_refuses_what_it_does_not_cover(kw, dtype, nc):
    fv = torch.zeros(1, 2, 3, 3, dtype=dtype)
    tex = torch.zeros(1, 2, 4, nc, dtype=dtype)
    with pytest.raises(ValueError):
        raster.soft_rasterize_split(fv, tex, 8, **kw)


def test_split_function_keeps_its_own_apply():
    """Wrapping SoftRasterizeFunction.apply and putting the saved attribute back (as call-capturing tests do) leaves a
    method bound to SoftRasterizeFunction in that class's dict; the split Function must still run its own forward and
    backward."""
    cls = raster.SoftRasterizeFunction
    had = "apply" in cls.__dict__
    saved = cls.__dict__.get("apply")
    orig = cls.apply
    try:
        cls.apply = staticmethod(lambda *a: orig(*a))
        cls.apply = orig
        assert not issubclass(raster.SoftRasterizeSplitFunction, cls)
        assert raster.SoftRasterizeSplitFunction.apply.__self__ is raster.SoftRasterizeSplitFunction
        with pytest.raises(ValueError):   # the split Function's own forward: float64 is refused before any device work
            raster.soft_rasterize_split(torch.zeros(1, 2, 3, 3, dtype=torch.float64), torch.zeros(1, 2, 4, 3,
                                                                                                  dtype=torch.float64), 8)
    finally:
        if had:
            cls.apply = saved
        else:
            del cls.apply


def test_split_function_needs_cuda_tensors():
    with pytest.raises(TypeError):
        raster.soft_rasterize_split(torch.zeros(1, 2, 3, 3), torch.zeros(1, 2, 4, 3), 8)


# --- render_split dispatch through a fake rasteriser ------------------------------------------------------------------
class _Recorder(object):
    """Differentiable stand-ins for the projection and the rasteriser: alpha is a function of the geometry only, RGB of
    the geometry and the textures, so the gradient routes are visible on CPU tensors."""

    def __init__(self, monkeypatch, renderer, fused):
        self.calls = []
        self.size = renderer.renderer.rasterizer.image_size
        rz = renderer.renderer.rasterizer
        monkeypatch.setattr(rz, "rasterize", self._raster("rasterize"), raising=False)
        monkeypatch.setattr(rz, "rasterize_split", self._raster("rasterize_split"), raising=False)
        if fused:
            monkeypatch.setattr(smr.SoftRenderer, "_fusable", lambda self, v: True)
            monkeypatch.setattr(smr, "project_faces", self._project)

    def _project(self, vertices, cams, faces, **kw):
        self.calls.append("project_faces")
        H = cams.shape[0] // vertices.shape[0]
        v = vertices.repeat_interleave(H, dim=0) * cams[:, None, :1]
        fv = v[:, faces.reshape(-1, 3).long()].reshape(cams.shape[0], -1, 3, 3) if faces.dim() == 2 else \
            torch.stack([v[b][faces[b // H].long()] for b in range(cams.shape[0])])
        return fv, None

    def _raster(self, name):
        def run(fv, tex):
            self.calls.append(name)
            B, S = fv.shape[0], self.size
            geo = fv.reshape(B, -1).sum(1)
            t = tex.reshape(tex.shape[0], -1).sum(1)
            t = t.repeat_interleave(B // t.shape[0]) if t.shape[0] not in (1, B) else t.expand(B)
            rgb = (geo + t).view(B, 1, 1, 1).expand(B, 3, S, S)
            alpha = torch.sigmoid(geo / 100).view(B, 1, 1, 1).expand(B, 1, S, S)
            if name == "rasterize_split":   # the split backward: alpha -> geometry, RGB -> textures
                rgb = (geo.detach() + t).view(B, 1, 1, 1).expand(B, 3, S, S)
            images = torch.cat((rgb, alpha), 1)
            return images, torch.zeros(B, fv.shape[1], 2), torch.zeros(B, 2, S, S)
        return run


def _inputs(B=2, H=4, V=6, F=5, T2=4):
    g = torch.Generator().manual_seed(0)
    vs = torch.rand(B, V, 3, generator=g).requires_grad_(True)
    fs = torch.randint(0, V, (B, F, 3), generator=g)
    cams = torch.rand(B * H, 7, generator=g).requires_grad_(True)
    tex = torch.rand(B, F, T2, 3, generator=g).requires_grad_(True)
    return vs, fs, cams, tex


@pytest.mark.parametrize("fused", [True, False])
def test_render_split_dispatch_and_gradient_routes(monkeypatch, fused):
    r = smr.SoftRenderer(8, "softmax")
    r.ambient_light_only()
    rec = _Recorder(monkeypatch, r, fused)
    vs, fs, cams, tex = _inputs()
    images, p2f, aggrs = r.render_split(vs, fs, cams, tex)
    assert images.shape == (cams.shape[0], 4, 8, 8)
    if fused:
        assert rec.calls == ["project_faces", "rasterize_split"]
    else:
        assert rec.calls == ["rasterize", "rasterize"]   # alpha of the live geometry, RGB of the detached one
    # RGB reaches the textures only
    g_v, g_c, g_t = torch.autograd.grad(images[:, :3].sum(), (vs, cams, tex), allow_unused=True)
    assert g_v is None or not g_v.any()
    assert g_c is None or not g_c.any()
    assert g_t is not None and g_t.abs().sum() > 0
    # alpha reaches the geometry and cameras, not the textures
    images, _, _ = r.render_split(vs, fs, cams, tex)
    g_v, g_c, g_t = torch.autograd.grad(images[:, 3].sum(), (vs, cams, tex), allow_unused=True)
    assert g_v.abs().sum() > 0 and g_c.abs().sum() > 0
    assert g_t is None or not g_t.any()


def test_render_split_outside_umr_configuration_composes(monkeypatch):
    r = smr.SoftRenderer(8, "softmax")
    r.renderer.rasterizer.aggr_func_alpha = "sum"   # no split kernel: two ordinary renders even when fusable
    assert not r.renderer.rasterizer.supports_split()
    rec = _Recorder(monkeypatch, r, fused=True)
    vs, fs, cams, tex = _inputs()
    r.render_split(vs, fs, cams, tex)
    assert rec.calls == ["project_faces", "rasterize", "project_faces", "rasterize"]


# --- MultiMaskTextureLoss ------------------------------------------------------------------------------------------------
def test_multi_mask_texture_loss_builds_with_train_s2_arguments():
    # train_s2.py:130-148: MultiMaskLoss(image_size, renderer_type, num_hypo_cams), MultiTextureLoss(batch_size / gpu_num)
    m = loss_utils.MultiMaskTextureLoss(16, num_hypo_cams=8, image_size=256, renderer_type="softmax", texture_loss_type="l1")
    assert isinstance(m.mask_loss_fn, loss_utils.MultiMaskLoss)
    assert isinstance(m.texture_loss_fn, loss_utils.MultiTextureLoss)
    assert m.mask_loss_fn.num_hypo_cams == m.texture_loss_fn.num_hypo_cams == m.num_hypo_cams == 8
    mr, tr = m.mask_loss_fn.renderer.renderer, m.texture_loss_fn.renderer.renderer
    for key in ("image_size", "sigma_val", "gamma_val", "eps", "dist_eps", "anti_aliasing", "aggr_func_rgb",
                "aggr_func_alpha", "dist_func", "texture_type", "near", "far", "fill_back"):
        assert getattr(mr.rasterizer, key) == getattr(tr.rasterizer, key), key
    assert tr.lighting.directionals[0].light_intensity == 0 and tr.lighting.ambient.light_intensity == 1
    assert tr.rasterizer.supports_split()
    n = loss_utils.MultiMaskTextureLoss(16, texture_loss_type="l1", renderer="nmr")
    assert isinstance(n.texture_loss_fn.renderer, loss_utils.NeuralRenderer)
