"""Host-side contract of the silhouette render (no GPU): the entry points are exported and refuse what they do not cover
before touching the device, `soft_rasterize_silhouettes` refuses float64, `SoftRenderer.render_silhouettes` takes one
projection without lighting and one silhouette raster in the fused configuration and the full render's alpha plane
elsewhere, and `MultiMaskLoss` routes through it."""
import ctypes

import pytest
import torch

from umr_b200 import _lib, raster
from umr_b200.nnutils import loss_utils, smr

FORWARD = ("umr_raster_forward_silhouette", "umr_raster_forward_silhouette_deterministic")
BACKWARD = ("umr_raster_backward_silhouette", "umr_raster_backward_silhouette_deterministic")
UMR_OK, UMR_ERR_UNSUPPORTED, UMR_ERR_BAD_ARG = 0, -1, -2


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def test_symbols_exported(lib):
    for name in FORWARD + BACKWARD:
        assert name in _lib.EXPORTS
        assert getattr(lib, name) is not None
        assert name + "_f64" not in _lib.EXPORTS   # float64 meshes take the full render
    assert lib.umr_version() == 204


def _params(**kw):
    cfg = dict(B=2, F=4, T2=1, image_size=8, anti_aliasing=False, background_color=(0, 0, 0), near=1, far=100,
               fill_back=True, eps=1e-3, sigma_val=1e-5, dist_func="euclidean", dist_eps=1e-4, gamma_val=1e-4,
               aggr_func_rgb="softmax", aggr_func_alpha="prod", texture_type="surface")
    cfg.update(kw)
    return raster.make_params(**cfg)


FAKE = ctypes.c_void_p(256)        # a non-NULL, aligned pointer: every case below is refused before a buffer is touched
ODD = ctypes.c_void_p(256 + 2)     # not 4-byte aligned


def _fwd(lib, name, p, fv=FAKE, alpha=FAKE, alpha_hi=FAKE, ws=FAKE):
    return getattr(lib, name)(fv, alpha, alpha_hi, ctypes.byref(p) if p is not None else None, ws, None)


def _bwd(lib, name, p, fv=FAKE, alpha_hi=FAKE, g=FAKE, gf=FAKE, ws=FAKE):
    return getattr(lib, name)(fv, alpha_hi, g, gf, ctypes.byref(p) if p is not None else None, ws, None)


CALLS = [(n, _fwd) for n in FORWARD] + [(n, _bwd) for n in BACKWARD]


@pytest.mark.parametrize("name,call", CALLS)
@pytest.mark.parametrize("mode", [dict(dist_func="barycentric"), dict(dist_func="hard"), dict(aggr_func_alpha="sum"),
                                  dict(aggr_func_alpha="hard"), dict(texture_type="vertex", T2=3)])
def test_generic_modes_are_refused(lib, name, call, mode):
    assert call(lib, name, _params(**mode)) == UMR_ERR_BAD_ARG


@pytest.mark.parametrize("name,call", CALLS)
def test_four_channels_are_refused(lib, name, call):
    p = _params()
    p.color_channels = 4
    assert call(lib, name, p) == UMR_ERR_BAD_ARG


@pytest.mark.parametrize("name,call", CALLS)
def test_params_are_checked_first(lib, name, call):
    assert call(lib, name, None) == UMR_ERR_BAD_ARG
    p = _params()
    p.batch_size = 0
    assert call(lib, name, p) == UMR_ERR_BAD_ARG
    p = _params()
    p.func_id_rgb = 7
    assert call(lib, name, p) == UMR_ERR_UNSUPPORTED


@pytest.mark.parametrize("name", FORWARD)
def test_forward_null_and_misaligned_buffers_are_refused(lib, name):
    p = _params()
    for kw in (dict(fv=None), dict(alpha=None), dict(ws=None), dict(fv=ODD), dict(alpha=ODD), dict(alpha_hi=ODD),
               dict(ws=ctypes.c_void_p(256 + 16))):
        assert _fwd(lib, name, p, **kw) == UMR_ERR_BAD_ARG, kw


@pytest.mark.parametrize("name", BACKWARD)
def test_backward_null_and_misaligned_buffers_are_refused(lib, name):
    p = _params()
    for kw in (dict(fv=None), dict(alpha_hi=None), dict(g=None), dict(gf=None), dict(ws=None), dict(fv=ODD),
               dict(alpha_hi=ODD), dict(g=ODD), dict(gf=ODD), dict(ws=ctypes.c_void_p(256 + 16))):
        assert _bwd(lib, name, p, **kw) == UMR_ERR_BAD_ARG, kw


def test_kernel_mode_resolves_the_silhouette_symbols():
    for name in ("umr_raster_forward_silhouette", "umr_raster_backward_silhouette"):
        assert raster.KernelMode(False).symbol(name, True)[1] == name
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(True)
        try:
            assert raster.KernelMode(False).symbol(name, True)[1] == name + "_deterministic"
        finally:
            torch.use_deterministic_algorithms(prev)


def test_silhouette_function_refuses_float64_and_cpu_tensors():
    with pytest.raises(TypeError):
        raster.soft_rasterize_silhouettes(torch.zeros(1, 2, 3, 3), 8)
    with pytest.raises((TypeError, ValueError)):
        raster.soft_rasterize_silhouettes(torch.zeros(1, 2, 3, 3, dtype=torch.float64), 8)


def test_raster_calls_wrapped_follows_apply():
    cls = raster.SoftRasterizeFunction
    had = "apply" in cls.__dict__
    saved = cls.__dict__.get("apply")
    orig = cls.apply
    assert not raster.raster_calls_wrapped()
    try:
        cls.apply = staticmethod(lambda *a: orig(*a))
        assert raster.raster_calls_wrapped()
        cls.apply = orig   # a capture that restores the attribute it read
        assert not raster.raster_calls_wrapped()
    finally:
        if had:
            cls.apply = saved
        else:
            del cls.apply
    assert not raster.raster_calls_wrapped()


# --- render_silhouettes dispatch through a fake rasteriser --------------------------------------------------------------
class _Recorder(object):
    """Differentiable stand-ins for the projection and the rasteriser (alpha a function of the geometry), so the dispatch
    and the gradient routes are visible on CPU tensors."""

    def __init__(self, monkeypatch, renderer, fused):
        self.calls = []
        self.size = renderer.renderer.rasterizer.image_size
        rz = renderer.renderer.rasterizer
        monkeypatch.setattr(rz, "rasterize", self._raster("rasterize"), raising=False)
        monkeypatch.setattr(rz, "rasterize_silhouettes", self._silhouettes, raising=False)
        if fused:
            monkeypatch.setattr(smr.SoftRenderer, "_fusable", lambda self, v: True)
            monkeypatch.setattr(smr, "project_faces", self._project)

    def _project(self, vertices, cams, faces, **kw):
        self.calls.append(("project_faces", kw.get("light")))
        H = cams.shape[0] // vertices.shape[0]
        v = vertices.repeat_interleave(H, dim=0) * cams[:, None, :1]
        fv = torch.stack([v[b][faces[b // H].long()] for b in range(cams.shape[0])])
        return fv, None

    def _alpha(self, fv):
        B, S = fv.shape[0], self.size
        return torch.sigmoid(fv.reshape(B, -1).sum(1) / 100).view(B, 1, 1).expand(B, S, S)

    def _raster(self, name):
        def run(fv, tex):
            self.calls.append((name, None))
            B, S = fv.shape[0], self.size
            rgb = (fv.reshape(B, -1).sum(1) + tex.reshape(tex.shape[0], -1).sum(1).mean()).view(B, 1, 1, 1).expand(B, 3, S, S)
            return torch.cat((rgb, self._alpha(fv)[:, None]), 1), torch.zeros(B, fv.shape[1], 2), torch.zeros(B, 2, S, S)
        return run

    def _silhouettes(self, fv):
        self.calls.append(("rasterize_silhouettes", None))
        return self._alpha(fv)


def _inputs(B=2, H=4, V=6, F=5):
    g = torch.Generator().manual_seed(0)
    vs = torch.rand(B, V, 3, generator=g).requires_grad_(True)
    fs = torch.randint(0, V, (B, F, 3), generator=g)
    cams = torch.rand(B * H, 7, generator=g).requires_grad_(True)
    return vs, fs, cams


@pytest.mark.parametrize("fused", [True, False])
def test_render_silhouettes_dispatch(monkeypatch, fused):
    r = smr.SoftRenderer(8, "softmax")   # the mask renderer keeps its directional light: the silhouette projects without it
    rec = _Recorder(monkeypatch, r, fused)
    vs, fs, cams = _inputs()
    alpha = r.render_silhouettes(vs, fs, cams)
    assert alpha.shape == (cams.shape[0], 8, 8)
    if fused:
        assert rec.calls == [("project_faces", None), ("rasterize_silhouettes", None)]
    else:
        assert rec.calls == [("rasterize", None)]   # the full render, alpha plane kept
    g_v, g_c = torch.autograd.grad(alpha.sum(), (vs, cams))
    assert g_v.abs().sum() > 0 and g_c.abs().sum() > 0


def test_render_silhouettes_fallback_equals_the_full_alpha(monkeypatch):
    r = smr.SoftRenderer(8, "softmax")
    _Recorder(monkeypatch, r, fused=False)
    vs, fs, cams = _inputs()
    assert torch.equal(r.render_silhouettes(vs, fs, cams), r(vs, fs, cams)[0][:, 3])


@pytest.mark.parametrize("change", [dict(aggr_func_alpha="sum"), dict(dist_func="barycentric"), "wrapped"])
def test_render_silhouettes_outside_its_kernels_renders_in_full(monkeypatch, change):
    r = smr.SoftRenderer(8, "softmax")
    if change == "wrapped":
        orig = raster.SoftRasterizeFunction.apply
        monkeypatch.setattr(raster.SoftRasterizeFunction, "apply", staticmethod(lambda *a: orig(*a)))
    else:
        for k, v in change.items():
            setattr(r.renderer.rasterizer, k, v)
    assert not r.renderer.rasterizer.supports_silhouettes()
    rec = _Recorder(monkeypatch, r, fused=True)
    vs, fs, cams = _inputs()
    r.render_silhouettes(vs, fs, cams)
    assert [c[0] for c in rec.calls] == ["project_faces", "rasterize"]


def test_supports_silhouettes_in_umr_configuration():
    for render_type in ("softmax", "hard"):
        assert smr.SoftRenderer(16, render_type).renderer.rasterizer.supports_silhouettes()


# --- MultiMaskLoss -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused", [True, False])
def test_multi_mask_loss_routes_through_render_silhouettes(monkeypatch, fused):
    H = 4
    # the IoU kernel is CUDA-only: a torch restatement (loss_utils.py:41-48, avg=False) on CPU tensors
    monkeypatch.setattr(loss_utils, "neg_iou_loss", lambda p, t, avg=True: 1 - (p * t).sum((1, 2)) / (p + t - p * t).sum((1, 2)))
    m = loss_utils.MultiMaskLoss(8, "softmax", H)
    rec = _Recorder(monkeypatch, m.renderer, fused)
    vs, fs, cams = _inputs(H=H)
    probs = torch.softmax(torch.rand(2, H), 1).requires_grad_(True)
    masks = (torch.rand(2, 8, 8) > 0.5).float()
    loss, mask_all = m(vs, fs, cams.view(2, H, 7), probs, masks)
    assert mask_all.shape == (2 * H, 8, 8)
    assert [c[0] for c in rec.calls] == (["project_faces", "rasterize_silhouettes"] if fused else ["rasterize"])
    # the loss of the alpha plane the renderer returned
    ref = loss_utils.expected_over_hypotheses(loss_utils.neg_iou_loss(mask_all, loss_utils.tile_hypotheses(masks, H),
                                                                      avg=False), probs)
    assert torch.equal(loss, ref)
    g_v, g_c, g_p = torch.autograd.grad(loss, (vs, cams, probs))
    assert g_v.abs().sum() > 0 and g_c.abs().sum() > 0 and g_p.abs().sum() > 0
