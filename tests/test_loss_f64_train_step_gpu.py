"""The train_s2-shaped loss step in float64 on the GPU against the CPU oracle composed in double.

The loss modules of `tests/test_train_step_gpu.py` (MultiMaskLoss, MultiTextureLoss(..., "l1", "smr"), CorrLossChamfer,
part_matching_loss) with its scene and constructor arguments, and LaplacianLoss / FlattenLoss as the step of
`tests/test_deterministic_losses_gpu.py` composes them, run with float64 leaves.  Every loss value and every leaf gradient
must be float64 and agree with `oracle/train_step.py`'s compositions over oracle B's double instantiation
(`oracle/softras.py`, dtype=float64), with the same exact-input protocol as the float32 test: the oracle rasterises the
face vertices the GPU path handed to its rasteriser (captured), and gradients flow through the oracle's own vertex chain.

Two inputs of the double oracle are set as in `tests/test_raster_f64_gpu.py`: the p2f grid is the kernels' (torch's
float32 linspace by its per-element definition), and the renderers' `eps` is one at which the device's float `expf` and
glibc's agree (the softmax seed expf(eps / gamma) is a float expression in the reference's double instantiation too).

Tolerances: rtol 1e-11 and 1e-11 of the largest reference value.  The float32 step differs from the float64 one by 1e-5
in the loss values and 0.2-1 % in the gradients (DESIGN.md §10), so this separates the two by six orders of magnitude or
more; the double renders are held to the same 1e-11 against oracle B (DESIGN.md §9).
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

import loss_ref as R
import softras
import train_step as O  # oracle/train_step.py (test infrastructure)
from test_train_step_gpu import Capture, _scene   # the float32 test's scene and face-vertex capture
from umr_b200 import soft_renderer as sr, synth
from umr_b200.nnutils import geom_utils, loss_utils
from util import rel_report

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D = torch.float64
B, H, IS, T = 2, 8, 32, 3


def kernel_grid(S, dtype=np.float64):
    """The kernels' p2f grid: torch's float32 linspace(-1, 1, S) by its per-element definition, widened."""
    step = np.float32(2.0) / np.float32(S - 1)
    i = np.arange(S)
    lo = (np.float32(-1.0) + step * i.astype(np.float32)).astype(np.float32)
    hi = (np.float32(1.0) - step * (S - 1 - i).astype(np.float32)).astype(np.float32)
    x = np.where(i * 2 < S, lo, hi)
    return np.ascontiguousarray(np.stack(np.broadcast_arrays(x[None, :], x[:, None]), axis=-1).astype(dtype))


def eps_for_oracle(gamma=1e-4):
    """An eps for which the device's expf(eps / gamma) equals glibc's."""
    libm = ctypes.CDLL("libm.so.6")
    libm.expf.restype, libm.expf.argtypes = ctypes.c_float, [ctypes.c_float]
    for eps in (1e-3, 2e-3, 5e-4, 1.5e-3, 3e-3, 7e-4, 1e-4):
        q = np.float32(eps) / np.float32(gamma)
        if float(torch.exp(torch.tensor(float(q), dtype=torch.float32, device=DEV))) == libm.expf(float(q)):
            return eps
    raise AssertionError("no eps found")


@pytest.fixture(autouse=True)
def _oracle_on_the_kernel_grid(monkeypatch):
    monkeypatch.setattr(softras, "standard_grid", kernel_grid)


class _Override(torch.autograd.Function):
    """The captured values exactly, with the identity gradient towards the oracle's own face vertices."""

    @staticmethod
    def forward(ctx, x, v):
        return v.clone()

    @staticmethod
    def backward(ctx, g):
        return g, None


class _Rasterize64(torch.autograd.Function):
    """SoftRasterizer.forward / backward (anti-aliased) over oracle B's double instantiation."""

    @staticmethod
    def forward(ctx, fv, tex, image_size, rgb, kw):
        cfg = softras.RasterCfg(image_size * 2, aggr_func_rgb=rgb, **kw)
        fwd = softras.forward(fv.detach().numpy().reshape(fv.shape[0], -1, 9), tex.detach().numpy(), cfg, impl="B",
                              dtype=np.float64)
        ctx.fwd, ctx.cfg, ctx.shape = fwd, cfg, tuple(fv.shape)
        p2f, aggr = torch.from_numpy(fwd["p2f_info"].copy()), torch.from_numpy(fwd["aggrs_info"].copy())
        ctx.mark_non_differentiable(p2f, aggr)
        return torch.from_numpy(np.ascontiguousarray(softras.avg_pool2(fwd["soft_colors"]))), p2f, aggr

    @staticmethod
    def backward(ctx, g, _gp, _ga):
        ghi = softras.avg_pool2_backward(np.ascontiguousarray(g.numpy(), np.float64))
        gf, gt = softras.backward(ctx.fwd, ghi, ctx.cfg, impl="B")
        return torch.from_numpy(gf).view(ctx.shape), torch.from_numpy(gt), None, None, None


class OracleRenderer64(O.OracleSoftRenderer):
    """oracle/train_step.py's renderer with the light and the raster in double (the package creates its lighting
    constants in float64 beside float64 vertices)."""

    def __init__(self, img_size, render_type, eps):
        super().__init__(img_size, render_type)
        self.kw = dict(O.UMR_KW, eps=eps)

    def __call__(self, vertices, faces, cams, textures=None):
        fv, pre = self.face_vertices(vertices, faces, cams)
        nb, nf = fv.shape[:2]
        if textures is None:
            textures = torch.ones(nb, nf, 1, 3, dtype=D)
        light = torch.full((nb, nf, 3), self.ambient, dtype=D)
        if self.directional != 0.0:
            n = TF.normalize(torch.cross(pre[:, :, 2] - pre[:, :, 1], pre[:, :, 0] - pre[:, :, 1], dim=2), p=2, dim=2,
                             eps=1e-6)
            light = light + self.directional * TF.relu((n * torch.tensor([0., 1., 0.], dtype=D)).sum(dim=2))[:, :, None]
        textures = textures.to(D) * light[:, :, None, :]
        ov = torch.from_numpy(np.asarray(self.overrides[self.used], np.float64)).view_as(fv)
        self.used += 1
        return _Rasterize64.apply(_Override.apply(fv, ov), textures, self.img_size, self.render_type, self.kw)

    forward = __call__


def _wide(t):
    return t.detach().to(D)


def _leaf(t, dev=None):
    t = _wide(t).clone()
    return (t.to(dev) if dev else t).requires_grad_(True)


def _set_eps(*renderers, eps):
    for r in renderers:
        r.rasterizer.eps = eps


def _cmp(name, got, ref, rtol=1e-11, ascale=1e-11):
    assert got.dtype == D, "%s is %s" % (name, got.dtype)
    got, ref = got.detach().cpu().numpy(), ref.detach().cpu().numpy()
    ok, msg = rel_report(name, got, ref, rtol, ascale * float(np.abs(ref).max()) + 1e-300)
    print(msg)
    assert ok and np.isfinite(got).all(), msg


def test_multi_mask_loss_f64():
    d, eps = _scene(), eps_for_oracle()
    m = loss_utils.MultiMaskLoss(IS, "softmax", H).to(DEV)
    _set_eps(m.renderer.renderer, eps=eps)
    vs, cams, probs = _leaf(d["vs"], DEV), _leaf(d["cams"], DEV), _leaf(d["probs"], DEV)
    with Capture() as cap:
        loss, mask_all = m(vs, d["fs"].to(DEV), cams, probs, _wide(d["masks"]).to(DEV))
    loss.backward()
    r = OracleRenderer64(IS, "softmax", eps)
    r.overrides = cap.fv
    ovs, ocams, oprobs = _leaf(d["vs"]), _leaf(d["cams"]), _leaf(d["probs"])
    oloss, omask = O.multi_mask_loss(r, ovs, d["fs"], ocams, oprobs, _wide(d["masks"]), H)
    oloss.backward()
    assert r.used == len(cap.fv) == 1
    _cmp("mask_loss", loss, oloss)
    _cmp("mask_all_hypo", mask_all, omask)
    _cmp("d/dverts", vs.grad, ovs.grad)
    _cmp("d/dcams", cams.grad, ocams.grad)
    _cmp("d/dcam_probs", probs.grad, oprobs.grad)


def test_multi_texture_loss_f64():
    d, eps = _scene(seed=22), eps_for_oracle()
    fs = d["fs"].to(DEV)
    masks_pred = _wide(torch.rand(B * H, IS, IS, generator=torch.Generator().manual_seed(3)))
    m = loss_utils.MultiTextureLoss(B, H, IS, "softmax", "l1", "smr").to(DEV)
    _set_eps(m.renderer.renderer, m.hard_renderer.renderer, eps=eps)
    flow = _leaf(d["flow"], DEV)
    imgs, masks, dts, vs, cams, probs = [_wide(d[k]) for k in ("imgs", "masks", "dts", "vs", "cams", "probs")]
    tx = geom_utils.sample_textures(flow, imgs.to(DEV)).contiguous().view(B, d["F"], T * T, 3)
    with Capture() as cap:
        out = m(vs.to(DEV), fs, cams.to(DEV), probs.to(DEV), cams[:, 0].to(DEV), imgs.to(DEV), masks.to(DEV),
                masks_pred.to(DEV), tx, flow, dts.to(DEV))
    tl, tdt, tcyc, pred = out
    (3.0 * tl + 3.0 * tdt + 1.0 * tcyc).backward()
    r, rh = OracleRenderer64(IS, "softmax", eps), OracleRenderer64(IS, "hard", eps)
    r.ambient_light_only()
    r.overrides, rh.overrides = cap.fv[0:1], cap.fv[1:2]
    oflow = _leaf(d["flow"])
    otx = O.L.sample_textures(oflow, imgs).contiguous().view(B, d["F"], T * T, 3)
    otl, otdt, otcyc, opred = O.multi_texture_loss(r, rh, vs, d["fs"], cams, probs, cams[:, 0], imgs, masks, masks_pred,
                                                   otx, oflow, dts, H)
    (3.0 * otl + 3.0 * otdt + 1.0 * otcyc).backward()
    assert len(cap.fv) == 2 and r.used == 1 and rh.used == 1
    _cmp("tex_loss", tl, otl)
    _cmp("tex_dt_loss", tdt, otdt)
    _cmp("tex_cycle_loss", tcyc, otcyc)
    _cmp("texture_pred", pred, opred)
    _cmp("d/dtex_flow", flow.grad, oflow.grad)


def test_corr_loss_chamfer_f64():
    d = _scene(seed=23)
    m = loss_utils.CorrLossChamfer(None, IS, part_vertices=[torch.from_numpy(p) for p in d["part_vertices"]])
    rep = lambda t: t.unsqueeze(1).repeat(1, H, 1, 1).view(-1, t.size(1), t.size(2))   # noqa: E731
    head, belly, neck, back = [_wide(p) for p in d["part_points"]]
    probs = _wide(d["probs"])
    mean_shape, cams = _leaf(d["vs"][0], DEV), _leaf(d["cams"], DEV)
    ms_rep = mean_shape.unsqueeze(0).repeat(B, 1, 1).unsqueeze(1).repeat(1, H, 1, 1).view(-1, d["V"], 3)
    loss = m(rep(head).to(DEV), rep(belly).to(DEV), rep(back).to(DEV), rep(neck).to(DEV), ms_rep, cams.view(-1, 7),
             avg=False)
    total = (loss.view(B, H) * probs.to(DEV)).sum(dim=1).mean()
    total.backward()
    oms, ocams = _leaf(d["vs"][0]), _leaf(d["cams"])
    oms_rep = oms.unsqueeze(0).repeat(B, 1, 1).unsqueeze(1).repeat(1, H, 1, 1).view(-1, d["V"], 3)
    oloss = O.corr_loss_chamfer(O.OracleSoftRenderer(IS), d["part_vertices"], rep(head), rep(belly), rep(back),
                                rep(neck), oms_rep, ocams.view(-1, 7), avg=False)
    ototal = (oloss.view(B, H) * probs).sum(dim=1).mean()
    ototal.backward()
    _cmp("corr per-render", loss, oloss)
    _cmp("corr_loss", total, ototal)
    _cmp("d/dmean_shape", mean_shape.grad, oms.grad)
    _cmp("d/dcams", cams.grad, ocams.grad)


@pytest.mark.parametrize("avg", [True, False])
def test_part_matching_loss_f64(avg):
    d, eps = _scene(seed=24), eps_for_oracle()
    m = loss_utils.part_matching_loss(None, None, 0, im_size=IS, batch_size=B, tex_size=T,
                                      stex_one_hot=d["one_hot"]).to(DEV)
    _set_eps(m.renderer.renderer, eps=eps)
    vs, cams = _leaf(d["vs"], DEV), _leaf(d["cams"][:, 0], DEV)
    probs = torch.softmax(torch.arange(B, dtype=D).view(B, 1), 0)
    segs = _wide(d["part_segs"])
    with Capture() as cap:
        loss, projs = m(vs, d["fs"].to(DEV), cams, segs.to(DEV), cam_probs=None if avg else probs.to(DEV), avg=avg)
    loss.backward()
    assert len(cap.fv) == 2 and np.array_equal(cap.fv[0], cap.fv[1])   # the generic path's two packed renders
    r = OracleRenderer64(IS, "softmax", eps)
    r.ambient_light_only()
    r.overrides = [cap.fv[0]] * 4   # the oracle renders the four part maps separately, of the same projected mesh
    ovs, ocams = _leaf(d["vs"]), _leaf(d["cams"][:, 0])
    oloss, oprojs = O.part_matching_loss(r, d["one_hot"].to(D), ovs, d["fs"], ocams, segs,
                                         cam_probs=None if avg else probs, avg=avg)
    oloss.backward()
    _cmp("part_loss", loss, oloss)
    for k, (p, op) in enumerate(zip(projs, oprojs)):
        _cmp("proj%d" % (k + 1), p, op)
    _cmp("d/dverts", vs.grad, ovs.grad)
    _cmp("d/dcams", cams.grad, ocams.grad)


def test_laplacian_and_flatten_f64():
    """As the step of test_deterministic_losses_gpu composes them: 0.1 * mean Laplacian + 0.005 * mean flatten of
    mean_shape + deformation."""
    rng = np.random.default_rng(21)
    v, f = synth.icosphere(2)
    fcpu = torch.from_numpy(f.astype(np.int64))
    lap, flat = sr.LaplacianLoss(torch.from_numpy(v), fcpu).to(DEV), sr.FlattenLoss(fcpu).to(DEV)
    ms0 = torch.from_numpy(v.astype(np.float32))
    dl0 = 0.05 * torch.from_numpy(synth.bird_like(v, rng, B) - v[None])
    ms, dl = _leaf(ms0, DEV), _leaf(dl0, DEV)
    pv = ms[None] + dl
    tri, fl = lap(pv).mean(), flat(pv).mean()
    (0.1 * tri + 0.005 * fl).backward()
    oms, odl = _leaf(ms0), _leaf(dl0)
    opv = oms[None] + odl
    otri = R.laplacian_ref(opv, lap.csr_rowptr.cpu(), lap.csr_col.cpu(), lap.csr_coef.cpu())[0].mean()
    ofl = R.flatten_ref(opv, flat.edge_table.cpu()).mean()
    (0.1 * otri + 0.005 * ofl).backward()
    _cmp("laplacian", tri, otri)
    _cmp("flatten", fl, ofl)
    _cmp("d/dmean_shape", ms.grad, oms.grad)
    _cmp("d/ddelta", dl.grad, odl.grad)
