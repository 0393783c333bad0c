"""The float64 loss and mesh-op kernels (`T = double` of umr_b200/csrc/losses.cuh, the `_f64` entry points of mesh_ops.cu
and vertex.cu) against the float64 reference (oracle/loss_ref.py, oracle/vertex_ref.py) across their accepted input
range, at the shapes of the double launch geometry: IoU partials of 2048 elements per CTA and the 1024-CTA cap of the
IoU / masked-L1 backward, masked L1 and the loss head at 2048 pixels per CTA, B = 128 for the loss head's one-warp
finalize and 600 x 600 for its grid-stride backward, TexCycle at 256 (image, face) pairs per CTA, the Laplacian at 256
vertices and flatten at 128 edges per CTA; the sampler at C = 1-4, H or W = 1, coordinates on +-1, on texel centres,
outside [-1, 1], at +-1e6 and at +-1e10 (past the int32 range); chamfer around a warp of points with duplicates and
exact dyadic ties; TexCycle from each of its three sources with ids naming no face; every CorrLossChamfer edge case
of test_vertex_range_gpu.py; a NaN in one image; flow / prob views at an odd element offset.

Every input is a contiguous view into a buffer whose guard bands hold a sentinel (NaN for floats, 0 - a valid index -
for integer tables, a face no id names for the face-id plane, 1 for the visibility bytes), so a read outside an input
changes a compared output or makes it non-finite; every check rejects NaN.

Tolerances are error bounds at u = 2^-53, gamma_n = n u / (1 - n u): |kernel - reference| <= gamma_n * M with M the
magnitude evaluation, and n = the kernel's longest chain of roundings + the reference's own (the reference is float64
too).  Torch's CPU sum order is unspecified, so a sum of k terms counts k - 1.  The double unit is built with
-fmad=false: every operation rounds once.  Kernel counts: a per-thread loop of k steps k, warp_sum 5, the second
warp_sum over a CTA's warp partials 5, the slot sum n_cta.  1 - I/U and the flatten loss get the first-order bounds of
test_loss_range_gpu.py at u = 2^-53.  Each check prints its largest error / bound ratio (`pytest -s`).
"""
import functools
import math

import numpy as np
import pytest
import torch

import loss_ref as R
import vertex_ref as VR
from loss_ref import U64
from test_vertex_range_gpu import CORR_CASES, _corr_case
from umr_b200 import ops
from umr_b200 import soft_renderer as sr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D = torch.float64
PAD = 4096   # guard elements on each side (keeps an offset-0 view 32-byte aligned)


def g64(n):
    return R.gamma(n, U64)


def guarded(t, offset=0, fill=float("nan")):
    """A contiguous CUDA copy of `t` inside a buffer filled with `fill` (PAD + offset elements before, PAD after)."""
    t = t.contiguous()
    buf = torch.full((t.numel() + 2 * PAD + offset,), fill, dtype=t.dtype, device=DEV)
    v = buf[PAD + offset:PAD + offset + t.numel()].view(t.shape)
    v.copy_(t.to(DEV))
    return v


def _check(name, got, ref, bound, mask=None):
    """|got - ref| <= bound everywhere (NaN fails); prints the largest error / bound ratio."""
    got = got.detach().double().cpu()
    ref = torch.as_tensor(ref).detach().double().cpu()
    bound = torch.as_tensor(bound).detach().double().cpu().expand_as(ref)
    err = (got - ref).abs()
    ok = err <= bound
    if mask is not None:
        ok = ok | ~mask
    sel = mask if mask is not None else torch.ones_like(ok)
    ratio = float((err / bound.clamp_min(1e-300))[sel].max()) if bool(sel.any()) else 0.0
    print("%-56s max err/bound = %.3e" % (name, ratio))
    assert torch.isfinite(got).all(), "%s: non-finite output (a read outside an input?)" % name
    assert bool(ok.all()), "%s: %d values outside the bound, worst ratio %.3g" % (name, int((~ok).sum()), ratio)


# -------------------------------------------------------------------------------------------------
# sampler
# -------------------------------------------------------------------------------------------------
def _flow(g, B, N, H, W):
    """[B,N,2] float64 coordinates: the corners and edges of [-1, 1], texel centres, random ones in [-1.2, 1.2],
    +-1e6, and rows 240-255 at +-1e10 (every corner out of range, `(int)floor` saturated)."""
    flow = torch.rand(B, N, 2, generator=g, dtype=D) * 2.4 - 1.2
    flow[:, :8] = torch.tensor([[-1.0, -1.0], [1.0, 1.0], [1.0, -1.0], [-1.0, 1.0], [0.0, 0.0], [1.0, 0.0],
                                [0.0, -1.0], [-1.0, 0.0]], dtype=D)
    k = torch.randint(0, 64, (B, 200, 2), generator=g).to(D)                       # texel centres
    flow[:, 8:208, 0] = 2 * (k[..., 0] % W) / max(W - 1, 1) - 1
    flow[:, 8:208, 1] = 2 * (k[..., 1] % H) / max(H - 1, 1) - 1
    flow[:, 208:240] = torch.tensor([1e6, -1e6, 3e5, -7e5], dtype=D)[torch.randint(0, 4, (B, 32, 2), generator=g)]
    flow[:, 240:256, 0] = torch.tensor([1e10, -1e10], dtype=D)[torch.randint(0, 2, (B, 16), generator=g)]
    flow[:, 248:256, 1] = torch.tensor([1e10, -1e10], dtype=D)[torch.randint(0, 2, (B, 8), generator=g)]
    flow[:, 240:248, 1] = flow[:, 240:248, 1].clamp(-1, 1)                          # one axis in range, one saturated
    return flow


@pytest.mark.parametrize("C", [1, 2, 3, 4])
@pytest.mark.parametrize("H,W", [(1, 7), (6, 1), (17, 23)])
def test_sampler(C, H, W):
    g = torch.Generator().manual_seed(C * 100 + H)
    B, N = 2, 1000                                                                  # N not a multiple of 256
    img = torch.rand(B, C, H, W, generator=g, dtype=D) * 2 - 1
    flow = _flow(g, B, N, H, W)
    up = torch.rand(B, N, C, generator=g, dtype=D) * 2 - 1
    ig = guarded(img).requires_grad_(True)
    fg = guarded(flow).requires_grad_(True)
    out = ops.bilinear_sample(ig, fg)
    assert out.dtype == D
    (out * up.to(DEV)).sum().backward()
    imd, fld = img.clone().requires_grad_(True), flow.clone().requires_grad_(True)
    ref = R.sample_ref(imd, fld, D)
    gi, gf = torch.autograd.grad((ref * up).sum(), (imd, fld))
    m_out, m_gf, m_gi, cnt = R.sample_magnitude(img, flow, up, D)
    tag = "sampler C=%d %dx%d" % (C, H, W)
    # both sides compute the same double coordinate map, so they share ix, iy and the corners.  out: weight
    # differences 1, weight products 1, corner products 1, the four-term sum 3 = 6, the reference the same 6
    _check(tag + " out", out, ref, g64(6 + 6) * m_out)
    # grad_flow: weights 2, difference / product / sum 3, the g product 1, C channels, the exact (W-1)/2 scale 1 =
    # C + 7; the reference's autograd (g a, times a weight, the channel sum, the four corner terms, the scale) <= C + 7
    _check(tag + " grad_flow", fg.grad, gf, g64(2 * C + 14) * m_gf)
    # grad_image (the cell-key gather): weight 1, two products, one add per term = cnt + 3; the reference's weight
    # product, g product and index_add of cnt terms = cnt + 3
    _check(tag + " grad_image", ig.grad, gi, g64(2 * cnt + 6) * m_gi)
    # +-1e10 on an axis longer than one texel: every corner out of range, so exactly 0 (an axis of one texel maps
    # every coordinate to 0)
    sat = ((flow[..., 0].abs() > 1e9) & (W > 1)) | ((flow[..., 1].abs() > 1e9) & (H > 1))
    assert int(sat.sum()) >= 16
    assert bool((out.cpu()[sat] == 0).all()) and bool((fg.grad.cpu()[sat] == 0).all()), tag + ": saturated samples not 0"


# -------------------------------------------------------------------------------------------------
# IoU
# -------------------------------------------------------------------------------------------------
def _iou_bounds(p, t, gl, n_cta, per_thread, grad_roundings):
    """(loss bound [B], grad bound [B,N]) of per-image 1 - I/U from k_iou_partial<double> (or k_losshead_partial)
    against iou_ref.  I: product 1, per-thread sum, two warp trees 10, n_cta slots; U: 2 + the same + the 1e-6; the
    reference: products 1 (U: 2) + a sum of N terms, N - 1 (U: + the 1e-6)."""
    li, I, U = R.iou_ref(p, t)
    _, Im, Um = R.iou_ref(p, t, magnitude=True)
    N = p[0].numel()
    eI = g64(1 + per_thread + 10 + n_cta + 1 + N - 1) * Im
    eU = g64(2 + per_thread + 10 + n_cta + 1 + 2 + N - 1 + 1) * Um
    # 1 - I/U: |d| <= eI / U + (I / U) eU / U to first order, and each side rounds the division and subtraction once
    lb = (eI + I / U * eU) / U + g64(4) * (I / U + li.abs())
    # grad = -g (t U - I (1 - t)) / U^2: first order in eI, eU, plus both sides' own roundings (`grad_roundings`)
    t2, a = t.reshape(t.shape[0], -1), gl.abs()[:, None]
    mag = t2.abs() * U[:, None] + I[:, None] * (1 - t2).abs()
    gb = a * ((1 - t2).abs() / U[:, None] ** 2 * eI[:, None] + (3 * mag) / U[:, None] ** 3 * eU[:, None]) \
        + g64(grad_roundings) * a * mag / U[:, None] ** 2
    return lb, gb


IOU_CASES = [(3, 2047, "dense"), (3, 2048, "dense"), (3, 2049, "dense"), (3, 3 * 2048 + 5, "dense"),
             (2, 2 ** 20 + 2049, "dense"), (3, 2 * 2048 + 4, "odd stride"), (3, 3 * 2048 + 5, "alpha"),
             (128, 2049, "dense")]


@pytest.mark.parametrize("B,N,layout", IOU_CASES)
def test_iou(B, N, layout):
    g = torch.Generator().manual_seed(N + B)
    p = torch.rand(B, N, generator=g, dtype=D)
    t = (torch.rand(B, N, generator=g) > 0.5).to(D)
    p[1], t[1] = 0, 0                                                               # an all-zero image
    gl = torch.rand(B, generator=g, dtype=D) + 0.5
    if layout == "odd stride":                                                      # batch stride N + 1, odd
        pg = guarded(torch.cat([p, torch.zeros(B, 1, dtype=D)], 1))[:, :N]
    elif layout == "alpha":                                                         # the alpha plane of an RGBA render
        pg = guarded(torch.cat([torch.rand(B, 3, N, generator=g, dtype=D), p[:, None]], 1))[:, 3]
    else:
        pg = guarded(p)
    pg.requires_grad_(True)
    loss = ops.neg_iou_per_image(pg, guarded(t))
    assert loss.dtype == D
    (loss * gl.to(DEV)).sum().backward()
    pd = p.clone().requires_grad_(True)
    li, _, _ = R.iou_ref(pd, t)
    gp, = torch.autograd.grad((li * gl).sum(), pd)
    # grad: k_iou_bwd 6 (U U, the division, 1 - t, the product with I, the subtraction, the product with k); the
    # reference's autograd through I / U and the two sums' backward (2 + 4 + 2) = 8
    lb, gb = _iou_bounds(p, t, gl, math.ceil(N / 2048), 8, 6 + 8)
    tag = "iou B=%d N=%d %s" % (B, N, layout)
    _check(tag + " loss", loss, li, lb)
    _check(tag + " grad", pg.grad, gp, gb)


# -------------------------------------------------------------------------------------------------
# masked L1
# -------------------------------------------------------------------------------------------------
def _l1_kinks(pred, gt, mgt, mpred):
    """[B,C,HW] elements whose sign the kernel may see differently (|d| within both sides' rounding of 0).  An exact
    d == 0 (a product compared with itself) is no kink: both sides round the same two products and subtract, so both
    see 0 and take the zero subgradient."""
    B, C = pred.shape[:2]
    a, b = pred.reshape(B, C, -1) * mpred.reshape(B, 1, -1), gt.reshape(B, C, -1) * mgt.reshape(B, 1, -1)
    d = a - b
    return (d != 0) & (d.abs() <= g64(4) * (a.abs() + b.abs()))


def _l1_grad_bound(rgba, gt, mgt, gl, C):
    """(bound, unmasked) of masked L1's gradient [B,4,HW] with respect to its RGBA render."""
    B, HW = rgba.shape[0], rgba.shape[2]
    kink = _l1_kinks(rgba[:, :C], gt, mgt, rgba[:, 3])
    k = (gl / (C * HW))[:, None, None]
    ok = torch.ones(B, 4, HW, dtype=torch.bool)
    ok[:, :C] = ~kink
    ok[:, 3] = ~kink.any(1)
    gbound = torch.zeros(B, 4, HW, dtype=D)
    # grad_pred: k (inv_n, gl inv_n) 2, the product with the mask 1; the reference's division and product 2
    gbound[:, :C] = g64(3 + 2) * k * rgba[:, 3:4]
    # grad_mask_pred: k 2, products 1, C - 1 adds; the reference's division, products, the channel sum C - 1
    gbound[:, 3] = g64((C + 2) + (C + 1)) * (k * rgba[:, :C]).sum(1)
    return gbound, ok


def _l1_loss_bound(C, HW):
    """n of masked L1's per-image value.  Kernel: |p a - g m| 2, 8 C per thread, warp trees 10, n_cta slots, inv_n and
    its product 2; the reference: products and difference 2, a sum of C HW terms, the division 1."""
    return (2 + 8 * C + 10 + math.ceil(HW / 2048) + 2) + (2 + C * HW)


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("HW", [2047, 2049, 3 * 2048 + 7, 2 ** 20 + 2049])
def test_masked_l1(C, HW):
    g = torch.Generator().manual_seed(C * HW)
    B = 3
    rgba = torch.rand(B, 4, HW, generator=g, dtype=D)
    gt = torch.rand(B, C, HW, generator=g, dtype=D)
    mgt = (torch.rand(B, HW, generator=g) > 0.4).to(D)
    gt[:, :, :64] = rgba[:, :C, :64] * rgba[:, 3:, :64]                            # kinks: d == 0 exactly
    mgt[:, :64] = 1
    gl = torch.rand(B, generator=g, dtype=D) + 0.5
    buf = guarded(rgba).requires_grad_(True)                                       # strided views of one RGBA render
    pred, mpred = buf[:, :C].reshape(B, C, HW, 1), buf[:, 3].reshape(B, HW, 1)
    loss = ops.masked_l1_per_image(pred, guarded(gt).reshape(B, C, HW, 1), guarded(mgt).reshape(B, HW, 1), mpred)
    (loss * gl.to(DEV)).sum().backward()
    rd = rgba.clone().requires_grad_(True)
    args = (rd[:, :C].reshape(B, C, HW, 1), gt.reshape(B, C, HW, 1), mgt, rd[:, 3])
    ref = R.masked_l1_ref(*args)
    gr, = torch.autograd.grad((ref * gl).sum(), rd)
    mag = R.masked_l1_ref(*[a.detach() for a in args], magnitude=True)
    tag = "masked l1 C=%d HW=%d" % (C, HW)
    _check(tag + " loss", loss, ref, g64(_l1_loss_bound(C, HW)) * mag)
    gbound, ok = _l1_grad_bound(rgba, gt, mgt, gl, C)
    _check(tag + " grad", buf.grad, gr, gbound, ok)


# -------------------------------------------------------------------------------------------------
# fused loss head
# -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W", [(1, 1, 2049), (33, 1, 2049), (128, 1, 2049), (2, 600, 600)])
def test_loss_head(B, H, W):
    g = torch.Generator().manual_seed(B * H * W)
    HW = H * W
    rgba = torch.rand(B, 4, H, W, generator=g, dtype=D)
    gt = torch.rand(B, 3, H, W, generator=g, dtype=D)
    mgt = (torch.rand(B, H, W, generator=g) > 0.4).to(D)
    w_iou, w_tex = 2.5, 3.0
    x = guarded(rgba).requires_grad_(True)
    loss, per = ops.mask_texture_loss(x, guarded(gt), guarded(mgt), w_iou, w_tex)
    loss.backward()
    rd = rgba.clone().requires_grad_(True)
    ref, per_ref = R.loss_head_ref(rd, gt, mgt, w_iou, w_tex)
    gr, = torch.autograd.grad(ref, rd)
    n_cta = math.ceil(HW / 2048)
    tag = "loss head B=%d %dx%d" % (B, H, W)
    gl_iou = torch.full((B,), w_iou / B, dtype=D)
    # alpha's IoU term: k_losshead_bwd's ki 3, the bracket 3, their product 1, the three L1 terms added 3 = 10; the
    # reference: the weight and the mean 2, the IoU autograd 8, the add of the L1 path 1 = 11
    lb_iou, gb_iou = _iou_bounds(rgba[:, 3], mgt, gl_iou, n_cta, 8, 10 + 11)
    args = (rgba[:, :3], gt, mgt, rgba[:, 3])
    # per-image L1: |.| 2, 24 per thread, warp trees 10, n_cta slots, inv_n and its product 2; the reference 3 + 3 HW - 1
    lb_tex = g64(2 + 24 + 10 + n_cta + 2 + 3 + 3 * HW - 1) * R.masked_l1_ref(*args, magnitude=True)
    _check(tag + " per-image 1 - IoU", per[:, 0], per_ref[:, 0], lb_iou)
    _check(tag + " per-image L1", per[:, 1], per_ref[:, 1], lb_tex)
    # finalize: one warp, ceil(B / 32) sequential adds per lane, the warp tree 5, / B, the weights and their sum 3;
    # the reference's means (B - 1 adds, the division), the weights and their sum 3
    Df = (math.ceil(B / 32) + 5 + 3) + (B + 3)
    lb = (w_iou * lb_iou.sum() + w_tex * lb_tex.sum()) / B \
        + g64(Df) * (w_iou * per_ref[:, 0].abs().mean() + w_tex * per_ref[:, 1].abs().mean())
    _check(tag + " loss", loss.reshape(1), ref.detach().reshape(1), lb.detach().reshape(1))
    kink = _l1_kinks(*args)
    kt = w_tex / (B * 3 * HW)
    ok = torch.ones(B, 4, HW, dtype=torch.bool)
    ok[:, :3] = ~kink.reshape(B, 3, HW)
    ok[:, 3] = ~kink.reshape(B, 3, HW).any(1)
    gb = torch.zeros(B, 4, HW, dtype=D)
    # rgb: kt 4, the product with alpha 1; the reference's weight, mean, 1 / (3 HW) and product 4
    gb[:, :3] = g64(5 + 4) * kt * rgba[:, 3:4].reshape(B, 1, HW)
    # alpha's L1 terms: kt 4, products 1, 3 adds; the reference's 3, products 1, channel sum 2, the add of the IoU path 1
    gb[:, 3] = gb_iou + g64(8 + 7) * kt * rgba[:, :3].reshape(B, 3, HW).sum(1)
    _check(tag + " grad", x.grad.reshape(B, 4, HW), gr.reshape(B, 4, HW), gb, ok)


# -------------------------------------------------------------------------------------------------
# chamfer
# -------------------------------------------------------------------------------------------------
CHAMFER_CASES = [(2, 1, 33, 2, "random"), (2, 31, 32, 3, "random"), (3, 32, 1, 2, "random"), (2, 33, 31, 3, "random"),
                 (2, 33, 70, 3, "dyadic"), (2, 64, 33, 2, "dyadic"), (1, 20000, 642, 3, "random")]


@pytest.mark.parametrize("B,N,M,Dm,kind", CHAMFER_CASES)
def test_chamfer(B, N, M, Dm, kind):
    g = torch.Generator().manual_seed(N * M + Dm)
    if kind == "dyadic":   # every product and sum exact in double: distances tie exactly, the lowest index must win
        a = torch.randint(-4, 5, (B, N, Dm), generator=g).to(D) / 8
        b = torch.randint(-4, 5, (B, M, Dm), generator=g).to(D) / 8
    else:
        a = torch.rand(B, N, Dm, generator=g, dtype=D) - 0.5
        b = torch.rand(B, M, Dm, generator=g, dtype=D) - 0.5
    a[:, 9 % N] = a[:, 4 % N]                                                       # duplicate points
    b[:, 5 % M] = b[:, 2 % M]
    w1, w2 = torch.rand(B, N, generator=g, dtype=D), torch.rand(B, M, generator=g, dtype=D)
    ag, bg = guarded(a).requires_grad_(True), guarded(b).requires_grad_(True)
    d_ab, d_ba, i_ab, i_ba = ops.dist_chamfer(ag, bg)
    ((d_ab * w1.to(DEV)).sum() + (d_ba * w2.to(DEV)).sum()).backward()
    _, _, r_ab, r_ba = R.chamfer_ref(a, b)
    i_ab, i_ba = i_ab.cpu().long(), i_ba.cpu().long()
    tag = "chamfer B=%d N=%d M=%d D=%d %s" % (B, N, M, Dm, kind)
    if kind == "dyadic":
        assert torch.equal(i_ab, r_ab) and torch.equal(i_ba, r_ba), tag + ": an exact tie did not take the lowest index"
    # distances: products 1, D - 1 adds, the two final roundings 2 = D + 2 on each side
    nd = 2 * (Dm + 2)
    assert R.near_tie(a, b, i_ab, r_ab, 2, nd, U64).all() and R.near_tie(b, a, i_ba, r_ba, 2, nd, U64).all()
    ar, br = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    e_ab, e_ba, _, _ = R.chamfer_ref(ar, br, i_ab, i_ba)
    ga, gb = torch.autograd.grad((e_ab * w1).sum() + (e_ba * w2).sum(), (ar, br))
    am, bm = a.abs().requires_grad_(True), b.abs().requires_grad_(True)
    m_ab, m_ba, _, _ = R.chamfer_ref(am, bm, i_ab, i_ba, magnitude=True)
    gam, gbm = torch.autograd.grad((m_ab * w1).sum() + (m_ba * w2).sum(), (am, bm))
    _check(tag + " d_ab", d_ab, e_ab, g64(nd) * m_ab)
    _check(tag + " d_ba", d_ba, e_ba, g64(nd) * m_ba)
    # a point's gradient: its own term + one per point that picked it.  The gather: 2 roundings a term, one add per
    # term, the warp tree 5, own + gathered 1; the reference: 3 a term, the sum of the terms, 2 to join the |q|^2,
    # |k|^2 and q.k paths
    cnt = 1 + max(int(torch.bincount(i_ba.reshape(-1) + N * torch.arange(B).repeat_interleave(M)).max()),
                  int(torch.bincount(i_ab.reshape(-1) + M * torch.arange(B).repeat_interleave(N)).max()))
    ng = (2 + cnt + 5 + 1) + (3 + cnt + 2)
    _check(tag + " grad a", ag.grad, ga, g64(ng) * gam)
    _check(tag + " grad b", bg.grad, gb, g64(ng) * gbm)


# -------------------------------------------------------------------------------------------------
# texture cycle
# -------------------------------------------------------------------------------------------------
SENTINEL_FACE = 1   # the guard value of the face-id plane: a face no id in the plane names


@pytest.mark.parametrize("source", ["plane64", "plane32", "visible"])
@pytest.mark.parametrize("T2", [1, 36, 64])
def test_texcycle(T2, source):
    g = torch.Generator().manual_seed(T2)
    B, F, P = 3, 301, 1023                                                          # B*F = 903: 4 CTAs; P % 4 != 0
    flow = torch.rand(B, F, T2, 2, generator=g, dtype=D) * 2 - 1
    prob = torch.rand(B, F, 2, generator=g, dtype=D) * 2 - 1
    ids = torch.randint(-F - 3, F + 3, (B, P), generator=g).to(D)                  # ids >= F, < -1 and < -F
    ids[1, :5] = torch.tensor([-1.0, -2.0, float(F), -float(F) - 2, 7.0], dtype=D)
    ids[(ids == SENTINEL_FACE) | (ids == SENTINEL_FACE - F)] = F + 1                # names no face
    vis = R.visible_ref(ids, F)
    assert not bool(vis[:, SENTINEL_FACE].any())
    gl = 0.75
    fg = guarded(flow).requires_grad_(True)
    pg = guarded(prob)
    if source == "visible":
        loss = ops.tex_cycle(fg, pg, None, guarded(vis.to(torch.uint8), fill=1))
    else:
        plane = ids if source == "plane64" else ids.float()
        loss = ops.tex_cycle(fg, pg, guarded(plane, fill=float(SENTINEL_FACE)))
    assert loss.dtype == D
    (loss * gl).backward()
    fd = flow.clone().requires_grad_(True)
    ref = R.texcycle_ref(fd, prob, vis)
    gf, = torch.autograd.grad(ref * gl, fd)
    mag = R.texcycle_ref(flow, prob, vis, magnitude=True)
    n_cta = math.ceil(B * F / 256)
    tag = "texcycle T2=%d %s" % (T2, source)
    # kernel: the T2-term sum T2 - 1, / T2, - p, square, + 4, warp trees 10, scale and its product 2, n_cta slots;
    # the reference: the mean T2, - p 1, square 1, the sum of 2 B F terms, the division 1
    _check(tag + " loss", loss, ref, g64((T2 + 3 + 10 + 2 + n_cta) + (T2 + 3 + 2 * B * F)) * mag)
    k = 2 * gl / (B * F * 2) / T2
    gm = k * (flow.abs().mean(2) + prob.abs()) * vis[:, :, None]
    # grad: k 3, the mean and difference T2 + 1, the product 1; the reference's difference T2 + 1 and 4 for the
    # backward of the square, the mean and the MSE scale
    _check(tag + " grad", fg.grad, gf, g64((T2 + 5) + (T2 + 5)) * gm[:, :, None, :].expand(-1, -1, T2, -1))


# -------------------------------------------------------------------------------------------------
# Laplacian and flatten
# -------------------------------------------------------------------------------------------------
def _deformed(v, f, B, seed):
    """[B,V,3] float64 shapes of one mesh: random radial noise, plus per item a planar cap (exactly flat dihedrals),
    a vertex pushed through the surface (folded dihedrals) and a vertex 1e-4 from a neighbour (edges < sqrt(eps))."""
    rng = np.random.default_rng(seed)
    x = v[None].astype(np.float64) * rng.uniform(0.7, 1.3, (B, len(v), 1))
    for b in range(B):
        kind = b % 4
        if kind == 1:
            x[b, :, 2] = np.minimum(x[b, :, 2], 0.6)
        elif kind == 2:
            x[b, rng.integers(len(v))] *= -0.3
        elif kind == 3:
            t = f[rng.integers(len(f))]
            x[b, t[0]] = x[b, t[1]] + rng.uniform(-1e-4, 1e-4, 3)
    return torch.from_numpy(x)


@functools.lru_cache(maxsize=None)
def _mesh_reference(mesh, B):
    """The float64 results and bounds of one (mesh, B) case (the flatten bound takes seconds)."""
    v, f = R.spiked_uv_sphere(*mesh)
    x = _deformed(v, f, B, sum(mesh))
    gl = torch.rand(B, generator=torch.Generator().manual_seed(B), dtype=D) + 0.5
    lap = sr.LaplacianLoss(torch.from_numpy(v), torch.from_numpy(f))
    flat = sr.FlattenLoss(torch.from_numpy(f))
    E, V = flat.edge_table.shape[0], len(v)
    deg = int(torch.diff(lap.csr_rowptr).max())
    xd = x.clone().requires_grad_(True)
    lref, _ = R.laplacian_ref(xd, lap.csr_rowptr, lap.csr_col, lap.csr_coef)
    lgrad, = torch.autograd.grad((lref * gl).sum(), xd)
    xm = x.abs().requires_grad_(True)
    lmag, _ = R.laplacian_ref(xm, lap.csr_rowptr, lap.csr_col, lap.csr_coef, magnitude=True)
    lgm, = torch.autograd.grad((lmag * gl).sum(), xm)
    # loss: y deg + 1, |y|^2 3, per thread 1, warp trees 10, ceil(V / 256) slots; the reference's y deg + 1, the square
    # 1, the sum of 3 V terms.  Gradient 2 g (y_j + sum tcoef y_i) with y's error: 2 deg + 5 on each side
    lap_bounds = (g64((deg + 4 + 1 + 10 + math.ceil(V / 256)) + (deg + 2 + 3 * V - 1)) * lmag,
                  g64(2 * (2 * deg + 5)) * lgm)
    # flatten: the first-order bound of loss_ref.flatten_error_bound at u = 2^-53 (its doubling covers the reference's
    # per-edge rounding).  The loss sum: per-thread 1, warp trees 10, CTAs, the reference's sum of E terms; the gradient:
    # the reference's index_add of a vertex's terms adds `count` more roundings to the gather's own
    eps = 1e-6
    xd = x.clone().requires_grad_(True)
    fref = R.flatten_ref(xd, flat.edge_table, eps)
    fgrad, = torch.autograd.grad((fref * gl).sum(), xd)
    lb, gb = R.flatten_error_bound(x, flat.edge_table, eps, gl, 1 + 10 + math.ceil(E / 128) + E - 1, U64)
    idx = flat.edge_table.long()
    P = x[:, idx].clone().requires_grad_(True)
    G, = torch.autograd.grad((R.flatten_ref(P.reshape(B, -1, 3), torch.arange(E * 4).view(E, 4), eps) * gl).sum(), P)
    count = int(torch.bincount(idx.reshape(-1), minlength=V).max())
    ga = torch.zeros(B, V, 3, dtype=D).index_add_(1, idx.reshape(-1), G.abs().reshape(B, E * 4, 3))
    flat_bounds = (lb, gb + g64(count) * ga)
    return v, f, x, gl, (lref.detach(), lgrad) + lap_bounds, (fref.detach(), fgrad) + flat_bounds


@pytest.mark.parametrize("mesh,B", [((21, 12, 15), 4), ((11, 12, 9), 64)])   # V = 257, E = 765; V = 131, E = 387
def test_laplacian_flatten(mesh, B):
    v, f, x, gl, lap_ref, flat_ref = _mesh_reference(mesh, B)
    lap = sr.LaplacianLoss(torch.from_numpy(v), torch.from_numpy(f)).to(DEV)
    flat = sr.FlattenLoss(torch.from_numpy(f)).to(DEV)
    tag = "V=%d E=%d B=%d" % (len(v), flat.edge_table.shape[0], B)
    xg = guarded(x).requires_grad_(True)
    tables = [guarded(t, fill=0) for t in (lap.csr_rowptr, lap.csr_col)]
    coefs = [guarded(t.double()) for t in (lap.csr_coef, lap.csr_tcoef)]
    loss = ops.LaplacianFunction.apply(xg, *tables, *coefs)
    (loss * gl.to(DEV)).sum().backward()
    ref, gref, lb, gb = lap_ref
    _check("laplacian " + tag + " loss", loss, ref, lb)
    _check("laplacian " + tag + " grad", xg.grad, gref, gb)
    xg = guarded(x).requires_grad_(True)
    loss = ops.FlattenFunction.apply(xg, guarded(flat.edge_table, fill=0), 1e-6, guarded(flat.vert_rowptr, fill=0),
                                     guarded(flat.vert_incidence, fill=0))
    (loss * gl.to(DEV)).sum().backward()
    ref, gref, lb, gb = flat_ref
    _check("flatten " + tag + " loss", loss, ref, lb)
    _check("flatten " + tag + " grad", xg.grad, gref, gb)


# -------------------------------------------------------------------------------------------------
# part chamfer (CorrLossChamfer)
# -------------------------------------------------------------------------------------------------
def _corr_f64(tag, parts, targets, weights, verts, cams, loss, vert2d, nn, gl, gv2, got_gv, got_gc, summed_renders=0):
    """test_vertex_range_gpu's comparison at u = 2^-53: each count is the float32 kernel's (the same templated body,
    -fmad=false in both precisions) once for the kernel and once for the reference, whose sums over the NS selected
    vertices add NS - 1."""
    B, NS = cams.shape[0], vert2d.shape[1]
    vd, cd = verts.clone().requires_grad_(True), cams.clone().requires_grad_(True)
    _, q64, idx64 = VR.corr_chamfer_ref(vd, cd, parts, targets, weights)
    nn = nn.long().cpu()
    with torch.no_grad():   # an index that differs from the float64 argmin must be a near-tie
        qm = VR.project_vertices(verts.abs()[:, torch.cat(parts)].expand(B, -1, -1), cams.abs())[..., :2]
        start = 0
        for p, t in zip(parts, targets):
            sl = slice(start, start + len(p))
            d = ((q64[:, sl, None, :] - t[:, None, :, :]) ** 2).sum(-1)
            dm = ((qm[:, sl, None, :] + t.abs()[:, None, :, :]) ** 2).sum(-1)
            pick = lambda x, i: torch.gather(x, 2, i[:, sl, None])[..., 0]   # noqa: E731
            tol = g64(2 * 15) * (pick(dm, nn) + pick(dm, idx64))
            assert bool(((pick(d, nn) - pick(d, idx64)).abs() <= tol).all()), tag + ": nearest differs beyond a near-tie"
            start += len(p)
    loss64, q64, _ = VR.corr_chamfer_ref(vd, cd, parts, targets, weights, nearest=nn)
    gv, gc = torch.autograd.grad((loss64 * gl).sum() + (q64 * gv2).sum(), (vd, cd))
    va, ca = verts.abs().requires_grad_(True), cams.abs().requires_grad_(True)
    lm, qm, _ = VR.corr_chamfer_ref(va, ca, parts, [t.abs() for t in targets], weights, nearest=nn, magnitude=True)
    mv, mc = torch.autograd.grad((lm * gl.abs()).sum() + (qm * gv2.abs()).sum(), (va, ca))
    _check(tag + " vert2d", vert2d, q64, g64(2 * 10) * qm)
    _check(tag + " loss", loss, loss64, g64(2 * (24 + math.ceil(NS / 8)) + NS) * lm)
    mult = int(torch.bincount(torch.cat(parts)).max()) if NS else 0
    if got_gv is not None:
        _check(tag + " grad vertices", got_gv, gv, g64(2 * (26 + mult + summed_renders)) * mv)
    if got_gc is not None:
        _check(tag + " grad cams", got_gc, gc, g64(2 * (39 + math.ceil(NS / 256)) + NS) * mc)


@pytest.mark.parametrize("B,sizes,counts,weights,mode", [c[:5] for c in CORR_CASES])
def test_corr_chamfer(B, sizes, counts, weights, mode):
    parts, targets, verts, cams = _corr_case(B, sizes, counts, mode, seed=B + sum(sizes) + sum(counts))
    targets, verts, cams = [t.double() for t in targets], verts.double(), cams.double()
    NS = sum(sizes)
    g = torch.Generator().manual_seed(NS)
    gl, gv2 = torch.randn(B, generator=g, dtype=D), torch.randn(B, NS, 2, generator=g, dtype=D)
    base = guarded(verts).requires_grad_(True)
    v = base.expand(B, -1, -1) if mode == "expanded" else base
    c = guarded(cams).requires_grad_(True)
    sel = torch.cat(parts).int()
    table = [guarded(t, fill=0) for t in ops._incidence_on(sel, verts.shape[1], "cpu")]
    loss, vert2d = ops.corr_chamfer(v, c, guarded(sel, fill=0), [guarded(t) for t in targets], np.cumsum(sizes).tolist(),
                                    weights, table)
    assert loss.dtype == D
    nn = loss.grad_fn.saved_tensors[4]
    torch.autograd.backward([loss, vert2d], [gl.to(DEV), gv2.to(DEV)])
    tag = "corr B%d NS%d m%s w%s %s" % (B, NS, counts, weights, mode)
    _corr_f64(tag, parts, targets, weights, verts, cams, loss, vert2d, nn, gl, gv2, base.grad, c.grad,
              summed_renders=B if mode != "per_render" else 0)


def test_corr_exact_ties_take_the_lowest_index():
    """test_vertex_range_gpu's exact-tie case in float64: identity camera, dyadic coordinates, so targets 1 and 2 and
    targets 5 and 37 are exactly as near as each other; the kernel must take the lowest index, as torch.min does."""
    B = 2
    verts = torch.tensor([[[0.25, 0.5, 0.125], [-0.5, 0.25, 0.0], [0.125, -0.25, 0.5], [0.0, 0.0, 0.0]]], dtype=D)
    cams = torch.tensor([[1.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]], dtype=D).repeat(B, 1)
    t0 = torch.full((B, 40, 2), 4.0, dtype=D)
    t0[:, 1] = torch.tensor([0.25 + 0.125, 0.5])
    t0[:, 2] = torch.tensor([0.25, 0.5 - 0.125])
    t0[:, 0] = torch.tensor([0.25, 0.5 + 0.25])
    t0[:, 5] = torch.tensor([-0.5 - 0.25, 0.25])
    t0[:, 37] = torch.tensor([-0.5, 0.25 + 0.25])
    targets = [t0] + [torch.rand(B, 3, 2, generator=torch.Generator().manual_seed(k), dtype=D) for k in range(3)]
    parts = [torch.tensor([0, 1]), torch.tensor([2]), torch.tensor([3]), torch.tensor([0])]
    verts = verts.expand(B, -1, -1).contiguous()
    v = guarded(verts).requires_grad_(True)
    c = guarded(cams).requires_grad_(True)
    loss, vert2d = ops.corr_chamfer(v, c, guarded(torch.cat(parts).int(), fill=0), [guarded(t) for t in targets],
                                    [2, 3, 4, 5], (1, 1, 1, 1))
    nn = loss.grad_fn.saved_tensors[4].cpu()
    loss.sum().backward()
    assert nn[:, 0].tolist() == [1] * B and nn[:, 1].tolist() == [5] * B, nn
    _, _, idx64 = VR.corr_chamfer_ref(verts, cams, parts, targets, (1, 1, 1, 1))
    assert torch.equal(nn.long(), idx64)
    _corr_f64("corr exact ties", parts, targets, (1, 1, 1, 1), verts, cams, loss, vert2d, nn, torch.ones(B, dtype=D),
              torch.zeros(B, 5, 2, dtype=D), v.grad, c.grad)


# -------------------------------------------------------------------------------------------------
# a NaN in one image stays in that image
# -------------------------------------------------------------------------------------------------
def test_nan_stays_in_its_image():
    g = torch.Generator().manual_seed(77)
    B, HW = 3, 3 * 2048 + 5
    rgba = torch.rand(B, 4, HW, generator=g, dtype=D)
    gt = torch.rand(B, 3, HW, generator=g, dtype=D)
    mgt = (torch.rand(B, HW, generator=g) > 0.4).to(D)
    bad = rgba.clone()
    bad[1, 3, 2049] = float("nan")                                                  # alpha: the IoU and L1 of image 1
    bad[1, 0, 5000] = float("nan")                                                  # rgb: the L1 of image 1
    keep = torch.tensor([True, False, True])
    n_cta = math.ceil(HW / 2048)
    gl = torch.rand(B, generator=g, dtype=D) + 0.5

    x = guarded(bad).requires_grad_(True)
    li = ops.neg_iou_per_image(x[:, 3], guarded(mgt))
    (li * gl.to(DEV)).sum().backward()
    assert bool(torch.isnan(li[1]))
    pd = rgba[:, 3].clone().requires_grad_(True)
    ref, _, _ = R.iou_ref(pd, mgt)
    gp, = torch.autograd.grad((ref * gl).sum(), pd)
    lb, gb = _iou_bounds(rgba[:, 3], mgt, gl, n_cta, 8, 6 + 8)
    _check("nan isolation iou loss", li[keep], ref[keep], lb[keep])
    _check("nan isolation iou grad", x.grad[keep, 3], gp[keep], gb[keep])

    x = guarded(bad).requires_grad_(True)
    l1 = ops.masked_l1_per_image(x[:, :3].reshape(B, 3, HW, 1), guarded(gt).reshape(B, 3, HW, 1),
                                 guarded(mgt).reshape(B, HW, 1), x[:, 3].reshape(B, HW, 1))
    (l1 * gl.to(DEV)).sum().backward()
    assert bool(torch.isnan(l1[1]))
    rd = rgba.clone().requires_grad_(True)
    args = (rd[:, :3].reshape(B, 3, HW, 1), gt.reshape(B, 3, HW, 1), mgt, rd[:, 3])
    ref = R.masked_l1_ref(*args)
    gr, = torch.autograd.grad((ref * gl).sum(), rd)
    mag = R.masked_l1_ref(*[a.detach() for a in args], magnitude=True)
    _check("nan isolation masked l1 loss", l1[keep], ref[keep], g64(_l1_loss_bound(3, HW)) * mag[keep])
    gbound, ok = _l1_grad_bound(rgba, gt, mgt, gl, 3)
    _check("nan isolation masked l1 grad", x.grad[keep], gr[keep], gbound[keep], ok[keep])
    args = (rgba[:, :3].reshape(B, 3, HW, 1), gt.reshape(B, 3, HW, 1), mgt, rgba[:, 3])

    x = guarded(bad.reshape(B, 4, 1, HW)).requires_grad_(True)
    loss, per = ops.mask_texture_loss(x, guarded(gt.reshape(B, 3, 1, HW)), guarded(mgt.reshape(B, 1, HW)), 2.5, 3.0)
    loss.backward()
    assert bool(torch.isnan(per[1]).all()) and bool(torch.isnan(loss))
    rd = rgba.reshape(B, 4, 1, HW).clone().requires_grad_(True)
    ref, per_ref = R.loss_head_ref(rd, gt.reshape(B, 3, 1, HW), mgt.reshape(B, 1, HW), 2.5, 3.0)
    gr, = torch.autograd.grad(ref, rd)
    lb_iou, gb_iou = _iou_bounds(rgba[:, 3], mgt, torch.full((B,), 2.5 / B, dtype=D), n_cta, 8, 10 + 11)
    lb_tex = g64(2 + 24 + 10 + n_cta + 2 + 3 + 3 * HW - 1) * R.masked_l1_ref(*args, magnitude=True)
    _check("nan isolation loss head 1 - IoU", per[keep, 0], per_ref[keep, 0], lb_iou[keep])
    _check("nan isolation loss head L1", per[keep, 1], per_ref[keep, 1], lb_tex[keep])
    kink = _l1_kinks(*args).reshape(B, 3, HW)
    kt = 3.0 / (B * 3 * HW)
    ok = torch.ones(B, 4, HW, dtype=torch.bool)
    ok[:, :3], ok[:, 3] = ~kink, ~kink.any(1)
    gbd = torch.zeros(B, 4, HW, dtype=D)
    gbd[:, :3] = g64(9) * kt * rgba[:, 3:4]
    gbd[:, 3] = gb_iou + g64(15) * kt * rgba[:, :3].sum(1)
    _check("nan isolation loss head grad", x.grad.reshape(B, 4, HW)[keep], gr.reshape(B, 4, HW)[keep], gbd[keep],
           ok[keep])


# -------------------------------------------------------------------------------------------------
# flow / prob views at an odd element offset: realigned by ops, bitwise the aligned result
# -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["default", "deterministic", "f64"])
def test_misaligned_views_match_the_aligned_call(mode):
    dt = D if mode == "f64" else torch.float32
    g = torch.Generator().manual_seed(5)
    img = (torch.rand(2, 3, 17, 23, generator=g, dtype=D) * 2 - 1).to(dt)
    flow = (torch.rand(2, 1000, 2, generator=g, dtype=D) * 2.4 - 1.2).to(dt)
    tflow = (torch.rand(3, 301, 36, 2, generator=g, dtype=D) * 2 - 1).to(dt)
    prob = (torch.rand(3, 301, 2, generator=g, dtype=D) * 2 - 1).to(dt)
    ids = torch.randint(-1, 301, (3, 1023), generator=g).float()
    up = torch.rand(2, 1000, 3, generator=g, dtype=D).to(dt).to(DEV)

    def run(offset):
        ig = guarded(img).requires_grad_(True)
        fg = guarded(flow, offset).requires_grad_(True)
        tg = guarded(tflow, offset).requires_grad_(True)
        pg = guarded(prob, offset)
        assert offset == 0 or (fg.data_ptr() % (2 * fg.element_size()) and pg.data_ptr() % (2 * pg.element_size()))
        out = ops.bilinear_sample(ig, fg)
        (out * up).sum().backward()
        tl = ops.tex_cycle(tg, pg, guarded(ids, fill=float(SENTINEL_FACE)))
        tl.backward()
        torch.cuda.synchronize()
        return [t.detach().cpu() for t in (out, ig.grad, fg.grad, tl, tg.grad)]

    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(mode == "deterministic")
    try:
        aligned, odd = run(0), run(1)
    finally:
        torch.use_deterministic_algorithms(prev)
    for k, (a, b) in enumerate(zip(aligned, odd)):
        assert a.dtype == b.dtype == dt and torch.isfinite(a).all()
        if mode == "default" and k in (1, 3):   # float atomics sum the image gradient and the TexCycle loss
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), "%s: output %d of the odd-offset call differs" % (mode, k)
        else:
            assert torch.equal(a, b), "%s: output %d of the odd-offset call differs" % (mode, k)
    print("misaligned views %s: bitwise equal to the aligned call" % mode)
