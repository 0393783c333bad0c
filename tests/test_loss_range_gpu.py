"""The loss and mesh-op kernels (umr_b200/csrc/losses.cu, mesh_ops.cu) against the float64 reference (oracle/loss_ref.py)
across their accepted input range: the sampler at C = 1-4, H or W = 1, coordinates on +-1, on texel centres and up to
+-1e6; IoU, masked L1 and the loss head with partial last CTAs, the scalar IoU path over several CTAs, up to 128 images
and the loss head backward's grid-stride loop; chamfer around a warp of points, with duplicates and at 20000 x 642;
TexCycle over several CTAs with odd plane sizes and ids outside [-1, F); the Laplacian and flatten losses on a closed
non-icosphere mesh with valence 3-13, near-flat and folded dihedrals and edges shorter than sqrt(eps); the distance
transform on tall, thin, 4096-wide and non-binary masks; `load_textures` at the edges of its uv range.

Every case runs with torch.use_deterministic_algorithms off and on (the deterministic reductions and gathers), against
the same reference.  Every float input is a contiguous view into a buffer with NaN before and after it, so a read
outside an input shows up as NaN in the compared outputs; every check rejects NaN.

Tolerances are error bounds.  u = 2^-24, gamma_n = n u / (1 - n u).  For the polynomial parts |kernel - exact| <=
gamma_D * M with M the magnitude evaluation (`loss_ref`, `magnitude=True`) and D counted from the kernel: the
per-thread sequential terms, + 5 for the warp tree, + 5 for the second warp_sum over the CTA's warp partials, + the
number of CTA partials (atomics or slots), + 1 for the float64 reference.  1 - I/U, the flatten loss and the EDT
sigmoid get first-order bounds (their comments derive them).  Each check prints its largest error / bound ratio.
"""
import functools
import math

import numpy as np
import pytest
import torch

import loss_ref as R
import mesh_oracle as MO
from loss_ref import U32, gamma
from umr_b200 import ops
from umr_b200 import soft_renderer as sr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PAD = 4096   # guard elements on each side (16 KB: keeps the view 16-byte aligned)


@pytest.fixture(params=[False, True], ids=["default", "deterministic"])
def det(request):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(request.param)
    yield request.param
    torch.use_deterministic_algorithms(prev)


def guarded(t, offset=0):
    """A contiguous CUDA copy of `t` inside a NaN-filled buffer (PAD + offset elements before, PAD after)."""
    t = t.contiguous()
    buf = torch.full((t.numel() + 2 * PAD + offset,), float("nan"), dtype=t.dtype, device=DEV)
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
    ratio = float((err / bound.clamp_min(1e-300))[mask if mask is not None else torch.ones_like(ok)].max()) \
        if err.numel() else 0.0
    print("%-52s max err/bound = %.3e" % (name, ratio))
    assert torch.isfinite(got).all(), "%s: non-finite output (a read outside an input?)" % name
    assert bool(ok.all()), "%s: %d values outside the bound, worst ratio %.3g" % (name, int((~ok).sum()), ratio)


# -------------------------------------------------------------------------------------------------
# sampler
# -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 2, 3, 4])
@pytest.mark.parametrize("H,W", [(1, 7), (6, 1), (17, 23)])
def test_sampler(det, C, H, W):
    g = torch.Generator().manual_seed(C * 100 + H)
    B, N = 2, 1000                                                                  # N not a multiple of 256
    img = torch.rand(B, C, H, W, generator=g) * 2 - 1
    flow = torch.rand(B, N, 2, generator=g) * 2.4 - 1.2
    flow[:, :8] = torch.tensor([[-1.0, -1.0], [1.0, 1.0], [1.0, -1.0], [-1.0, 1.0], [0.0, 0.0], [1.0, 0.0],
                                [0.0, -1.0], [-1.0, 0.0]])
    k = torch.randint(0, 64, (B, 200, 2), generator=g).float()                     # texel centres
    flow[:, 8:208, 0] = (2 * (k[..., 0] % max(W, 1)) / max(W - 1, 1) - 1).float()
    flow[:, 8:208, 1] = (2 * (k[..., 1] % max(H, 1)) / max(H - 1, 1) - 1).float()
    flow[:, 208:240] = torch.tensor([1e6, -1e6, 3e5, -7e5])[torch.randint(0, 4, (B, 32, 2), generator=g)]
    up = torch.rand(B, N, C, generator=g) * 2 - 1
    ig = guarded(img).requires_grad_(True)
    fg = guarded(flow).requires_grad_(True)
    out = ops.bilinear_sample(ig, fg)
    (out * up.to(DEV)).sum().backward()
    imd = img.double().requires_grad_(True)
    fld = flow.double().requires_grad_(True)
    ref = R.sample_ref(imd, fld)
    gi, gf = torch.autograd.grad((ref * up.double()).sum(), (imd, fld))
    m_out, m_gf, m_gi, cnt = R.sample_magnitude(img.double(), flow, up.double())
    tag = "sampler C=%d %dx%d %s" % (C, H, W, "det" if det else "")
    _check(tag + " out", out, ref, gamma(8 + 1) * m_out)                          # weights 3, products 1, sums 3
    _check(tag + " grad_flow", fg.grad, gf, gamma(8 + C + 2) * m_gf)             # weights 2, diff/mul/add 3, C, scale 2
    _check(tag + " grad_image", ig.grad, gi, gamma(5 + cnt + 1) * m_gi)          # per term 5, one add per term


# -------------------------------------------------------------------------------------------------
# IoU
# -------------------------------------------------------------------------------------------------
def _iou_bounds(p, t, gl, n_cta, per_thread):
    """(loss bound [B], grad bound [B,N], I, U) for per-image 1 - I/U summed in float32 by k_iou_partial."""
    li, I, U = R.iou_ref(p, t)
    _, Im, Um = R.iou_ref(p, t, magnitude=True)
    D = 3 + per_thread + 5 + 5 + n_cta + 1
    eI, eU = gamma(D) * Im, gamma(D + 1) * Um                                      # U: + the 1e-6
    # 1 - I/U: |d| <= eI / U + (I / U) eU / U, and the division and subtraction round once each
    lb = (eI + I / U * eU) / U + gamma(2) * (I / U + li.abs())
    # grad = -g (t U - I (1 - t)) / U^2 with the kernel's I, U: first order in eI, eU plus its own roundings (6 in
    # k_iou_bwd; 8 in k_losshead_bwd, whose alpha gradient then adds the three L1 terms)
    t2, a = t.reshape(t.shape[0], -1), gl.abs()[:, None]
    mag = t2.abs() * U[:, None] + I[:, None] * (1 - t2).abs()
    gb = a * ((1 - t2).abs() / U[:, None] ** 2 * eI[:, None] + (3 * mag) / U[:, None] ** 3 * eU[:, None]) \
        + gamma(12) * a * mag / U[:, None] ** 2
    return lb, gb


@pytest.mark.parametrize("N,stride", [(4096, 0), (16383, 0), (16385, 0), (3 * 16384 + 5, 0), (2 * 16384 + 4, 1)])
def test_iou(det, N, stride):
    g = torch.Generator().manual_seed(N)
    B = 3
    p = torch.rand(B, N, generator=g)
    t = (torch.rand(B, N, generator=g) > 0.5).float()
    p[2], t[2] = 0, 0                                                               # all-zero image
    gl = torch.rand(B, generator=g) + 0.5
    if stride:                                                                      # odd batch stride: scalar path
        full = guarded(torch.cat([p, torch.zeros(B, 1)], 1))
        pg = full[:, :N]
    else:
        pg = guarded(p)
    pg.requires_grad_(True)
    loss = ops.neg_iou_per_image(pg, guarded(t))
    (loss * gl.to(DEV)).sum().backward()
    pd = p.double().requires_grad_(True)
    li, _, _ = R.iou_ref(pd, t.double())
    gp, = torch.autograd.grad((li * gl.double()).sum(), pd)
    n_cta = math.ceil(N / 16384)
    lb, gb = _iou_bounds(p.double(), t.double(), gl.double(), n_cta, 32)
    tag = "iou N=%d%s %s" % (N, " strided" if stride else "", "det" if det else "")
    _check(tag + " loss", loss, li, lb)
    _check(tag + " grad", pg.grad, gp, gb)


# -------------------------------------------------------------------------------------------------
# masked L1
# -------------------------------------------------------------------------------------------------
def _l1_kinks(pred, gt, mgt, mpred):
    """[B,C,HW] elements whose sign the float32 kernel may see differently (|d| within its rounding bound of 0)."""
    B, C = pred.shape[:2]
    a, b = pred.reshape(B, C, -1) * mpred.reshape(B, 1, -1), gt.reshape(B, C, -1) * mgt.reshape(B, 1, -1)
    return (a - b).abs() <= gamma(3) * (a.abs() + b.abs())


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("HW", [1600, 2049, 3 * 2048 + 7])
def test_masked_l1(det, C, HW):
    g = torch.Generator().manual_seed(C * HW)
    B = 3
    rgba = torch.rand(B, 4, HW, generator=g)
    gt = torch.rand(B, C, HW, generator=g)
    mgt = (torch.rand(B, HW, generator=g) > 0.4).float()
    gl = torch.rand(B, generator=g) + 0.5
    buf = guarded(rgba).requires_grad_(True)                                       # strided views of one RGBA render
    pred, mpred = buf[:, :C].reshape(B, C, HW, 1), buf[:, 3].reshape(B, HW, 1)
    loss = ops.masked_l1_per_image(pred, guarded(gt).reshape(B, C, HW, 1), guarded(mgt).reshape(B, HW, 1), mpred)
    (loss * gl.to(DEV)).sum().backward()
    rd = rgba.double().requires_grad_(True)
    args = (rd[:, :C].reshape(B, C, HW, 1), gt.double().reshape(B, C, HW, 1), mgt.double(), rd[:, 3])
    ref = R.masked_l1_ref(*args)
    gr, = torch.autograd.grad((ref * gl.double()).sum(), rd)
    mag = R.masked_l1_ref(*[a.detach() for a in args], magnitude=True)
    n_cta = math.ceil(HW / 2048)
    tag = "masked l1 C=%d HW=%d %s" % (C, HW, "det" if det else "")
    _check(tag + " loss", loss, ref, gamma(3 + 8 * C + 5 + 5 + n_cta + 2 + 1) * mag)
    kink = _l1_kinks(rgba[:, :C].double(), gt.double(), mgt.double(), rgba[:, 3].double())
    k = (gl.double() / (C * HW))[:, None, None]
    ok = torch.ones(B, 4, HW, dtype=torch.bool)
    ok[:, :C] = ~kink
    ok[:, 3] = ~kink.any(1)
    gbound = torch.zeros(B, 4, HW, dtype=torch.float64)
    gbound[:, :C] = gamma(4) * k * rgba[:, 3:4].double()
    gbound[:, 3] = gamma(C + 4) * (k * rgba[:, :C].double()).sum(1)
    _check(tag + " grad", buf.grad, gr, gbound, ok)


# -------------------------------------------------------------------------------------------------
# fused loss head
# -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W", [(1, 1, 2049), (33, 1, 2049), (128, 1, 2049), (2, 600, 600)])
def test_loss_head(det, B, H, W):
    g = torch.Generator().manual_seed(B * H * W)
    HW = H * W
    rgba = torch.rand(B, 4, H, W, generator=g)
    gt = torch.rand(B, 3, H, W, generator=g)
    mgt = (torch.rand(B, H, W, generator=g) > 0.4).float()
    w_iou, w_tex = 2.5, 3.0
    x = guarded(rgba).requires_grad_(True)
    loss, per = ops.mask_texture_loss(x, guarded(gt), guarded(mgt), w_iou, w_tex)
    loss.backward()
    rd = rgba.double().requires_grad_(True)
    ref, per_ref = R.loss_head_ref(rd, gt.double(), mgt.double(), w_iou, w_tex)
    gr, = torch.autograd.grad(ref, rd)
    n_cta = math.ceil(HW / 2048)
    tag = "loss head B=%d %dx%d %s" % (B, H, W, "det" if det else "")
    gl_iou = torch.full((B,), w_iou / B, dtype=torch.float64)
    lb_iou, gb_iou = _iou_bounds(rgba[:, 3].double(), mgt.double(), gl_iou, n_cta, 8)
    args = (rgba[:, :3].double(), gt.double(), mgt.double(), rgba[:, 3].double())
    lb_tex = gamma(3 + 24 + 5 + 5 + n_cta + 2 + 1) * R.masked_l1_ref(*args, magnitude=True)
    _check(tag + " per-image 1 - IoU", per[:, 0], per_ref[:, 0], lb_iou)
    _check(tag + " per-image L1", per[:, 1], per_ref[:, 1], lb_tex)
    # finalize: one warp, ceil(B / 32) sequential adds per lane, the warp tree, / B, the weights and their sum
    Df = math.ceil(B / 32) + 5 + 4 + 1
    lb = (w_iou * lb_iou.sum() + w_tex * lb_tex.sum()) / B \
        + gamma(Df) * (w_iou * per_ref[:, 0].abs().mean() + w_tex * per_ref[:, 1].abs().mean())
    _check(tag + " loss", loss, ref, lb.detach())
    kink = _l1_kinks(*args)
    kt = w_tex / (B * 3 * HW)
    ok = torch.ones(B, 4, HW, dtype=torch.bool)
    ok[:, :3] = ~kink.reshape(B, 3, HW)
    ok[:, 3] = ~kink.reshape(B, 3, HW).any(1)
    gb = torch.zeros(B, 4, HW, dtype=torch.float64)
    gb[:, :3] = gamma(6) * kt * rgba[:, 3:4].reshape(B, 1, HW).double()
    gb[:, 3] = gb_iou + gamma(3 + 6) * kt * rgba[:, :3].reshape(B, 3, HW).double().sum(1)
    _check(tag + " grad", x.grad.reshape(B, 4, HW), gr.reshape(B, 4, HW), gb, ok)


# -------------------------------------------------------------------------------------------------
# chamfer
# -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,N,M,D", [(2, 20, 7, 2), (2, 33, 33, 3), (3, 31, 33, 2), (1, 20000, 642, 3)])
def test_chamfer(det, B, N, M, D):
    g = torch.Generator().manual_seed(N * M + D)
    a = torch.rand(B, N, D, generator=g) - 0.5
    b = torch.rand(B, M, D, generator=g) - 0.5
    a[:, 9 % N] = a[:, 4]                                                           # duplicate points
    b[:, 5] = b[:, 2]
    w1, w2 = torch.rand(B, N, generator=g), torch.rand(B, M, generator=g)
    ag, bg = guarded(a).requires_grad_(True), guarded(b).requires_grad_(True)
    d_ab, d_ba, i_ab, i_ba = ops.dist_chamfer(ag, bg)
    ((d_ab * w1.to(DEV)).sum() + (d_ba * w2.to(DEV)).sum()).backward()
    ad, bd = a.double(), b.double()
    _, _, r_ab, r_ba = R.chamfer_ref(ad, bd)
    i_ab, i_ba = i_ab.cpu().long(), i_ba.cpu().long()
    assert R.near_tie(ad, bd, i_ab, r_ab, 2).all() and R.near_tie(bd, ad, i_ba, r_ba, 2).all()
    ar, br = ad.clone().requires_grad_(True), bd.clone().requires_grad_(True)
    e_ab, e_ba, _, _ = R.chamfer_ref(ar, br, i_ab, i_ba)
    ga, gb = torch.autograd.grad((e_ab * w1.double()).sum() + (e_ba * w2.double()).sum(), (ar, br))
    am, bm = ad.abs().requires_grad_(True), bd.abs().requires_grad_(True)
    m_ab, m_ba, _, _ = R.chamfer_ref(am, bm, i_ab, i_ba, magnitude=True)
    gam, gbm = torch.autograd.grad((m_ab * w1.double()).sum() + (m_ba * w2.double()).sum(), (am, bm))
    tag = "chamfer B=%d N=%d M=%d D=%d %s" % (B, N, M, D, "det" if det else "")
    _check(tag + " d_ab", d_ab, e_ab, gamma(6 + 1) * m_ab)
    _check(tag + " d_ba", d_ba, e_ba, gamma(6 + 1) * m_ba)
    # a point's gradient: its own term + one per point that picked it; 2 roundings a term, the gather adds its tree
    cnt = 1 + max(int(torch.bincount(i_ba.reshape(-1) + N * torch.arange(B).repeat_interleave(M)).max()),
                  int(torch.bincount(i_ab.reshape(-1) + M * torch.arange(B).repeat_interleave(N)).max()))
    _check(tag + " grad a", ag.grad, ga, gamma(2 + cnt + 6 + 1) * gam)
    _check(tag + " grad b", bg.grad, gb, gamma(2 + cnt + 6 + 1) * gbm)


# -------------------------------------------------------------------------------------------------
# texture cycle
# -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T2", [1, 36, 64])
def test_texcycle(det, T2):
    g = torch.Generator().manual_seed(T2)
    B, F, P = 3, 200, 1023                                                          # B*F = 600: 3 CTAs; P % 4 != 0
    flow = torch.rand(B, F, T2, 2, generator=g) * 2 - 1
    prob = torch.rand(B, F, 2, generator=g) * 2 - 1
    ids = torch.randint(-F - 3, F + 3, (B, P), generator=g).float()               # ids >= F, < -1 and < -F
    ids[1, :5] = torch.tensor([-1.0, -2.0, float(F), -float(F) - 2, 7.0])
    gl = 0.75
    fg = guarded(flow).requires_grad_(True)
    loss = ops.tex_cycle(fg, guarded(prob), guarded(ids))
    (loss * gl).backward()
    vis = R.visible_ref(ids, F)
    fd = flow.double().requires_grad_(True)
    ref = R.texcycle_ref(fd, prob.double(), vis)
    gf, = torch.autograd.grad(ref * gl, fd)
    mag = R.texcycle_ref(flow.double(), prob.double(), vis, magnitude=True)
    n_cta = math.ceil(B * F / 256)
    tag = "texcycle T2=%d %s" % (T2, "det" if det else "")
    _check(tag + " loss", loss, ref, gamma(T2 + 4 + 5 + 5 + n_cta + 2 + 1) * mag)
    k = 2 * gl / (B * F * 2) / T2
    gm = k * (flow.double().abs().mean(2) + prob.double().abs()) * vis[:, :, None]
    _check(tag + " grad", fg.grad, gf, gamma(T2 + 6 + 1) * gm[:, :, None, :].expand(-1, -1, T2, -1))


# -------------------------------------------------------------------------------------------------
# Laplacian and flatten
# -------------------------------------------------------------------------------------------------
def _deformed(v, f, B, seed):
    """[B,V,3] float32 shapes of one mesh: random radial noise, plus per item a planar cap (exactly flat dihedrals),
    a vertex pushed through the surface (folded dihedrals) and a vertex 1e-4 from a neighbour (edges < sqrt(eps))."""
    rng = np.random.default_rng(seed)
    x = v[None] * rng.uniform(0.7, 1.3, (B, len(v), 1))
    for b in range(B):
        kind = b % 4
        if kind == 1:
            x[b, :, 2] = np.minimum(x[b, :, 2], 0.6)
        elif kind == 2:
            k = rng.integers(len(v))
            x[b, k] *= -0.3
        elif kind == 3:
            t = f[rng.integers(len(f))]
            x[b, t[0]] = x[b, t[1]] + rng.uniform(-1e-4, 1e-4, 3)
    return torch.from_numpy(x.astype(np.float32))


@functools.lru_cache(maxsize=None)
def _mesh_reference(mesh, B):
    """The float64 results and bounds of one (mesh, B) case, shared by both modes (the flatten bound takes seconds)."""
    v, f = R.spiked_uv_sphere(*mesh)
    x = _deformed(v, f, B, sum(mesh))
    gl = torch.rand(B, generator=torch.Generator().manual_seed(B)) + 0.5
    lap = sr.LaplacianLoss(torch.from_numpy(v), torch.from_numpy(f))
    flat = sr.FlattenLoss(torch.from_numpy(f))
    E, V = flat.edge_table.shape[0], len(v)
    deg = int(torch.diff(lap.csr_rowptr).max())
    # Laplacian: y = deg + 1 roundings, |y|^2 3 more; the gradient 2 g (y_j + sum tcoef y_i)
    xd = x.double().requires_grad_(True)
    lref, _ = R.laplacian_ref(xd, lap.csr_rowptr, lap.csr_col, lap.csr_coef)
    lgrad, = torch.autograd.grad((lref * gl.double()).sum(), xd)
    xm = x.double().abs().requires_grad_(True)
    lmag, _ = R.laplacian_ref(xm, lap.csr_rowptr, lap.csr_col, lap.csr_coef, magnitude=True)
    lgm, = torch.autograd.grad((lmag * gl.double()).sum(), xm)
    lap_bounds = (gamma(deg + 4 + 5 + 5 + math.ceil(V / 256) + 1) * lmag, gamma(2 * deg + 6) * lgm)
    # flatten: first-order bound (loss_ref.flatten_error_bound); the loss sum: per-thread 1, warp trees 10, CTAs
    eps = float(np.float32(1e-6))
    xd = x.double().requires_grad_(True)
    fref = R.flatten_ref(xd, flat.edge_table, eps)
    fgrad, = torch.autograd.grad((fref * gl.double()).sum(), xd)
    fb = R.flatten_error_bound(x, flat.edge_table, eps, gl, 1 + 10 + math.ceil(E / 128) + 1)
    return v, f, x, gl, (lref.detach(), lgrad) + lap_bounds, (fref.detach(), fgrad) + fb


@pytest.mark.parametrize("mesh,B", [((21, 12, 15), 4), ((11, 12, 9), 64)])   # V = 257; E = 387
def test_laplacian_flatten(det, mesh, B):
    v, f, x, gl, lap_ref, flat_ref = _mesh_reference(mesh, B)
    lap = sr.LaplacianLoss(torch.from_numpy(v), torch.from_numpy(f)).to(DEV)
    flat = sr.FlattenLoss(torch.from_numpy(f)).to(DEV)
    tag = "V=%d E=%d B=%d %s" % (len(v), flat.edge_table.shape[0], B, "det" if det else "")
    for name, mod, (ref, gref, lb, gb) in (("laplacian", lap, lap_ref), ("flatten", flat, flat_ref)):
        xg = guarded(x).requires_grad_(True)
        loss = mod(xg)
        (loss * gl.to(DEV)).sum().backward()
        _check(name + " " + tag + " loss", loss, ref, lb)
        _check(name + " " + tag + " grad", xg.grad, gref, gb)


# -------------------------------------------------------------------------------------------------
# distance transform
# -------------------------------------------------------------------------------------------------
def _edt_cases():
    rng = np.random.default_rng(11)
    tall = (rng.uniform(size=(3, 61, 17)) > 0.7).astype(np.float32)
    row = (rng.uniform(size=(2, 1, 50)) > 0.8).astype(np.float32)
    col = (rng.uniform(size=(2, 50, 1)) > 0.8).astype(np.float32)
    wide = np.zeros((2, 3, 4096), np.float32)
    wide[0, 1, 4000] = 1
    wide[1, :, :2048] = 1
    dots = np.zeros((3, 20, 24), np.float32)
    dots[0, 0, 0] = 1
    dots[1, 19, 23] = 1
    dots[2] = 1
    dots[2, 10, 11] = 0
    nonbin = rng.choice(np.float32([0, 0.25, 0.5, 1, 2]), size=(2, 19, 21)).astype(np.float32)
    degenerate = np.stack([np.zeros((7, 9), np.float32), np.ones((7, 9), np.float32), np.full((7, 9), 0.5, np.float32)])
    return {"tall": tall, "row": row, "column": col, "4096 wide": wide, "one pixel": dots, "non-binary": nonbin,
            "degenerate": degenerate}


@pytest.mark.parametrize("name", list(_edt_cases()))
def test_dt_barrier(det, name):
    m = _edt_cases()[name]
    got = ops.dt_barrier(guarded(torch.from_numpy(m))).cpu().double()
    k = 50.0
    ref = np.stack([R.dt_barrier_ref(mi, k) for mi in m])
    # the kernel rounds its double result to float once (1 ulp of float32(ref) covers it and the float64 reference),
    # and multiplies by float32(1 / max(H, W)): a relative error u of k * diff moves the sigmoid s by s (1 - s) |k diff| u
    d2o, d2i = zip(*[R.edt_sq_brute(mi) for mi in m])
    kd = k * np.abs(np.sqrt(np.stack(d2o)) - np.sqrt(np.stack(d2i))) / max(m.shape[1:])
    bound = np.spacing(ref.astype(np.float32)).astype(np.float64) + ref * (1 - ref) * kd * U32
    _check("dt_barrier %s %s" % (name, "det" if det else ""), got, torch.from_numpy(ref.astype(np.float32)),
           torch.from_numpy(bound))


def test_dt_barrier_width_limit():
    ops.dt_barrier(torch.zeros(1, 2, 4096, device=DEV))
    with pytest.raises(RuntimeError):
        ops.dt_barrier(torch.zeros(1, 2, 4097, device=DEV))


# -------------------------------------------------------------------------------------------------
# texture atlas
# -------------------------------------------------------------------------------------------------
def edge_uv_faces(rng, n):
    """Faces at the edges of the uv range: whole faces on u or v = 0 or 1, the four corners, negative uv."""
    faces = []
    for c in (0.0, 1.0):
        for axis in (0, 1):
            f = rng.uniform(0, 1, size=(3, 2))
            f[:, axis] = c
            faces.append(f)
    faces += [np.full((3, 2), c) for c in (0.0, 1.0)]
    faces += [np.array([[0, 1], [1, 1], [1, 0]]), np.array([[1, 1], [1, 1], [0, 0]])]
    faces += [rng.uniform(-1.5, 0.0, size=(3, 2)), rng.uniform(-0.2, 1.0, size=(3, 2)), np.full((3, 2), -1.0)]
    faces = np.stack(faces).astype(np.float32)
    return faces[np.arange(n) % len(faces)]


@pytest.mark.parametrize("R_,H,W", [(1, 2, 2), (1, 17, 9), (4, 2, 2), (5, 64, 48)])
def test_load_textures_edges(det, R_, H, W):
    rng = np.random.default_rng(R_ * H * W)
    F = 26
    image = rng.uniform(0, 1, size=(H, W, 3)).astype(np.float32)
    uv = edge_uv_faces(rng, F)
    upd = np.ones(F, np.int32)
    upd[3] = 0
    base = rng.uniform(0, 1, size=(F, R_ * R_, 3)).astype(np.float32)
    tex = guarded(torch.from_numpy(base))
    ops.load_textures(guarded(torch.from_numpy(image)), guarded(torch.from_numpy(uv)), tex, torch.from_numpy(upd).to(DEV))
    got = tex.cpu().numpy()
    ref = MO.load_textures_np(image, uv, upd, base)
    assert np.isfinite(got).all(), "load_textures read outside the image (NaN from the guard band)"
    assert np.array_equal(got, ref), "max diff %g" % np.abs(got - ref).max()
    print("load_textures R=%d %dx%d: bit-exact, finite" % (R_, H, W))


def test_create_texture_image_one_texel_many_faces():
    F, R_, res = 5120, 1, 4
    rng = np.random.default_rng(12)
    tex = rng.uniform(0, 1, size=(F, R_ * R_, 3)).astype(np.float32)
    img, vt = sr.functional.create_texture_image(guarded(torch.from_numpy(tex)), res)
    tile_width = int((F - 1.) ** 0.5) + 1
    tile_height = int((F - 1.) / tile_width) + 1
    n = np.arange(F)
    col, row = (n % tile_width).astype(np.float32), (n // tile_width).astype(np.float32)
    v = np.zeros((F, 3, 2), np.float32)
    v[:, 0, 0] = col * res + res / 2; v[:, 0, 1] = row * res + 1
    v[:, 1, 0] = col * res + 1;       v[:, 1, 1] = (row + 1) * res - 1 - 1
    v[:, 2, 0] = (col + 1) * res - 1 - 1; v[:, 2, 1] = (row + 1) * res - 1 - 1
    ref = MO.create_texture_image_np(v, tex, np.ones((tile_height * res, tile_width * res, 3), np.float32))[::-1]
    assert np.isfinite(img).all() and np.array_equal(img, ref)
