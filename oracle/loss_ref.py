"""Float64 reference of the loss and mesh-op kernels (umr_b200/csrc/losses.cu, mesh_ops.cu) -- TEST INFRASTRUCTURE ONLY.

Restates, in float64 torch on the CPU, the reference expression each kernel implements; gradients come from autograd.
Each function cites the reference lines it follows:

  sample_ref        nnutils/geom_utils.py:41-59 `sample_textures`, loss_utils.py:59-64: grid_sample, bilinear, zeros
                    padding, the torch-1.1 coordinate map (align_corners=True) ix = ((x + 1) / 2) * (W - 1)
  iou_ref           nnutils/loss_utils.py:41-48 `neg_iou_loss` (per image, avg=False form)
  masked_l1_ref     nnutils/loss_utils.py:103-116 `texture_loss_masks` (per image, avg=False form)
  loss_head_ref     the two above on one RGBA render, weighted batch means (train_s1.py:211-215)
  chamfer_ref       nnutils/chamfer_python.py:43-64 `distChamfer`, expanded form |q|^2 + |k|^2 - 2 q.k
  visible_ref / texcycle_ref   nnutils/loss_utils.py:152-182 `TexCycle.forward`
  laplacian_ref     SoftRas/losses.py:6-37 `LaplacianLoss` (the row-normalised matrix as a neighbour list)
  flatten_ref       SoftRas/losses.py:39-114 `FlattenLoss`
  edt_sq_brute / dt_barrier_ref   utils/image.py:130-141 `compute_dt_barrier` (scipy's distance_transform_edt)

Two places keep float32 on purpose:
* The sampler's coordinate map is computed in float32, as torch and the kernel do: `floor` of it then falls on the same
  side of a texel boundary, and everything after it is float64.  Its gradient is the exact (W - 1) / 2.
* Chamfer: the caller may pass the kernel's nearest indices after checking that each differing one is a near-tie; the
  distances and gradients then follow that choice.

`magnitude=True` (where offered) evaluates the same expression tree on |inputs| with every subtraction turned into an
addition.  For a polynomial computed in floating point with one rounding per operation, |fl(e) - e| <= gamma_n * e_abs,
where e_abs is that evaluation and n the longest chain of roundings (Higham, Accuracy and Stability of Numerical
Algorithms, §3.1).  The flatten loss is not polynomial (sqrt, divisions): `flatten_error_bound` gives a first-order
bound from the sensitivity of the result to a relative perturbation of every rounded operation.
"""
import numpy as np
import torch

from vertex_ref import U32, gamma

__all__ = ["U32", "gamma", "sample_ref", "sample_magnitude", "iou_ref", "masked_l1_ref", "loss_head_ref", "chamfer_ref",
           "near_tie", "visible_ref", "texcycle_ref", "laplacian_ref", "flatten_ref", "flatten_error_bound", "spiked_uv_sphere",
           "edt_sq_brute", "dt_barrier_ref"]


# -------------------------------------------------------------------------------------------------
# bilinear sampler
# -------------------------------------------------------------------------------------------------
def _coords(flow, W, H):
    """float32 pixel coordinates of flow [B,N,2] exactly as torch / k_sample_* compute them, as float64 tensors that
    carry the map's exact derivative (W - 1) / 2 when `flow` requires grad."""
    f = flow.detach().float()
    ix32 = ((f[..., 0] + 1) / 2) * (W - 1)
    iy32 = ((f[..., 1] + 1) / 2) * (H - 1)
    ix, iy = ix32.double(), iy32.double()
    if flow.requires_grad:
        fx, fy = flow[..., 0].double(), flow[..., 1].double()
        ix = ix + (fx * ((W - 1) / 2) - (fx * ((W - 1) / 2)).detach())
        iy = iy + (fy * ((H - 1) / 2) - (fy * ((H - 1) / 2)).detach())
    return ix32, iy32, ix, iy


def _corners(image, ix32, iy32):
    """The four corners of every sample: [(x, y, valid [B,N], value [B,C,N])] in the order 00, 10, 01, 11."""
    B, C, H, W = image.shape
    x0, y0 = torch.floor(ix32).double(), torch.floor(iy32).double()
    out = []
    for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
        x, y = x0 + dx, y0 + dy
        ok = (x >= 0) & (x < W) & (y >= 0) & (y < H)
        flat = torch.where(ok, y.clamp(0, H - 1) * W + x.clamp(0, W - 1), torch.zeros_like(x)).long()
        val = torch.gather(image.reshape(B, C, H * W), 2, flat[:, None, :].expand(B, C, -1))
        out.append((x, y, ok, torch.where(ok[:, None, :], val, torch.zeros_like(val))))
    return out


def sample_ref(image, flow):
    """grid_sample(image, flow, bilinear, zeros, align_corners=True): image [B,C,H,W] float64, flow [B,N,2] (float32
    values; float64 leaves for gradients) -> [B,N,C] float64."""
    B, C, H, W = image.shape
    ix32, iy32, ix, iy = _coords(flow, W, H)
    (x0, y0, _, a00), (x1, _, _, a10), (_, y1, _, a01), (_, _, _, a11) = _corners(image, ix32, iy32)
    wx1, wx0, wy1, wy0 = x1 - ix, ix - x0, y1 - iy, iy - y0
    out = a00 * (wx1 * wy1)[:, None] + a10 * (wx0 * wy1)[:, None] + a01 * (wx1 * wy0)[:, None] + a11 * (wx0 * wy0)[:, None]
    return out.permute(0, 2, 1)


def sample_magnitude(image, flow, g):
    """Magnitudes of the sampler's outputs for the error bounds: (out [B,N,C], grad_flow [B,N,2], grad_image [B,C,H,W],
    the largest number of corner terms one pixel receives).  g [B,N,C] is the upstream gradient."""
    B, C, H, W = image.shape
    ix32, iy32, ix, iy = _coords(flow.detach(), W, H)
    cs = _corners(image.abs(), ix32, iy32)
    (x0, y0, k00, a00), (x1, _, k10, a10), (_, y1, k01, a01), (_, _, k11, a11) = cs
    wx1, wx0, wy1, wy0 = x1 - ix, ix - x0, y1 - iy, iy - y0
    w = (wx1 * wy1, wx0 * wy1, wx1 * wy0, wx0 * wy0)
    out = sum(a * wk[:, None] for (_, _, _, a), wk in zip(cs, w)).permute(0, 2, 1)
    ga = g.abs().permute(0, 2, 1)                                                   # [B,C,N]
    gx = (ga * ((a10 + a00) * wy1[:, None] + (a11 + a01) * wy0[:, None])).sum(1) * ((W - 1) / 2)
    gy = (ga * ((a01 + a00) * wx1[:, None] + (a11 + a10) * wx0[:, None])).sum(1) * ((H - 1) / 2)
    gimg = torch.zeros(B, C, H * W, dtype=torch.float64)
    cnt = torch.zeros(B, H * W, dtype=torch.float64)
    for (x, y, ok, _), wk in zip(cs, w):
        flat = torch.where(ok, y * W + x, torch.zeros_like(x)).long()
        gimg.scatter_add_(2, flat[:, None, :].expand(B, C, -1), ga * (wk * ok)[:, None])
        cnt.scatter_add_(1, flat, ok.double())
    return out, torch.stack([gx, gy], -1), gimg.reshape(B, C, H, W), int(cnt.max())


# -------------------------------------------------------------------------------------------------
# IoU, masked L1, fused loss head
# -------------------------------------------------------------------------------------------------
def iou_ref(p, t, magnitude=False):
    """loss_utils.py:41-48 per image: p, t [B, ...] -> (1 - I/U [B], I [B], U [B]) with U including the 1e-6."""
    p, t = p.reshape(p.shape[0], -1), t.reshape(t.shape[0], -1)
    if magnitude:
        p, t = p.abs(), t.abs()
        return None, (p * t).sum(1), (p + t + p * t).sum(1) + 1e-6
    inter = (p * t).sum(1)                                                          # :44
    union = (p + t - p * t).sum(1) + 1e-6                                           # :45
    return 1 - inter / union, inter, union                                          # :48


def masked_l1_ref(img_pred, img_gt, mask_gt, mask_pred, magnitude=False):
    """loss_utils.py:103-116, avg=False: per image mean over (C,H,W) of |img_pred * mask_pred - img_gt * mask_gt|."""
    B, C, H, W = img_pred.shape
    a, b = img_pred * mask_pred.reshape(B, 1, H, W), img_gt * mask_gt.reshape(B, 1, H, W)
    d = (a.abs() + b.abs()) if magnitude else (a - b).abs()
    return d.sum((1, 2, 3)) / (C * H * W)


def loss_head_ref(rgba, img_gt, mask_gt, w_iou, w_tex):
    """`ops.mask_texture_loss`: w_iou * mean_b neg_iou(alpha, mask) + w_tex * mean_b masked_l1(rgb, gt, mask, alpha)
    -> (loss, per_image [B,2])."""
    li, _, _ = iou_ref(rgba[:, 3], mask_gt)
    lt = masked_l1_ref(rgba[:, :3], img_gt, mask_gt, rgba[:, 3])
    return w_iou * li.mean() + w_tex * lt.mean(), torch.stack([li, lt], 1)


# -------------------------------------------------------------------------------------------------
# chamfer
# -------------------------------------------------------------------------------------------------
def _sqdist(q, k, magnitude=False):
    """chamfer_python.py:56-63 expanded: [B,NQ,NK] = |q|^2 + |k|^2 - 2 q.k (magnitude: + 2 q.k, on |q|, |k| the caller
    passes, so that autograd through them gives the gradients' magnitudes)."""
    qq, kk = (q * q).sum(-1), (k * k).sum(-1)
    zz = torch.einsum("bnd,bmd->bnm", q, k)
    s = qq[:, :, None] + kk[:, None, :]
    return s + 2 * zz if magnitude else s - 2 * zz


def chamfer_ref(a, b, idx_ab=None, idx_ba=None, magnitude=False):
    """distChamfer (chamfer_python.py:43-64) in float64: a [B,N,D], b [B,M,D] -> (d_ab [B,N], d_ba [B,M], idx_ab,
    idx_ba).  The nearest point is the float64 argmin (lowest index on ties, as torch.min) unless idx_* is given.
    magnitude=True: the caller passes |a|, |b| and the nearest indices."""
    P = _sqdist(a, b, magnitude)
    if idx_ab is None:
        idx_ab = torch.argmin(P.detach(), 2)
    if idx_ba is None:
        idx_ba = torch.argmin(P.detach(), 1)
    d_ab = torch.gather(P, 2, idx_ab.long()[:, :, None])[:, :, 0]
    d_ba = torch.gather(P, 1, idx_ba.long()[:, None, :])[:, 0, :]
    return d_ab, d_ba, idx_ab, idx_ba


def near_tie(a, b, idx_kernel, idx_ref, dim):
    """True where the kernel's nearest index is the float64 one or a near-tie of it: the two float64 distances differ
    by no more than both distances' float32 rounding bound (the rule of test_losses_gpu.py::test_chamfer, with the
    bound gamma_6 * magnitude of the expanded form instead of a fixed 4.8e-7)."""
    P, Pm = _sqdist(a, b), _sqdist(a.abs(), b.abs(), magnitude=True)
    pick = lambda X, i: torch.gather(X, dim, i.long().unsqueeze(dim)).squeeze(dim)   # noqa: E731
    diff = (pick(P, idx_kernel) - pick(P, idx_ref)).abs()
    return (idx_kernel.long() == idx_ref.long()) | (diff <= gamma(6) * (pick(Pm, idx_kernel) + pick(Pm, idx_ref)))


# -------------------------------------------------------------------------------------------------
# texture cycle
# -------------------------------------------------------------------------------------------------
def visible_ref(ids, F):
    """loss_utils.py:174-179: the faces whose id appears in each face-id plane ids [B,P] -> [B,F] bool.  An id in
    [-F, -1] marks face id + F, as Python indexing does there (-1, the background, marks the last face).  Ids >= F or
    < -F name no face and mark nothing (the reference's indexing raises on them)."""
    B = ids.shape[0]
    f = ids.long()                                   # the kernel's (int) truncates toward zero, as .long() does
    f = torch.where(f < 0, f + F, f)
    vis = torch.zeros(B, F + 1, dtype=torch.bool)
    f = torch.where((f >= 0) & (f < F), f, torch.full_like(f, F))
    vis.scatter_(1, f, torch.ones_like(f, dtype=torch.bool))
    return vis[:, :F]


def texcycle_ref(flow, prob, vis, magnitude=False):
    """loss_utils.py:156-182: flow [B,F,T2,2], prob [B,F,2], vis [B,F] -> MSE over B*F*2 of (mean_t flow - prob) on the
    visible faces (0 elsewhere)."""
    B, F = prob.shape[:2]
    m = vis.to(flow.dtype)[:, :, None]
    avg = flow.abs().mean(2) if magnitude else flow.mean(2)                        # :170
    d = (avg + prob.abs()) if magnitude else (avg - prob)
    return ((d * m) ** 2).sum() / (B * F * 2)                                       # :181 MSELoss (mean)


# -------------------------------------------------------------------------------------------------
# mesh regularisers
# -------------------------------------------------------------------------------------------------
def laplacian_ref(x, rowptr, col, coef, magnitude=False):
    """SoftRas/losses.py:31-37 with the row-normalised Laplacian given as CSR off-diagonal entries (coef = -1/deg as
    float32, `LaplacianLoss`'s own values): x [B,V,3] -> (sum_i |y_i|^2 [B], y [B,V,3]), y = x + L_off x.
    magnitude=True: the caller passes |x| (a leaf, so that autograd through it gives the gradient's magnitude)."""
    V = x.shape[1]
    rows = torch.repeat_interleave(torch.arange(V), torch.diff(torch.as_tensor(rowptr).long()))
    c = torch.as_tensor(coef).double()
    if magnitude:
        c = c.abs()
    y = x.index_add(1, rows, x[:, torch.as_tensor(col).long()] * c[None, :, None])
    return (y * y).sum((1, 2)), y


class _Rounder:
    """Marks each rounded operation of an expression with a relative perturbation: r(x) = x (1 + d_f) + (x - x)' d_b,
    d_f, d_b = 0.  d_f perturbs the value, d_b (zero in value) the gradient flowing back through it, so derivatives of
    a result or of an autograd gradient with respect to them are the first-order effects of one rounding there."""

    def __init__(self, on):
        self.on, self.deltas = on, []

    def __call__(self, x):
        if not self.on:
            return x
        df = torch.zeros_like(x, requires_grad=True)
        db = torch.zeros_like(x, requires_grad=True)
        self.deltas += [df, db]
        return x * (1 + df) + (x - x.detach()) * db


def _flatten_terms(P, eps, r):
    """k_flatten's per-edge expression, one r() per rounded operation: P [B,E,4,3] corners (v0, v1, v2, v3) -> [B,E]
    (cos + 1)^2 (SoftRas/losses.py:71-108)."""
    def dot(u, v):
        return r(r(r(u[..., 0] * v[..., 0]) + r(u[..., 1] * v[..., 1])) + r(u[..., 2] * v[..., 2]))

    def perp(a, b):                                                                 # losses.py:77-90 (and :92-105)
        al2, bl2 = dot(a, a), dot(b, b)
        al1, bl1 = r(torch.sqrt(r(al2 + eps))), r(torch.sqrt(r(bl2 + eps)))
        ab = dot(a, b)
        cos = r(ab / r(r(al1 * bl1) + eps))
        sin = r(torch.sqrt(r(r(1 - r(cos * cos)) + eps)))
        k = r(ab / r(al2 + eps))
        return r(b - r(a * k[..., None])), r(bl1 * sin)
    v0, v1, v2, v3 = P.unbind(2)
    a = r(v1 - v0)
    cb1, l1 = perp(a, r(v2 - v0))
    cb2, l2 = perp(a, r(v3 - v0))
    cos = r(dot(cb1, cb2) / r(r(l1 * l2) + eps))                                   # :107
    return r(r(cos + 1) * r(cos + 1))                                               # :108


def flatten_ref(vertices, edges, eps=1e-6):
    """SoftRas/losses.py:71-114, average=False: vertices [B,V,3], edges [E,4] (v0, v1, v2, v3) -> [B]."""
    P = vertices[:, torch.as_tensor(edges).long()]                                  # [B,E,4,3]
    return _flatten_terms(P, eps, _Rounder(False)).sum(1)


def flatten_error_bound(vertices, edges, eps, grad_loss, reduce_depth):
    """First-order bounds on k_flatten's float32 error: (loss [B], grad_vertices [B,V,3]).

    Every rounded operation of the kernel is one `_Rounder` perturbation of relative size <= u, so the error of an
    edge's term is at most u * sum |d term / d delta| to first order.  The forward is one perturbation per operation,
    as the kernel computes it.  The kernel's hand-derived backward forms each local derivative of that tree with at
    most 4 roundings, so the gradient sensitivities count 4 times.  Both are doubled to cover second-order terms and
    the float64 reference's own rounding.  The sums over edges add gamma_{reduce_depth} (loss) or gamma_{count + 2}
    (one rounding per term a vertex receives, 2 more for v0's term -(da + db1 + db2)) times the sum of |terms|."""
    E = edges.shape[0]
    B, V = vertices.shape[:2]
    idx = torch.as_tensor(edges).long()
    P = vertices.detach().double()[:, idx].clone().requires_grad_(True)
    r = _Rounder(True)
    t = _flatten_terms(P, float(eps), r)
    gl = grad_loss.detach().double()[:, None]
    G, = torch.autograd.grad((t * gl).sum(), P, create_graph=True)                 # [B,E,4,3] per-edge terms
    per_edge = lambda ds: sum(d.abs().reshape(B, E, -1).sum(-1) for d in ds if d is not None)   # noqa: E731
    sens_t = per_edge(torch.autograd.grad(t.sum(), r.deltas, retain_graph=True, allow_unused=True))
    loss_bound = 2 * U32 * sens_t.sum(1) + gamma(reduce_depth) * t.detach().abs().sum(1)
    sens_g = torch.zeros(B, E, 4, 3, dtype=torch.float64)
    for k in range(4):
        for d in range(3):
            ds = torch.autograd.grad(G[:, :, k, d].sum(), r.deltas, retain_graph=True, allow_unused=True)
            sens_g[:, :, k, d] = per_edge(ds)
    Gd = G.detach()
    term_bound = 8 * U32 * sens_g
    term_bound[:, :, 0] += gamma(2) * Gd[:, :, 1:].abs().sum(2)
    count = torch.bincount(idx.reshape(-1), minlength=V).max().item()
    flat = idx.reshape(-1)
    gb = torch.zeros(B, V, 3, dtype=torch.float64).index_add_(1, flat, term_bound.reshape(B, E * 4, 3))
    ga = torch.zeros(B, V, 3, dtype=torch.float64).index_add_(1, flat, Gd.abs().reshape(B, E * 4, 3))
    return loss_bound, gb + gamma(count + 2) * ga


def spiked_uv_sphere(n_lat, n_lon, n_spikes):
    """A closed non-icosphere mesh: a latitude / longitude sphere (poles of valence n_lon, ring vertices 6) with a
    vertex inserted at the centroid of `n_spikes` faces (valence 3)."""
    v = [[0.0, 0.0, 1.0]]
    for i in range(1, n_lat):
        th = np.pi * i / n_lat
        for j in range(n_lon):
            ph = 2 * np.pi * j / n_lon
            v.append([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
    v.append([0.0, 0.0, -1.0])
    ring = lambda i, j: 1 + (i - 1) * n_lon + j % n_lon   # noqa: E731
    f = [[0, ring(1, j), ring(1, j + 1)] for j in range(n_lon)]
    for i in range(1, n_lat - 1):
        for j in range(n_lon):
            f += [[ring(i, j), ring(i + 1, j), ring(i + 1, j + 1)], [ring(i, j), ring(i + 1, j + 1), ring(i, j + 1)]]
    S = len(v) - 1
    f += [[S, ring(n_lat - 1, j + 1), ring(n_lat - 1, j)] for j in range(n_lon)]
    v, f = np.array(v), [list(t) for t in f]
    step = max(1, len(f) // max(n_spikes, 1))
    for k in range(n_spikes):
        a, b, c = f[k * step]
        vn = len(v)
        v = np.vstack([v, v[[a, b, c]].mean(0) * 1.02])
        f[k * step] = [a, b, vn]
        f += [[b, c, vn], [c, a, vn]]
    return v.astype(np.float32), np.array(f, np.int64)


# -------------------------------------------------------------------------------------------------
# distance transform
# -------------------------------------------------------------------------------------------------
def edt_sq_brute(mask):
    """Exact squared Euclidean distances of scipy's `distance_transform_edt(1 - mask)` and `(mask)` by brute force over
    every pixel pair: mask [H,W] -> (d2_out, d2_in) int64 [H,W].  The features of d2_out are the pixels equal to 1, of
    d2_in those equal to 0.  With no feature pixel at all, scipy measures from a virtual pixel at (row -1, column 0)."""
    m = np.asarray(mask)
    H, W = m.shape
    yy, xx = np.mgrid[0:H, 0:W]
    out = []
    for feat in (m == 1, m == 0):
        fy, fx = np.nonzero(feat)
        if fy.size == 0:
            fy, fx = np.array([-1]), np.array([0])
        d2 = np.full((H, W), np.iinfo(np.int64).max, np.int64)
        for k in range(0, fy.size, 256):                                            # bounded memory
            dy = yy[..., None] - fy[None, None, k:k + 256]
            dx = xx[..., None] - fx[None, None, k:k + 256]
            d2 = np.minimum(d2, (dy * dy + dx * dx).min(-1))
        out.append(d2)
    return out[0], out[1]


def dt_barrier_ref(mask, k=50.0):
    """utils/image.py:130-141 from the exact squared distances, in float64: mask [H,W] -> [H,W]."""
    d2o, d2i = edt_sq_brute(mask)
    diff = (np.sqrt(d2o.astype(np.float64)) - np.sqrt(d2i.astype(np.float64))) / max(np.asarray(mask).shape)
    return 1. / (1 + np.exp(k * -diff))
