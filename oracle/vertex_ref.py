"""Float64 reference of the fused vertex kernels (umr_b200/csrc/vertex.cu) -- TEST INFRASTRUCTURE ONLY.

Restates, in float64 torch on the CPU, the reference chain that `k_project_faces` fuses and that `k_corr_fwd`
implements; gradients come from autograd.  Each step cites the reference line it follows:

  nnutils/geom_utils.py:74-91     orthographic_proj_withz: quat_rotate (:147-165, two hamilton_product :119-144),
                                  scale, translate, z offset
  nnutils/smr.py:36               y *= -1
  SoftRas functional/look_at.py:48-60   v - eye, then R; for an eye on the negative z axis R is the identity
  SoftRas functional/orthogonal.py:13-16   x, y *= viewing_scale
  SoftRas functional/face_vertices.py:16-22   gather [B,F,3,3]
  SoftRas mesh.py:112-118         n = normalize(cross(v2 - v1, v0 - v1), eps=1e-6) on the flipped, pre-look_at corners
  SoftRas lighting.py:50-57, functional/ambient_lighting.py:17, functional/directional_lighting.py:26-27
                                  light = Ia * ca + Id * (cd * relu(n . d))   (d is used as given, not normalised)
  nnutils/loss_utils.py:194-248   CorrLossChamfer: project the part vertices, nearest target of each part
                                  (chamfer_python.py:43-64, expanded form |q|^2 + |t|^2 - 2 q.t), weighted mean

`magnitude=True` evaluates the same expression tree with every subtraction turned into an addition; the caller
passes |inputs| (as leaves, so that autograd sees them) and the light stage, which is not polynomial, is left out.  For a polynomial computed in floating point with one
rounding per operation, |fl(e) - e| <= gamma_n * e_abs, where e_abs is that evaluation and n the longest chain of
roundings (Higham, Accuracy and Stability of Numerical Algorithms, §3.1); autograd through the magnitude tree
with |upstream gradients| gives e_abs of each gradient.  tests/test_vertex_range_gpu.py builds its tolerances
from it.
"""
import operator

import torch


def _hamilton(qa, qb, sub):
    """geom_utils.py:119-144, with `sub` for each minus sign."""
    a0, a1, a2, a3 = qa.unbind(-1)
    b0, b1, b2, b3 = qb.unbind(-1)
    q0 = sub(sub(sub(a0 * b0, a1 * b1), a2 * b2), a3 * b3)
    q1 = sub(a0 * b1 + a1 * b0 + a2 * b3, a3 * b2)
    q2 = sub(a0 * b2, a1 * b3) + a2 * b0 + a3 * b1
    q3 = sub(a0 * b3 + a1 * b2, a2 * b1) + a3 * b0
    return torch.stack([q0, q1, q2, q3], dim=-1)


def project_vertices(X, cams, offset_z=0.0, magnitude=False):
    """orthographic_proj_withz (geom_utils.py:74-91): X [B,V,3], cams [B,7] (scale, tx, ty, quaternion) -> [B,V,3]."""
    sub = operator.add if magnitude else operator.sub
    q = cams[:, None, 3:7].expand(-1, X.shape[1], -1)
    conj = q if magnitude else torch.cat([q[..., :1], -q[..., 1:]], dim=-1)        # quat_rotate :159
    Xq = torch.cat([X[..., :1] * 0, X], dim=-1)                                     # :160
    r = _hamilton(q, _hamilton(Xq, conj, sub), sub)[..., 1:]                        # :161-165
    s = cams[:, None, 0:1]
    xy = s * r[..., :2] + cams[:, None, 1:3]
    z = s * r[..., 2:] + offset_z
    return torch.cat([xy, z], dim=-1)


def _face_index(faces, B, H):
    """faces [F,3], [1,F,3] or [Bv,F,3] -> [B,F,3] long: render b uses mesh b // H (H camera hypotheses per mesh)."""
    f = faces.long()
    if f.dim() == 2:
        f = f[None]
    if f.shape[0] == 1:
        return f.expand(B, -1, -1)
    return f.repeat_interleave(H, dim=0)


def _gather(v, idx):
    """face_vertices.py:16-22: v [B,V,3], idx [B,F,3] -> [B,F,3,3]."""
    B, F = idx.shape[:2]
    return torch.gather(v, 1, idx.reshape(B, F * 3, 1).expand(-1, -1, 3)).reshape(B, F, 3, 3)


def project_faces_ref(vertices, cams, faces, offset_z=5.0, eye_z=-2.732, viewing_scale=1.0, flip_y=True, light=None,
                      magnitude=False, with_pre=False):
    """vertices [Bv,V,3], cams [Bv*H,7], faces [F,3] | [1,F,3] | [Bv,F,3] -> (fv [B,F,3,3], light [B,F,3] | None),
    B = Bv*H.  light = (Ia, colour_a, Id, colour_d, direction) as `umr_b200.vertex.project_faces` takes it.
    with_pre: also return the flipped pre-look_at corners [B,F,3,3] (the normals' input, mesh.py:112-118)."""
    B, Bv = cams.shape[0], vertices.shape[0]
    H = B // Bv
    X = vertices.repeat_interleave(H, dim=0) if H > 1 else vertices
    p = project_vertices(X, cams, offset_z, magnitude)                              # smr.py:82
    if flip_y and not magnitude:
        p = p * torch.tensor([1.0, -1.0, 1.0], dtype=p.dtype)                       # smr.py:36
    ez = abs(eye_z) if magnitude else -eye_z
    vs = abs(viewing_scale) if magnitude else viewing_scale
    out = torch.stack([p[..., 0] * vs, p[..., 1] * vs, p[..., 2] + ez], dim=-1)    # look_at (R = I), orthogonal
    idx = _face_index(faces, B, H)
    fv, pre = _gather(out, idx), _gather(p, idx)
    lt = None
    if light is not None and not magnitude:
        ia, ca, idir, cd, d = light
        ca, cd, d = (torch.as_tensor(x, dtype=fv.dtype) for x in (ca, cd, d))
        n = torch.cross(pre[:, :, 2] - pre[:, :, 1], pre[:, :, 0] - pre[:, :, 1], dim=2)  # mesh.py:114-116
        n = torch.nn.functional.normalize(n, p=2, dim=2, eps=1e-6)
        cosine = torch.relu((n * d).sum(2))                                         # directional_lighting.py:26
        lt = ia * ca + idir * (cd * cosine[:, :, None])                             # ambient :17, directional :27
    if with_pre:
        return fv, lt, pre
    return fv, lt


U32 = 2.0 ** -24   # unit roundoff of float32


def gamma(n):
    """gamma_n = n u / (1 - n u): the relative error bound of n float32 roundings in a chain."""
    return n * U32 / (1 - n * U32)


def normal_conditioning(vertices, cams, faces, offset_z, flip_y, exact_corners=False):
    """Per face: (n exact [B,F,3], |n| clamped at the 1e-6 eps [B,F], kappa = |n_abs| / max(|n|, eps) [B,F],
    |a_abs| + |b_abs| [B,F]) where a = v2 - v1, b = v0 - v1 and *_abs is the magnitude evaluation.
    exact_corners: the caller knows the float32 corners are exact (e.g. an identity camera on dyadic coordinates),
    so a and b carry no rounding and their magnitudes are |a|, |b|."""
    _, _, pre = project_faces_ref(vertices, cams, faces, offset_z, -1.0, 1.0, flip_y, None, with_pre=True)
    _, _, pre_m = project_faces_ref(vertices.abs(), cams.abs(), faces, abs(offset_z), -1.0, 1.0, flip_y, None,
                                    magnitude=True, with_pre=True)
    a, b = pre[:, :, 2] - pre[:, :, 1], pre[:, :, 0] - pre[:, :, 1]
    am, bm = pre_m[:, :, 2] + pre_m[:, :, 1], pre_m[:, :, 0] + pre_m[:, :, 1]
    if exact_corners:
        am, bm = a.abs(), b.abs()
    n = torch.cross(a, b, dim=2)
    nm = torch.stack([am[..., 1] * bm[..., 2] + am[..., 2] * bm[..., 1], am[..., 2] * bm[..., 0] + am[..., 0] * bm[..., 2],
                      am[..., 0] * bm[..., 1] + am[..., 1] * bm[..., 0]], dim=-1)
    N = n.norm(dim=2).clamp_min(1e-6)
    return n, N, nm.norm(dim=2) / N, am.norm(dim=2) + bm.norm(dim=2)


def light_error_bound(vertices, cams, faces, offset_z, flip_y, light, exact_corners=False):
    """Bound [B,F,3] on |light_float32 - light| of `k_project_faces` (and of any float32 chain of the same ops).

    The normal n = a x b is a polynomial of the inputs 13 roundings deep, so |dn| <= gamma_13 |n_abs|.  Normalising
    is Lipschitz: |d n_hat| <= 2 |dn| / max(|n|, eps) + gamma_5 (|x|^2 sum, sqrt, divide) <= gamma_13 (2 kappa + 1).
    The dot with d adds gamma_3 |d|, and relu is 1-Lipschitz.  The last three roundings (Id * (cd * cos),
    Ia * ca + ...) add gamma_3 of the light's magnitude.  With 24 >= 13 + 5 + 3 + 3:
        |d light_c| <= gamma_24 (|Ia ca_c| + |Id cd_c| (|cos| + (2 kappa + 1) |d|_2))."""
    ia, ca, idir, cd, d = light
    ca, cd, d = (torch.as_tensor(x, dtype=torch.float64) for x in (ca, cd, d))
    n, N, kappa, _ = normal_conditioning(vertices, cams, faces, offset_z, flip_y, exact_corners)
    cos = ((n / N[..., None]) * d).sum(2).abs()
    dn = d.norm()
    return gamma(24) * (abs(ia) * ca.abs() + abs(idir) * cd.abs() * (cos + (2 * kappa + 1) * dn)[..., None])


def light_grad_magnitude(vertices, cams, faces, offset_z, flip_y, light, g_light, exact_corners=False):
    """Per face corner [B,F,3,3]: a first-order bound, in units of gamma_D, on the error of the light's contribution to
    the corner gradients in `k_scatter_face_grads`, for faces that are lit (the relu passes) -- 0 elsewhere.

    With G = gc d, gc = Id sum_c cd_c g_c, and N = max(|n|, eps), the kernel forms G_n = (G - n_hat (n_hat . G)) / N
    (G / N on the eps branch), |G_n| <= 2 |G| / N, and d/dn of G_n is at most 3 |G| / N^2.  A relative error
    gamma kappa of n therefore moves G_n by 3 gamma kappa |G| / N, its own roundings by gamma 2|G| / N; the corner
    terms b x G_n and G_n x a then carry |db| |G_n| + |b| |dG_n| + 2 gamma |b| |G_n|.  Collected with |b| <= |b_abs|:
        <= gamma (9 + 3 kappa) |G| (|a_abs| + |b_abs|) / N  <=  gamma 12 (kappa + 1) |G| (|a_abs| + |b_abs|) / N
    per component and per corner."""
    ia, ca, idir, cd, d = light
    cd, d = (torch.as_tensor(x, dtype=torch.float64) for x in (cd, d))
    n, N, kappa, ab = normal_conditioning(vertices, cams, faces, offset_z, flip_y, exact_corners)
    lit = ((n / N[..., None]) * d).sum(2) > 0
    G = abs(idir) * (cd.abs() * g_light.abs()).sum(2) * d.norm()
    m = torch.where(lit, 12 * (kappa + 1) * G * ab / N, torch.zeros_like(N))
    return m[:, :, None, None].expand(-1, -1, 3, 3)


def project_grad_magnitude(vertices, cams, faces, offset_z, eye_z, viewing_scale, g_fv, g_pre=None):
    """(vertices, cams) gradient magnitudes: autograd through the magnitude evaluation of the projection with
    upstream |g_fv| on the raster-space corners and `g_pre` (>= 0) on the pre-look_at corners."""
    va = vertices.detach().abs().requires_grad_(True)
    ca = cams.detach().abs().requires_grad_(True)
    fv, _, pre = project_faces_ref(va, ca, faces, abs(offset_z), eye_z, viewing_scale, False, None, magnitude=True,
                                   with_pre=True)
    s = (fv * g_fv.abs()).sum()
    if g_pre is not None:
        s = s + (pre * g_pre).sum()
    gv, gc = torch.autograd.grad(s, (va, ca))
    return gv, gc


def corr_chamfer_ref(verts, cams, parts, targets, weights=(1, 1, 0, 0), nearest=None, magnitude=False):
    """CorrLossChamfer (loss_utils.py:194-248) in float64.

    verts [1,V,3] (one mesh for every render) or [B,V,3]; cams [B,7]; parts = 4 index tensors (head, belly, neck,
    back); targets = 4 tensors [B,m_g,2]; weights = 4 floats.  -> (loss [B], vert2d [B,NS,2], nearest [B,NS] long).
    The nearest target of each vertex is the brute-force argmin over its own part, lowest index on ties as
    torch.min; `nearest` overrides it (a test passes the kernel's choice once it has checked it is a near-tie)."""
    sel = torch.cat([torch.as_tensor(p).long() for p in parts])
    B = cams.shape[0]
    X = verts[:, sel, :]
    if X.shape[0] == 1 and B > 1:
        X = X.expand(B, -1, -1)
    q = project_vertices(X, cams, 0.0, magnitude)[..., :2]                          # smr.py:76-78, loss_utils.py:231
    add_or_sub = operator.add if magnitude else operator.sub
    terms, idx, start = [], [], 0
    for p, t, w in zip(parts, targets, weights):
        n = len(p)
        qp = q[:, start:start + n]
        qq = (qp * qp).sum(-1)                                                      # chamfer_python.py:56-63
        kk = (t * t).sum(-1)
        zz = torch.einsum("bnd,bmd->bnm", qp, t)
        P = add_or_sub(qq[:, :, None] + kk[:, None, :], 2 * zz)
        if nearest is None:
            i = torch.argmin(P.detach(), dim=2) if n else torch.zeros(B, 0, dtype=torch.long)
        else:
            i = nearest[:, start:start + n].long()
        idx.append(i)
        terms.append(torch.gather(P, 2, i[:, :, None])[:, :, 0] * (abs(w) if magnitude else w))  # loss_utils.py:236
        start += n
    loss = torch.cat(terms, 1).mean(1)                                              # :239
    return loss, q, torch.cat(idx, 1)
