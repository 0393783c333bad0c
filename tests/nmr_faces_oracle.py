"""CPU oracle of the functional rasteriser's geometry gradient (DESIGN.md §14) -- test infrastructure.

A numpy float32 restatement of what `umr_nmr_backward_faces` computes, on top of the render oracle `oracle/nmr.py`:
every edge and depth term is evaluated with one rounding per operation in the contract's order, so it is the kernel's
term bit for bit; the terms are then summed in float64.  The kernel sums the same terms in float32 in its own order,
so `magnitude=True` also returns sum |term| and the number of terms per coordinate, what that sum's error bound needs.

    faces    [B,F,3,3] float32 NDC face coordinates (the functional API's input)
    textures [B,F,T,T,T,3] float32 or None
    grad_*   output adjoints: rgb [B,3,is,is], alpha / depth [B,is,is], or None
"""
import numpy as np

import nmr

f32 = np.float32


def zbuffer(faces, image_size, anti_aliasing=True, near=0.1, far=100.0):
    """The forward's face-index and raster-depth planes for face coordinates: one copy per face, eye_z = 0."""
    faces = np.asarray(faces, f32)
    B, F = faces.shape[:2]
    idx = np.arange(3 * F).reshape(1, F, 3).repeat(B, 0)
    return nmr.zbuffer(faces.reshape(B, 3 * F, 3), idx, image_size, anti_aliasing, False, 0.0, near, far)


def render(faces, textures=None, image_size=256, anti_aliasing=True, near=0.1, far=100.0, background_color=(0, 0, 0)):
    """The functional forward: oracle/nmr.py's render with fill_back off, eye_z = 0 and light exactly 1."""
    faces = np.asarray(faces, f32)
    B, F = faces.shape[:2]
    idx = np.arange(3 * F).reshape(1, F, 3).repeat(B, 0)
    return nmr.render(faces.reshape(B, 3 * F, 3), idx, textures, image_size, anti_aliasing, False, 0.0, near, far,
                      1.0, 0.0, background_color=background_color)


def raster_colour(faces, textures, fidx, background_color=(0, 0, 0)):
    """[B,S,S,3] colour at raster resolution (the background where no face wins), k_nmr_shade's op sequence."""
    faces = np.asarray(faces, f32)
    B, F = faces.shape[:2]
    S = fidx.shape[1]
    idx = np.arange(3 * F).reshape(1, F, 3).repeat(B, 0)
    verts = faces.reshape(B, 3 * F, 3)
    T = textures.shape[2]
    light = nmr.lights(nmr.face_copies(verts, idx, False), 1.0, 0.0)
    out = np.empty((B, S, S, 3), f32)
    out[:] = np.asarray(background_color, f32)
    b, yi, xi, f, fc, texel, weight = nmr._samples(fidx, verts, idx, T, False, 0.0, S)
    tex = np.asarray(textures, f32).reshape(B, F, T ** 3, 3)[b, f]
    for c in range(3):
        s = np.zeros(len(b), f32)
        for pn in range(8):
            s = s + weight[:, pn] * (tex[np.arange(len(b)), texel[:, pn], c] * light[b, fc, c])
        out[b, yi, xi, c] = s
    return out


def raster_grad(g, S, anti_aliasing):
    """Output adjoint [B,(C,)is,is] -> raster resolution [B,S,S(,C)] float32: flip, and / 4 with anti-aliasing."""
    g = np.asarray(g, f32)
    if g.ndim == 4:
        g = np.moveaxis(g, 1, -1)
    if anti_aliasing:
        g = np.repeat(np.repeat(g, 2, axis=1), 2, axis=2) / f32(4)
    return np.ascontiguousarray(g[:, ::-1]).astype(f32)


class _Acc:
    def __init__(self, shape):
        self.grad = np.zeros(shape)
        self.mag = np.zeros(shape)
        self.cnt = np.zeros(shape, np.int64)

    def add(self, at, terms):
        t = np.asarray(terms, f32).astype(np.float64)
        self.grad[at] += t.sum()
        self.mag[at] += np.abs(t).sum()
        self.cnt[at] += t.size


def grad_faces(faces, textures=None, grad_rgb=None, grad_alpha=None, grad_depth=None, image_size=256,
               anti_aliasing=True, near=0.1, far=100.0, eps=1e-4, background_color=(0, 0, 0), zbuf=None,
               magnitude=False):
    """The contract's geometry gradient [B,F,3,3] (float64 sums of the float32 terms).  `magnitude` also returns the sum
    of |term| and the number of terms per coordinate."""
    faces = np.asarray(faces, f32)
    B, F = faces.shape[:2]
    S = image_size * (2 if anti_aliasing else 1)
    Sf, eps = f32(S), f32(eps)
    if zbuf is None:
        zbuf = zbuffer(faces, image_size, anti_aliasing, near, far)
    fidx = zbuf[0]
    A = (fidx >= 0).astype(f32)
    use_rgb, use_alpha = grad_rgb is not None, grad_alpha is not None
    R = raster_colour(faces, textures, fidx, background_color) if use_rgb else None
    gR = raster_grad(grad_rgb, S, anti_aliasing) if use_rgb else None
    gA = raster_grad(grad_alpha, S, anti_aliasing) if use_alpha else None
    acc = _Acc((B, F, 3, 3))
    with np.errstate(all="ignore"):
        if use_rgb or use_alpha:
            for b in range(B):
                for f in range(F):
                    _edge_terms(acc, b, f, faces[b, f], fidx[b], A[b], None if R is None else R[b],
                                None if gA is None else gA[b], None if gR is None else gR[b], S, Sf, eps)
        if grad_depth is not None:
            _depth_terms(acc, faces, fidx, raster_grad(grad_depth, S, anti_aliasing), S)
    if magnitude:
        return acc.grad, acc.mag, acc.cnt
    return acc.grad


def _edge_terms(acc, b, f, face, fidx, A, R, gA, gR, S, Sf, eps):
    x, y = face[:, 0], face[:, 1]
    if not np.isfinite(face).all():
        return
    if (y[2] - y[0]) * (x[1] - x[0]) < (y[1] - y[0]) * (x[2] - x[0]):  # back-facing
        return
    px = f32(0.5) * ((x * Sf + Sf) - f32(1))
    py = f32(0.5) * ((y * Sf + Sf) - f32(1))
    for e in range(3):
        ka, kb, ko = e, (e + 1) % 3, (e + 2) % 3
        for axis in range(2):
            U, W = (px, py) if axis == 0 else (py, px)
            ua, ub, uo, va, vb, vo = U[ka], U[kb], U[ko], W[ka], W[kb], W[ko]
            if ua == ub:
                continue
            direction = (-1 if ua < ub else 1) if axis == 0 else (1 if ua < ub else -1)
            comp = 1 if axis == 0 else 0
            lo = max(np.ceil(min(ua, ub)), f32(0))
            hi = min(np.floor(max(ua, ub)), f32(S - 1))
            for d0 in range(int(lo), int(hi) + 1) if lo <= hi else ():
                d0f = f32(d0)
                vc = ((vb - va) / (ub - ua)) * (d0f - ua) + va
                fin = np.floor(vc) if direction > 0 else np.ceil(vc)
                if not (f32(0) <= fin <= Sf - f32(1)):
                    continue
                i_in = int(fin)
                i_out = i_in + direction
                if not 0 <= i_out < S:
                    continue
                line = (slice(None), d0) if axis == 0 else (d0, slice(None))
                fl, al = fidx[line], A[line]
                rl, gal, grl = (None if R is None else R[line]), (None if gA is None else gA[line]), \
                    (None if gR is None else gR[line])

                def terms(ps, ref):
                    diff = np.zeros(len(ps), f32)
                    if gal is not None:
                        diff = diff + (al[ps] - al[ref]) * gal[ps]
                    if grl is not None:
                        for ch in range(3):
                            diff = diff + (rl[ps, ch] - rl[ref, ch]) * grl[ps, ch]
                    keep = diff > 0
                    ps, diff = ps[keep], diff[keep]
                    dd = ps.astype(f32) - vc
                    if ub != d0f:
                        dist = ((((ub - ua) / (ub - d0f)) * dd) * f32(2)) / Sf
                        dist = np.where(dist > 0, dist + eps, dist - eps)
                        acc.add((b, f, ka, comp), -(diff / dist))
                    if ua != d0f:
                        dist = ((((ub - ua) / (d0f - ua)) * dd) * f32(2)) / Sf
                        dist = np.where(dist > 0, dist + eps, dist - eps)
                        acc.add((b, f, kb, comp), -(diff / dist))
                if fl[i_in] == f:   # growing: out .. border
                    terms(np.arange(i_out, S) if direction > 0 else np.arange(0, i_out + 1), i_in)
                if (d0f - ua) * (d0f - uo) < 0:
                    xc = ((vo - va) / (uo - ua)) * (d0f - ua) + va
                else:
                    xc = ((vb - vo) / (ub - uo)) * (d0f - uo) + vo
                lf = np.ceil(xc) if direction > 0 else np.floor(xc)
                lf = fin if np.isnan(lf) else min(max(lf, f32(-1)), Sf)
                lim = int(lf)
                ps = np.arange(max(min(i_in, lim), 0), min(max(i_in, lim), S - 1) + 1)
                terms(ps[fl[ps] == f], i_out)   # shrinking: this face's pixels from in to the other edge


def _depth_terms(acc, faces, fidx, gD, S):
    B, F = faces.shape[:2]
    idx = np.arange(3 * F).reshape(1, F, 3).repeat(B, 0)
    fv = nmr.face_copies(faces.reshape(B, 3 * F, 3), idx, False)
    _, z, inv = nmr._records(fv, S, 0.0)
    half = f32(0.5) * f32(S)
    b, yi, xi = np.nonzero(fidx >= 0)
    g = gD[b, yi, xi]
    keep = g != 0
    b, yi, xi, g = b[keep], yi[keep], xi[keep], g[keep]
    fc = fidx[b, yi, xi].astype(np.int64)
    w, zp = nmr.bary(inv[b, fc], z[b, fc], xi.astype(f32), yi.astype(f32))
    zz = z[b, fc]
    iv = inv[b, fc]
    a = (zp * zp) * g
    sx = (iv[:, 0, 0] / zz[:, 0] + iv[:, 1, 0] / zz[:, 1]) + iv[:, 2, 0] / zz[:, 2]
    sy = (iv[:, 0, 1] / zz[:, 0] + iv[:, 1, 1] / zz[:, 1]) + iv[:, 2, 1] / zz[:, 2]
    for k in range(3):
        t = a * w[k]
        for comp, term in ((0, (t * sx) * half), (1, (t * sy) * half), (2, t / (zz[:, k] * zz[:, k]))):
            term = term.astype(f32).astype(np.float64)
            np.add.at(acc.grad, (b, fc, k, comp), term)
            np.add.at(acc.mag, (b, fc, k, comp), np.abs(term))
            np.add.at(acc.cnt, (b, fc, k, comp), 1)
