"""CPU oracle of the NMR render contract (DESIGN.md §7) -- TEST INFRASTRUCTURE ONLY (never imported by umr_b200/).

A numpy float32 restatement of what `umr_nmr_forward` / `umr_nmr_backward_textures` compute: one rounding per
operation, in the contract's order, with NMR's double-literal clamps written as the selections they are (NaN -> 0,
like the device's fmax).  The z-buffer walks the face copies in ascending order with a strict '<', as NMR's
per-pixel loop does.  The texture gradient is the exact adjoint of the (texture-linear) render, in float64.

    vertices [B,V,3] f32  (after orthographic_proj_withz(..., offset_z=5) and the y flip, before look_at)
    faces    [B,F,3] int
    textures [B,F,T,T,T,3] f32
"""
import numpy as np

f32 = np.float32


def pixel_coords(S):
    """(2 i + 1 - S) / S in double, stored as float (NMR's pixel centres)."""
    i = np.arange(S, dtype=np.float64)
    return ((2.0 * i + 1.0 - S) / S).astype(f32)


def face_copies(vertices, faces, fill_back=True):
    """[B,Fc,3,3] f32 vertices of every face copy; copies F..2F-1 have the vertex order reversed.  A vertex index
    outside [0,V) gives NaN coordinates (that face is never drawn)."""
    vertices = np.asarray(vertices, f32)
    faces = np.asarray(faces).astype(np.int64)
    if fill_back:
        faces = np.concatenate([faces, faces[:, :, ::-1]], axis=1)
    V = vertices.shape[1]
    ok = (faces >= 0) & (faces < V)
    fv = np.take_along_axis(vertices[:, None], np.where(ok, faces, 0)[..., None], axis=2)
    fv = fv.reshape(faces.shape + (3,)).copy()
    fv[~ok] = np.nan
    return fv


def lights(fv, Ia=0.5, Id=0.5, ca=(1, 1, 1), cd=(1, 1, 1), direction=(0, 1, 0)):
    """[B,Fc,3]: Ia*ca + Id*(cd*relu(n.d)), n = normalize(cross(v0 - v1, v2 - v1), eps=1e-5), from the vertices before
    look_at.  A term whose intensity is 0 is not added (NMR adds it only when non-zero)."""
    ca, cd, d = (np.asarray(x, f32) for x in (ca, cd, direction))
    Ia, Id = f32(Ia), f32(Id)
    with np.errstate(all="ignore"):
        a = fv[..., 0, :] - fv[..., 1, :]
        b = fv[..., 2, :] - fv[..., 1, :]
        c0 = a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1]
        c1 = a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2]
        c2 = a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]
        den = np.fmax(np.sqrt((c0 * c0 + c1 * c1) + c2 * c2), f32(1e-5))
        cos = ((c0 / den) * d[0] + (c1 / den) * d[1]) + (c2 / den) * d[2]
        cos = np.where(cos < 0, f32(0), cos)
        light = np.zeros(fv.shape[:2] + (3,), f32)
        if Ia != 0:
            light = light + Ia * ca
        if Id != 0:
            light = light + Id * (cd * cos[..., None])
    return light.astype(f32)


def _records(fv, S, eye_z):
    """NDC xy [..,3,2], depth after look_at [..,3], pixel-unit barycentric inverse [..,3,3]."""
    Sf = f32(S)
    xy = fv[..., :2]
    z = fv[..., 2] - f32(eye_z)
    p = f32(0.5) * ((xy * Sf + Sf) - f32(1))
    px, py = p[..., 0], p[..., 1]
    inv = np.stack([py[..., 1] - py[..., 2], px[..., 2] - px[..., 1], px[..., 1] * py[..., 2] - px[..., 2] * py[..., 1],
                    py[..., 2] - py[..., 0], px[..., 0] - px[..., 2], px[..., 2] * py[..., 0] - px[..., 0] * py[..., 2],
                    py[..., 0] - py[..., 1], px[..., 1] - px[..., 0], px[..., 0] * py[..., 1] - px[..., 1] * py[..., 0]],
                   axis=-1)
    den = (px[..., 2] * (py[..., 0] - py[..., 1]) + px[..., 0] * (py[..., 1] - py[..., 2])) + px[..., 1] * (py[..., 2] - py[..., 0])
    with np.errstate(all="ignore"):
        inv = (inv / den[..., None]).reshape(fv.shape[:-2] + (3, 3))
    return xy, z.astype(f32), inv.astype(f32)


def bary(inv, z, xi, yi):
    """w = clamp01(inv . (xi, yi, 1)) renormalised by its sum, zp = 1 / (w0/z0 + w1/z1 + w2/z2).  inv [..,3,3],
    z [..,3], xi / yi float32 arrays broadcasting against the leading dims."""
    with np.errstate(all="ignore"):
        w = [np.fmin(np.fmax((inv[..., k, 0] * xi + inv[..., k, 1] * yi) + inv[..., k, 2], f32(0)), f32(1))
             for k in range(3)]
        s = ((f32(0) + w[0]) + w[1]) + w[2]
        w = [wk / s for wk in w]
        zp = f32(1) / ((w[0] / z[..., 0] + w[1] / z[..., 1]) + w[2] / z[..., 2])
    return w, zp


def _region(xy, S, exhaustive):
    """Pixel rectangle (c0, c1, r0, r1) that holds every pixel the edge tests of this face can admit: the bounding
    box widened by 4 px + 1e-3 (1 + max|coord|) NDC; the whole image for thin (sine of the smallest angle below 1e-2)
    or non-finite faces."""
    if exhaustive:
        return 0, S - 1, 0, S - 1
    q = xy.astype(np.float64)
    m = np.abs(q).max()
    (x0, y0), (x1, y1), (x2, y2) = q
    l = sorted([(x1 - x0) ** 2 + (y1 - y0) ** 2, (x2 - x0) ** 2 + (y2 - y0) ** 2, (x2 - x1) ** 2 + (y2 - y1) ** 2])
    a2 = (x2 * (y0 - y1) + x0 * (y1 - y2) + x1 * (y2 - y0)) ** 2
    if not np.isfinite(m) or m >= 1e6 or not a2 >= 1e-4 * l[1] * l[2]:
        return 0, S - 1, 0, S - 1
    marg = 4 + 1e-3 * (1 + m) * S
    p = 0.5 * (q * S + S - 1)
    c0 = max(int(np.floor(p[:, 0].min() - marg)), 0)
    c1 = min(int(np.ceil(p[:, 0].max() + marg)), S - 1)
    r0 = max(int(np.floor(p[:, 1].min() - marg)), 0)
    r1 = min(int(np.ceil(p[:, 1].max() + marg)), S - 1)
    return c0, c1, r0, r1


def zbuffer(vertices, faces, image_size, anti_aliasing=True, fill_back=True, eye_z=-2.732, near=0.1, far=100.0,
            exhaustive=False, window=None):
    """Contract steps 1 and 3.  Returns (face_index [B,S,S] int32, raster depth [B,S,S] f32), raster row order.
    `window` = (c0, c1, r0, r1), inclusive raster columns and rows: only that rectangle is computed and returned
    ([B, r1-r0+1, c1-c0+1]), for rasters too large to walk whole."""
    S = image_size * (2 if anti_aliasing else 1)
    wc0, wc1, wr0, wr1 = (0, S - 1, 0, S - 1) if window is None else window
    assert 0 <= wc0 <= wc1 < S and 0 <= wr0 <= wr1 < S, window
    fv = face_copies(vertices, faces, fill_back)
    xy, z, inv = _records(fv, S, eye_z)
    B, Fc = fv.shape[:2]
    cp = pixel_coords(S)
    idx = np.arange(S, dtype=f32)
    near, far = f32(near), f32(far)
    fidx = np.full((B, wr1 - wr0 + 1, wc1 - wc0 + 1), -1, np.int32)
    depth = np.full((B, wr1 - wr0 + 1, wc1 - wc0 + 1), far, f32)
    with np.errstate(all="ignore"):
        for b in range(B):
            for f in range(Fc):
                (x0, y0), (x1, y1), (x2, y2) = xy[b, f]
                if (y2 - y0) * (x1 - x0) < (y1 - y0) * (x2 - x0):  # back-facing
                    continue
                c0, c1, r0, r1 = _region(xy[b, f], S, exhaustive)
                c0, c1, r0, r1 = max(c0, wc0), min(c1, wc1), max(r0, wr0), min(r1, wr1)
                if c0 > c1 or r0 > r1:
                    continue
                xp, yp = cp[None, c0:c1 + 1], cp[r0:r1 + 1, None]
                out = (((yp - y0) * (x1 - x0) < (xp - x0) * (y1 - y0)) | ((yp - y1) * (x2 - x1) < (xp - x1) * (y2 - y1))
                       | ((yp - y2) * (x0 - x2) < (xp - x2) * (y0 - y2)))
                if out.all():
                    continue
                _, zp = bary(inv[b, f], z[b, f], idx[None, c0:c1 + 1], idx[r0:r1 + 1, None])
                cur = depth[b, r0 - wr0:r1 - wr0 + 1, c0 - wc0:c1 - wc0 + 1]
                win = ~out & (zp > near) & (zp < far) & (zp < cur)
                cur[win] = zp[win]
                fidx[b, r0 - wr0:r1 - wr0 + 1, c0 - wc0:c1 - wc0 + 1][win] = f
    return fidx, depth


def _samples(fidx, vertices, faces, T, fill_back, eye_z, S):
    """Per covered raster pixel: (batch, pixel coords, face, is_back, 8 texel indices into the ORIGINAL cube,
    8 weights) -- contract step 4."""
    fv = face_copies(vertices, faces, fill_back)
    _, z, inv = _records(fv, S, eye_z)
    F = np.asarray(faces).shape[1]
    b, yi, xi = np.nonzero(fidx >= 0)
    fc = fidx[b, yi, xi].astype(np.int64)
    w, zp = bary(inv[b, fc], z[b, fc], xi.astype(f32), yi.astype(f32))
    tm1, lim = f32(T - 1), f32(T - 1) - f32(1e-3)
    with np.errstate(all="ignore"):
        tif = [np.fmin(np.fmax((w[k] * tm1) * (zp / z[b, fc, k]), f32(0)), lim) for k in range(3)]
    ti = [t.astype(np.int64) for t in tif]
    back = fc >= F
    texel, weight = [], []
    for pn in range(8):
        wt = np.ones_like(zp)
        ii = []
        for k in range(3):
            frac = tif[k] - ti[k].astype(f32)
            if (pn >> k) & 1 == 0:
                wt = wt * (f32(1) - frac)
                ii.append(ti[k])
            else:
                wt = wt * frac
                ii.append(ti[k] + 1)
        texel.append(np.where(back, (ii[2] * T + ii[1]) * T + ii[0], (ii[0] * T + ii[1]) * T + ii[2]))
        weight.append(wt)
    return b, yi, xi, np.where(back, fc - F, fc), fc, np.stack(texel, 1), np.stack(weight, 1)


def flip_pool(planes, anti_aliasing):
    """[B,C,S,S] raster planes -> flipped vertically, then 2x2 average-pooled (row-major window sum, / 4)."""
    p = planes[:, :, ::-1, :]
    if not anti_aliasing:
        return np.ascontiguousarray(p)
    s = ((p[:, :, 0::2, 0::2] + p[:, :, 0::2, 1::2]) + p[:, :, 1::2, 0::2]) + p[:, :, 1::2, 1::2]
    return (s / p.dtype.type(4)).astype(p.dtype)


def render(vertices, faces, textures=None, image_size=256, anti_aliasing=True, fill_back=True, eye_z=-2.732,
           near=0.1, far=100.0, light_intensity_ambient=0.5, light_intensity_directional=0.5,
           light_color_ambient=(1, 1, 1), light_color_directional=(1, 1, 1), light_direction=(0, 1, 0),
           background_color=(0, 0, 0), shared_textures=1, zbuf=None, exhaustive=False):
    """The whole contract.  Returns a dict: face_index / raster_depth [B,S,S], alpha / depth [B,is,is] and, with
    textures, rgb [B,3,is,is].  `zbuf` = a (face_index, raster_depth) pair from zbuffer() to reuse."""
    S = image_size * (2 if anti_aliasing else 1)
    if zbuf is None:
        zbuf = zbuffer(vertices, faces, image_size, anti_aliasing, fill_back, eye_z, near, far, exhaustive)
    fidx, rdepth = zbuf
    out = {"face_index": fidx, "raster_depth": rdepth,
           "alpha": flip_pool((fidx >= 0).astype(f32)[:, None], anti_aliasing)[:, 0],
           "depth": flip_pool(rdepth[:, None], anti_aliasing)[:, 0]}
    if textures is None:
        return out
    textures = np.asarray(textures, f32)
    B, T = fidx.shape[0], textures.shape[2]
    light = lights(face_copies(vertices, faces, fill_back), light_intensity_ambient, light_intensity_directional,
                   light_color_ambient, light_color_directional, light_direction)
    rgb = np.empty((B, 3, S, S), f32)
    rgb[:] = np.asarray(background_color, f32)[None, :, None, None]
    b, yi, xi, f, fc, texel, weight = _samples(fidx, vertices, faces, T, fill_back, eye_z, S)
    tex = textures.reshape(textures.shape[0], textures.shape[1], T ** 3, 3)[b // shared_textures, f]  # [N, T^3, 3]
    lit = light[b, fc]
    for c in range(3):
        s = np.zeros(len(b), f32)
        for pn in range(8):
            s = s + weight[:, pn] * (tex[np.arange(len(b)), texel[:, pn], c] * lit[:, c])
        rgb[b, c, yi, xi] = s
    out["rgb"] = flip_pool(rgb, anti_aliasing)
    return out


def _raster_grad(grad_rgb, S, anti_aliasing):
    """Adjoint of flip_pool: [B,3,is,is] -> [B,3,S,S] float64."""
    g = np.asarray(grad_rgb, np.float64)
    if anti_aliasing:
        g = np.repeat(np.repeat(g, 2, axis=2), 2, axis=3) / 4.0
    return g[:, :, ::-1, :]


def render_rgb_linear(textures, vertices, faces, image_size, zbuf, anti_aliasing=True, fill_back=True, eye_z=-2.732,
                      shared_textures=1, **light):
    """The texture-dependent part of rgb (no background) in float64 with the contract's float32 weights and light:
    the linear map whose adjoint is grad_textures()."""
    fidx = zbuf[0]
    S = fidx.shape[1]
    T = textures.shape[2]
    lit = lights(face_copies(vertices, faces, fill_back), **light).astype(np.float64)
    b, yi, xi, f, fc, texel, weight = _samples(fidx, vertices, faces, T, fill_back, eye_z, S)
    tex = np.asarray(textures, np.float64).reshape(textures.shape[0], textures.shape[1], T ** 3, 3)
    rgb = np.zeros((fidx.shape[0], 3, S, S))
    for pn in range(8):
        vals = tex[b // shared_textures, f, texel[:, pn]] * lit[b, fc] * weight[:, pn, None].astype(np.float64)
        rgb[b, :, yi, xi] += vals
    p = rgb[:, :, ::-1, :]
    if anti_aliasing:
        p = (((p[:, :, 0::2, 0::2] + p[:, :, 0::2, 1::2]) + p[:, :, 1::2, 0::2]) + p[:, :, 1::2, 1::2]) / 4.0
    return p


def grad_textures(grad_rgb, vertices, faces, texture_shape, zbuf, anti_aliasing=True, fill_back=True, eye_z=-2.732,
                  shared_textures=1, magnitude=False, counts=False, **light):
    """Contract step 6 in float64: light * w_pn * grad_rgb at the 8 texels of every covered raster pixel, back copies
    on the transposed texel, through the adjoint of the flip and the pool.  Returns texture_shape [B/G,F,T,T,T,3].
    `magnitude` also returns the sum of the terms' absolute values per element, `counts` the number of terms that
    land on each texel ([B/G,F,T,T,T]): what a float32 summation in any order needs for its error bound."""
    fidx = zbuf[0]
    S = fidx.shape[1]
    T = texture_shape[2]
    lit = lights(face_copies(vertices, faces, fill_back), **light).astype(np.float64)
    b, yi, xi, f, fc, texel, weight = _samples(fidx, vertices, faces, T, fill_back, eye_z, S)
    g = _raster_grad(grad_rgb, S, anti_aliasing)[b, :, yi, xi]  # [N,3]
    out = np.zeros((texture_shape[0], texture_shape[1], T ** 3, 3))
    mag = np.zeros_like(out)
    cnt = np.zeros(out.shape[:3], np.int64)
    for pn in range(8):
        at = (b // shared_textures, f, texel[:, pn])
        term = lit[b, fc] * weight[:, pn, None].astype(np.float64) * g
        np.add.at(out, at, term)
        np.add.at(mag, at, np.abs(term))
        np.add.at(cnt, at, 1)
    res = (out.reshape(texture_shape),)
    if magnitude:
        res += (mag.reshape(texture_shape),)
    if counts:
        res += (cnt.reshape(tuple(texture_shape[:-1])),)
    return res if len(res) > 1 else res[0]
