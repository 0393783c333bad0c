"""Edge-case scenes for the NMR renderer (csrc/nmr.cu, oracle/nmr.py) and per-pixel counts that show each scene's
feature occurs: depth ties, near / far clipping, faces that take the z-buffer's whole-image path.  Shared by
tests/test_nmr_range_cpu.py (the oracle against its exhaustive walk) and tests/test_nmr_range_gpu.py (the kernels
against the oracle).  Vertices are the renderer's input [B,V,3] float32 (NDC x, y; z before look_at), faces [B,F,3]
int32."""
import numpy as np

import nmr as oracle
from umr_b200 import synth

f32 = np.float32
EYE = -2.732


def centre(i, S):
    """NDC x (or y) of raster pixel column (row) i: exactly the oracle's pixel centre."""
    return float(oracle.pixel_coords(S)[i])


def mesh(B=1, subdiv=1, seed=0, soup=4, scale=0.8):
    """A closed, lumpy sphere around z = 5 plus `soup` open triangles of both orientations in front of it."""
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(subdiv)
    verts = synth.bird_like(v, rng, B).astype(np.float64) * scale
    verts[..., 2] += 5.0
    verts[..., 1] *= -1
    faces = np.repeat(f[None], B, 0)
    if soup:
        sv = rng.uniform(-0.9, 0.9, size=(B, 3 * soup, 3))
        sv[..., 2] = rng.uniform(3.5, 4.5, size=(B, 3 * soup))
        verts = np.concatenate([verts, sv], 1)
        faces = np.concatenate([faces, (v.shape[0] + np.arange(3 * soup).reshape(soup, 3))[None].repeat(B, 0)], 1)
    return verts.astype(f32), faces.astype(np.int32)


def append(verts, faces, extra_v, extra_f):
    """Scene + extra vertices [V',3] and faces [F',3] (indices into extra_v), the same in every batch item."""
    B, V = verts.shape[:2]
    ev = np.repeat(np.asarray(extra_v, f32)[None], B, 0)
    ef = np.repeat((np.asarray(extra_f, np.int64) + V)[None], B, 0)
    return np.concatenate([verts, ev], 1), np.concatenate([faces, ef.astype(np.int32)], 1)


def grid(S, n=6, step=4, z=5.0):
    """A flat n x n grid of quads (two CCW triangles each) at constant z with every vertex on a pixel centre, so each
    shared edge runs through pixel centres that both of its faces admit."""
    i0 = (S - n * step) // 2
    xs = [centre(i0 + k * step, S) for k in range(n + 1)]
    v = np.array([[x, y, z] for y in xs for x in xs], f32)
    f = []
    for r in range(n):
        for c in range(n):
            a, b, d, e = r * (n + 1) + c, r * (n + 1) + c + 1, (r + 1) * (n + 1) + c, (r + 1) * (n + 1) + c + 1
            if (r + c) % 2:
                f += [[a, b, e], [a, e, d]]
            else:
                f += [[a, b, d], [b, e, d]]
    return v[None], np.array(f, np.int32)[None]


def duplicates(verts, faces, k=12):
    """The first k faces appended again as they are, then again with their vertex order rotated."""
    f0 = faces[:, :k]
    return verts, np.concatenate([faces, f0, np.roll(f0, 1, axis=2)], 1).astype(np.int32)


def zero_area(S):
    """Degenerate faces: collinear vertices on pixel centres (a diagonal, a row, a column), two equal vertices, one
    point, and slivers whose orientation test rounds to zero -- both copies of each face pass the back-face test."""
    c = lambda i: centre(i, S)  # noqa: E731
    v, f = [], []

    def tri(p, q, r):
        f.append([len(v), len(v) + 1, len(v) + 2])
        v.extend([p, q, r])
    tri((c(2), c(2), 5.0), (c(S // 2), c(S // 2), 5.2), (c(S - 3), c(S - 3), 5.4))
    tri((c(1), c(S // 3), 5.0), (c(S // 2), c(S // 3), 4.8), (c(S - 2), c(S // 3), 4.6))
    tri((c(S // 3), c(1), 5.0), (c(S // 3), c(S - 2), 5.1), (c(S // 3), c(S // 2), 5.3))
    tri((c(3), c(S - 4), 5.0), (c(3), c(S - 4), 5.0), (c(S - 4), c(3), 5.0))
    tri((c(S // 2), c(S // 2), 4.0), (c(S // 2), c(S // 2), 4.0), (c(S // 2), c(S // 2), 4.0))
    rng = np.random.default_rng(11)
    n = 0
    while n < 6:  # a sliver: a third vertex one float32 ulp off the line of the other two
        p = rng.uniform(-0.9, 0.9, 2).astype(f32)
        q = rng.uniform(-0.9, 0.9, 2).astype(f32)
        t = f32(rng.uniform(0.2, 0.8))
        r = (p + t * (q - p)).astype(f32)
        r[1] = np.nextafter(r[1], f32(np.inf))
        (x0, y0), (x1, y1), (x2, y2) = p, q, r
        if (y2 - y0) * (x1 - x0) == (y1 - y0) * (x2 - x0):
            tri((x0, y0, 4.5), (x1, y1, 4.7), (x2, y2, 4.9))
            n += 1
    return np.array(v, f32)[None], np.array(f, np.int32)[None]


def thin(S, seed=0, eps=0.02):
    """Long thin faces whose smallest angle has a sine of (1 +- eps) * 1e-2, either side of the z-buffer's pixel-box
    threshold, at 8 orientations; fat faces reaching off-screen to |coord| just under 1e6 and at 1e6; and faces with
    every vertex on a pixel centre.  Depth varies over each face."""
    rng = np.random.default_rng(seed)
    v, f = [], []

    def tri(p, q, r):
        f.append([len(v), len(v) + 1, len(v) + 2])
        v.extend([p, q, r])
    for k in range(8):
        phi = 2 * np.pi * k / 8 + 0.1
        for s in (1 + eps, 1 - eps):
            th = np.arcsin(1e-2 * s)
            a = rng.uniform(-0.7, 0.7, 2)
            L = rng.uniform(0.8, 1.6)
            z = rng.uniform(4.0, 6.0, 3)
            tri((a[0], a[1], z[0]), (a[0] + L * np.cos(phi), a[1] + L * np.sin(phi), z[1]),
                (a[0] + L * np.cos(phi + th), a[1] + L * np.sin(phi + th), z[2]))
    M = float(np.nextafter(f32(1e6), f32(0)))
    tri((-0.3, -0.4, 6.5), (M, -0.5 * M, 6.6), (0.3 * M, M, 6.4))
    tri((-M, -M, 7.0), (M, -M, 7.2), (0.0, M, 6.8))
    tri((0.5, 0.2, 6.0), (1e6, 0.3, 6.1), (0.6, 1e6, 6.2))
    tri((-0.9, 0.9, 6.3), (-1e6, -1e6, 6.4), (0.1, -0.2, 6.5))
    c = lambda i: centre(i, S)  # noqa: E731
    # wedges with the sharp vertex on screen, one edge along a pixel row (column) and the far vertices at 1e4 / 1e5:
    # the edge tests admit pixels on that row well past the sharp vertex, which only the box margin's m term covers
    for k, L in enumerate((1e4, 1e5, 1e4, 1e5)):
        a = (c(S // 4 + 3 * k), c(S // 3 + 5 * k))
        sg = 1 if k % 2 else -1
        t = L * np.cos(np.arcsin(1e-2 * (1 + eps)))
        h = L * 1e-2 * (1 + eps)
        if k < 2:   # along a row, opening towards +x or -x (CCW either way)
            tri((a[0], a[1], 3.0), (a[0] + sg * L, a[1], 3.1), (a[0] + sg * t, a[1] + sg * h, 3.2))
        else:       # along a column
            tri((a[0], a[1], 3.0), (a[0] - sg * h, a[1] + sg * t, 3.2), (a[0], a[1] + sg * L, 3.1))
    tri((c(S // 8), c(S // 8), 5.5), (c(S // 2), c(S // 8 + 1), 5.0), (c(S // 4), c(S // 2 + 3), 5.9))
    tri((c(S // 2), c(S // 8 + 1), 5.0), (c(7 * S // 8), c(3 * S // 4), 5.2), (c(S // 4), c(S // 2 + 3), 5.9))
    return np.array(v, f32)[None], np.array(f, np.int32)[None]


def invalid(B=1, seed=3):
    """mesh() plus faces with indices -1, V and 2^31-1, faces with a repeated vertex index, and faces in front of the
    mesh with a NaN, +inf or -inf in exactly one of x, y, z.  All but the +inf z face are never drawn; that one has a
    vertex at infinite depth and is drawn where the other two weights give a finite depth.  Returns (verts, faces,
    number of clean faces)."""
    verts, faces = mesh(B, subdiv=1, seed=seed, soup=4)
    F0 = faces.shape[1]
    ev, ef = [], []
    for d in range(3):
        for bad in (np.nan, np.inf, -np.inf):
            p = [[-0.6, -0.5, 3.0], [0.7, -0.4, 3.1], [0.1, 0.8, 3.2]]
            p[d % 3][d] = bad
            ef.append([len(ev), len(ev) + 1, len(ev) + 2])
            ev.extend(p)
    verts, faces = append(verts, faces, ev, ef)
    V = verts.shape[1]
    raw =np.array([[-1, 0, 1], [2, V, 3], [4, 5, 2 ** 31 - 1], [6, 6, 7], [8, 9, 8]], np.int64)
    faces = np.concatenate([faces, np.repeat(raw[None], B, 0).astype(np.int32)], 1)
    return verts, faces, F0


def clipped(B=1, seed=5):
    """Faces spanning z from behind the eye (z - eye <= 0) to far away, so near / far planes cut through them."""
    rng = np.random.default_rng(seed)
    v, f = [], []
    for k in range(10):
        a = rng.uniform(-0.8, 0.8, 2)
        za, zb = rng.uniform(-6.0, 2.0), rng.uniform(4.0, 12.0)
        p = [(a[0], a[1], za), (a[0] + 0.9, a[1] + 0.1, zb), (a[0] + 0.2, a[1] + 0.8, 0.5 * (za + zb))]
        f.append([len(v), len(v) + 1, len(v) + 2])
        v.extend(p)
    return np.repeat(np.array(v, f32)[None], B, 0), np.repeat(np.array(f, np.int32)[None], B, 0)


def signed_zero():
    """For eye_z = +0 and a negative near plane: two pairs of equal triangles, one vertex at z = +0 in one and z = -0
    in the other, so depths +0 and -0 meet on most of each pair's pixels.  In the left pair the lower face index has
    +0, in the right pair -0."""
    v, f = [], []
    for x0, zs in ((-0.9, (0.0, -0.0)), (0.1, (-0.0, 0.0))):
        for z2 in zs:
            f.append([len(v), len(v) + 1, len(v) + 2])
            v.extend([(x0, -0.8, 2.0), (x0 + 0.8, -0.7, 3.0), (x0 + 0.3, 0.8, z2)])
    return np.array(v, f32)[None], np.array(f, np.int32)[None]


# ---------------------------------------------------------------------------------------------------------------------
# feature counts
# ---------------------------------------------------------------------------------------------------------------------
def whole_image_copies(verts, faces, fill_back=True):
    """Face copies that k_nmr_prep sends to the whole-image path (front-facing, and thin, non-finite or m >= 1e6),
    by the kernel's float32 expression."""
    fv = oracle.face_copies(verts, faces, fill_back)
    x0, y0, x1, y1, x2, y2 = (fv[..., k, d] for k in range(3) for d in range(2))
    with np.errstate(all="ignore"):
        front = ~((y2 - y0) * (x1 - x0) < (y1 - y0) * (x2 - x0))
        l01 = (x1 - x0) * (x1 - x0) + (y1 - y0) * (y1 - y0)
        l02 = (x2 - x0) * (x2 - x0) + (y2 - y0) * (y2 - y0)
        l12 = (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1)
        lmin = np.fmin(np.fmin(l01, l02), l12)
        prod2 = (l01 * l02 * l12) / np.fmax(lmin, f32(1e-30))
        a2 = x2 * (y0 - y1) + x0 * (y1 - y2) + x1 * (y2 - y0)
        m = np.abs(fv[..., :2]).max(axis=(-1, -2))
        whole = ~(a2 * a2 >= f32(1e-4) * prod2) | ~(m < f32(1e6))
    return int((front & whole).sum()), int((front & ~whole).sum())


def pixel_stats(verts, faces, image_size, anti_aliasing=True, fill_back=True, eye_z=EYE, near=0.1, far=100.0):
    """Every face copy tested on every pixel (small S only).  Returns the number of pixels where two or more copies
    share the smallest admitted depth (`ties`), where an admitted copy's depth is <= near (`near`) or >= far (`far`),
    and where the smallest admitted depth is zero (`zero`)."""
    S = image_size * (2 if anti_aliasing else 1)
    fv = oracle.face_copies(verts, faces, fill_back)
    xy, z, inv = oracle._records(fv, S, eye_z)
    B, Fc = fv.shape[:2]
    cp, idx = oracle.pixel_coords(S), np.arange(S, dtype=f32)
    near, far = f32(near), f32(far)
    zmin = np.full((B, S, S), np.inf, f32)
    nmin = np.zeros((B, S, S), np.int64)
    ncut, fcut = np.zeros((B, S, S), bool), np.zeros((B, S, S), bool)
    xp, yp = cp[None, :], cp[:, None]
    with np.errstate(all="ignore"):
        for b in range(B):
            for f in range(Fc):
                (x0, y0), (x1, y1), (x2, y2) = xy[b, f]
                if (y2 - y0) * (x1 - x0) < (y1 - y0) * (x2 - x0):
                    continue
                out = (((yp - y0) * (x1 - x0) < (xp - x0) * (y1 - y0)) | ((yp - y1) * (x2 - x1) < (xp - x1) * (y2 - y1))
                       | ((yp - y2) * (x0 - x2) < (xp - x2) * (y0 - y2)))
                _, zp = oracle.bary(inv[b, f], z[b, f], idx[None, :], idx[:, None])
                adm = ~out & ~np.isnan(zp)
                ncut[b] |= adm & (zp <= near)
                fcut[b] |= adm & (zp >= far)
                ok = adm & (zp > near) & (zp < far)
                lt, eq = ok & (zp < zmin[b]), ok & (zp == zmin[b])
                nmin[b][eq] += 1
                nmin[b][lt] = 1
                zmin[b][lt] = zp[lt]
    return dict(ties=int((nmin >= 2).sum()), near=int(ncut.sum()), far=int(fcut.sum()), zero=int((zmin == 0).sum()))
