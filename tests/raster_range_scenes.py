"""Seeded scenes for the range tests of the two bitwise-reproducible soft rasterisers (float64 and deterministic float32),
and host restatements of the kernels' cull-box and tile arithmetic, so that each scene's claimed property can be checked
without a GPU (test_raster_gather_range_cpu.py) and counted where it runs (test_raster_gather_range_gpu.py).

Box arithmetic (k_prep_f64 / k_prep, DESIGN.md §3):
  float64  r = sqrt(double(float(dist_eps_log) * float(sigma))), box = min - r and max + r in double, pixel centre
           (2i + 1 - S) / S in double;
  float32  the same in float32 (one IEEE operation each; the raster code is built with -fmad=false).
The forward lists a face for a 16x16 tile when its box meets the tile's pixel-centre extents; k_raster_fwd_f64 tests
faces in windows of WINDOW = 1024 and consumes its 2048-entry list before the last window only when more than 1024
listed faces are waiting.

The default float32 path (raster_stream.cuh, raster_fwd3.cuh, raster_fwd4.cuh, test_raster_fast_range_gpu.py): k_bin_coarse
lists, per 64x64-pixel coarse bin (CB), the faces whose box meets the bin's pixel-centre extents, in ascending order;
k_raster_fwd3 walks its bin's list in windows of LCAP = 512 entries, keeps the entries whose box meets its 16x16 tile (one
tile-list segment per window) and reserves, per segment with a pair, popc(meet) pair blocks per listed face plus 2 header
words, where meet holds the 8x4-pixel warp blocks whose columns and rows the box reaches (fwd3_blocks restates it).  A
block holds the survivors of one face in one warp block: at most 32 records.  k_raster_fwd4 holds FWD4_CAP = 1536
tile-list entries; a longer coarse list takes its windowed path.  The recompute fallback lists faces in windows of
FACE_WINDOW = 65536."""
import math

import numpy as np

TILE, WINDOW, LIST_CAP = 16, 1024, 2048
CB, LCAP, FWD4_CAP, FACE_WINDOW = 64, 512, 1536, 65536
# soft edges of the range scenes: r = 0.0096 (about a third of a pixel at S = 66)
KW = dict(sigma_val=1e-5, dist_eps=1e-4, gamma_val=1e-3)


def kernel_grid(S, dtype=np.float64):
    """The p2f grid of the kernels: torch's float32 linspace(-1, 1, S) by its per-element definition (start + step * i in the
    lower half, end - step * (S - 1 - i) in the upper), widened.  torch's vectorised CPU linspace, which
    softras.standard_grid calls, rounds some elements one float ulp away from it, so the oracle is handed this grid.
    S = 1 is torch 1.1's linspace(-1, 1, 1) = [-1], a step of 0."""
    step = np.float32(2.0) / np.float32(S - 1) if S > 1 else np.float32(0.0)
    i = np.arange(S)
    lo = (np.float32(-1.0) + step * i.astype(np.float32)).astype(np.float32)
    hi = (np.float32(1.0) - step * (S - 1 - i).astype(np.float32)).astype(np.float32)
    x = np.where(i * 2 < S, lo, hi)
    return np.ascontiguousarray(np.stack(np.broadcast_arrays(x[None, :], x[:, None]), axis=-1).astype(dtype))


# ---------------------------------------------------------------------------------------------------------------------
# restated arithmetic
# ---------------------------------------------------------------------------------------------------------------------
def cull_radius(dtype, sigma_val=KW["sigma_val"], dist_eps=KW["dist_eps"]):
    thr = np.float32(math.log(1.0 / dist_eps - 1.0)) * np.float32(sigma_val)   # float * float, as kernel.cu:333
    return np.float64(math.sqrt(float(thr))) if dtype == np.float64 else np.sqrt(np.float32(thr))


def pixel_centre(i, S, dtype):
    i = np.asarray(i)
    if dtype == np.float64:
        return (2.0 * i + 1.0 - S) / S
    return (np.asarray(2 * i + 1 - S).astype(np.float32) / np.float32(S)).astype(np.float32)


def boxes(fv, dtype, r=None):
    """[..., 4] = xlo, xhi, ylo, yhi of every face, as k_prep(_f64) stores them: fmin / fmax drop a NaN coordinate, so a
    face with a NaN vertex has the box of its finite coordinates (NaN only where all three are)."""
    fv = np.asarray(fv, dtype)
    r = cull_radius(dtype) if r is None else r
    x, y = fv[..., 0::3], fv[..., 1::3]
    with np.errstate(invalid="ignore"):
        return np.stack([np.fmin.reduce(x, -1) - r, np.fmax.reduce(x, -1) + r, np.fmin.reduce(y, -1) - r,
                         np.fmax.reduce(y, -1) + r], -1).astype(dtype)


def tile_hits(box, S, tx, ty, dtype, side=TILE):
    """Faces whose box meets tile (tx, ty) of `side` pixels (ty counts image rows from the top), as the forward's tile
    test (and, for side = CB, the coarse binning) decides."""
    x0, x1 = pixel_centre(tx * side, S, dtype), pixel_centre(min(tx * side + side - 1, S - 1), S, dtype)
    top, bot = pixel_centre(S - 1 - ty * side, S, dtype), pixel_centre(S - 1 - min(ty * side + side - 1, S - 1), S, dtype)
    return ~((x0 > box[..., 1]) | (x1 < box[..., 0]) | (bot > box[..., 3]) | (top < box[..., 2]))


def window_hits(box, S, dtype, tx=0, ty=0):
    """Listed faces per 1024-face window of one image, tile (tx, ty)."""
    h = tile_hits(box, S, tx, ty, dtype)
    return [int(h[w:w + WINDOW].sum()) for w in range(0, h.shape[0], WINDOW)]


def consumes(counts):
    """The list lengths at which k_raster_fwd_f64 consumes its tile list, for these per-window hit counts."""
    out, n = [], 0
    for w, c in enumerate(counts):
        n += c
        if n <= LIST_CAP - WINDOW and w + 1 < len(counts):
            continue
        out.append(n)
        n = 0
    return out


def fwd3_segments(box, S, tx=0, ty=0, dtype=np.float32):
    """k_raster_fwd3's tile-list segments of 16x16 tile (tx, ty): per LCAP window of its coarse bin's list, (listed
    faces, pair blocks).  A face's blocks are popc(cm) * popc(rm): the 8-column halves and 4-row bands of the tile
    holding a live pixel centre inside the face's box."""
    cl = np.flatnonzero(tile_hits(box, S, tx * TILE // CB, ty * TILE // CB, dtype, CB))
    ncol, nrow = min(TILE, S - tx * TILE), min(TILE, S - ty * TILE)
    xs = pixel_centre(tx * TILE + np.arange(ncol), S, dtype)
    ys = pixel_centre(S - 1 - (ty * TILE + np.arange(nrow)), S, dtype)
    out = []
    for w0 in range(0, len(cl), LCAP):
        f = cl[w0:w0 + LCAP]
        b = box[f[tile_hits(box[f], S, tx, ty, dtype)]]
        with np.errstate(invalid="ignore"):
            col = ~((xs[None] > b[:, 1:2]) | (xs[None] < b[:, 0:1]))
            row = ~((ys[None] > b[:, 3:4]) | (ys[None] < b[:, 2:3]))
        nc = col[:, :8].any(1).astype(int) + col[:, 8:].any(1)
        nr = sum(row[:, 4 * k:4 * k + 4].any(1).astype(int) for k in range(4))
        out.append((len(b), int((nc * nr).sum())))
    return out


def fwd3_blocks_wanted(fv, S, dtype=np.float32):
    """The pair buffer's block cursor after a k_raster_fwd3 forward with room for every tile: per segment holding a
    block, its blocks plus 2 header words."""
    nt = (S + TILE - 1) // TILE
    total = 0
    for img in np.asarray(fv, dtype):
        box = boxes(img, dtype)
        for ty in range(nt):
            for tx in range(nt):
                total += sum(nb + 2 for _, nb in fwd3_segments(box, S, tx, ty, dtype) if nb > 0)
    return total


def survivors(fv, S, near=1.0, far=100.0, sigma_val=KW["sigma_val"], dist_eps=KW["dist_eps"]):
    """[F, S, S] (image rows from the top): the (face, pixel) pairs the euclidean-distance forward keeps -- inside the
    box, inside the triangle or nearer its edges than sqrt(thr), depth in (near, far) -- evaluated in double, with a
    check that no pixel lies within 1e-6 (relative) of a decision."""
    thr = float(np.float32(math.log(1.0 / dist_eps - 1.0)) * np.float32(sigma_val))
    c = pixel_centre(np.arange(S), S, np.float64)
    xp, yp = np.meshgrid(c, c[::-1])
    out = []
    for f in np.asarray(fv, np.float64):
        v = f.reshape(3, 3)
        box = boxes(f[None], np.float32)[0].astype(np.float64)
        inbox = (xp >= box[0]) & (xp <= box[1]) & (yp >= box[2]) & (yp <= box[3])
        d2 = np.full(xp.shape, np.inf)
        for a, b in ((0, 1), (1, 2), (2, 0)):
            e = v[b, :2] - v[a, :2]
            t = np.clip(((xp - v[a, 0]) * e[0] + (yp - v[a, 1]) * e[1]) / (e @ e), 0, 1)
            d2 = np.minimum(d2, (xp - v[a, 0] - t * e[0]) ** 2 + (yp - v[a, 1] - t * e[1]) ** 2)
        det = (v[1, 0] - v[0, 0]) * (v[2, 1] - v[0, 1]) - (v[2, 0] - v[0, 0]) * (v[1, 1] - v[0, 1])
        side = [((v[b, 0] - v[a, 0]) * (yp - v[a, 1]) - (v[b, 1] - v[a, 1]) * (xp - v[a, 0])) * np.sign(det)
                for a, b in ((0, 1), (1, 2), (2, 0))]
        inside = np.minimum(np.minimum(side[0], side[1]), side[2]) >= 0
        assert not (inbox & ~inside & (np.abs(d2 - thr) < 1e-6 * thr)).any(), "a pixel on the distance cut-off"
        z = v[:, 2]
        assert near < z.min() and z.max() < far, "the depth test would decide pairs"
        out.append(inbox & (inside | (d2 < thr)))
    return np.array(out)


def tile_records(fv, S, side=TILE):
    """Saved records per tile of `side` pixels for one image's faces (survivors summed over faces and tile pixels)."""
    s = survivors(fv, S).sum(0)
    nt = (S + side - 1) // side
    return np.array([[int(s[ty * side:(ty + 1) * side, tx * side:(tx + 1) * side].sum()) for tx in range(nt)] for ty in range(nt)])


def texel_index(c0, c1, R):
    """texel_index of the kernels on already clipped barycentrics (float64 arrays)."""
    wx, wy = (c0 * R).astype(np.int64), (c1 * R).astype(np.int64)
    return np.where((c0 + c1) * R - wx - wy <= 1, wy * R + wx, (R - 1 - wy) * R + (R - 1 - wx))


def texels_per_segment(fv, S, T2):
    """For one face [9] covering the raster, (lanes, distinct texels) of every 32-lane row segment of the backward's
    walk, evaluated in double at pixel centres."""
    R = int(math.isqrt(T2))
    x0, y0, _, x1, y1, _, x2, y2, _ = np.asarray(fv, np.float64)
    c = pixel_centre(np.arange(S), S, np.float64)
    xp, yp = np.meshgrid(c, c[::-1])
    det = x2 * (y0 - y1) + x0 * (y1 - y2) + x1 * (y2 - y0)
    w0 = ((y1 - y2) * xp + (x2 - x1) * yp + (x1 * y2 - x2 * y1)) / det
    w1 = ((y2 - y0) * xp + (x0 - x2) * yp + (x2 * y0 - x0 * y2)) / det
    w2 = 1 - w0 - w1
    k = [np.clip(w, 1e-5, 1 - 1e-5) for w in (w0, w1, w2)]
    s = k[0] + k[1] + k[2]
    t = texel_index(k[0] / s, k[1] / s, R)
    return [(len(t[row, x:x + 32]), len(np.unique(t[row, x:x + 32]))) for row in range(S) for x in range(0, S, 32)]


# ---------------------------------------------------------------------------------------------------------------------
# scenes: face_vertices [B, F, 9], textures [B, F, T2, 3] in `dtype`
# ---------------------------------------------------------------------------------------------------------------------
OFF = np.array([5.0, 5.0, 2.0, 5.5, 5.0, 2.0, 5.0, 5.5, 2.0])   # far right of the raster: listed in no tile


def crowd(counts, S, dtype=np.float64, seed=0, T2=4):
    """len(counts) windows of 1024 faces (the last one may be short); window w has counts[w] faces on tile (0, 0) at random
    positions in the window, the others off screen.  Each listed face contains one pixel centre of the tile and reaches
    less than half a pixel from it; every fifth listed face repeats an earlier listed face exactly, so the hard z-test
    breaks depth ties by face order across windows and consumes."""
    rng = np.random.default_rng(seed)
    F = WINDOW * (len(counts) - 1) + max(counts[-1], 1)
    fv = np.tile(OFF, (F, 1)) + rng.uniform(0, 0.2, size=(F, 9)) * np.array([1, 1, 0] * 3)
    hit = []
    for w, c in enumerate(counts):
        n = min(WINDOW, F - w * WINDOW)
        hit += sorted((w * WINDOW + rng.choice(n, size=c, replace=False)).tolist())
    px = 2.0 / S
    m = min(TILE, S)
    for j, f in enumerate(hit):
        if j >= 5 and j % 5 == 0:
            fv[f] = fv[hit[rng.integers(0, j)]]
            continue
        ci, cj = rng.integers(0, m, size=2)
        cx, cy = pixel_centre(ci, S, np.float64), pixel_centre(S - 1 - cj, S, np.float64)
        a, b, c_, d = rng.uniform(0.05, 0.4, size=4) * px
        z = rng.choice([2.0, 2.5, 3.0])
        fv[f] = [cx - a, cy - b, z, cx + c_, cy - b, z, cx, cy + d, z]
    fv = fv[None].astype(dtype)
    tex = rng.uniform(0, 1, size=(1, F, T2, 3)).astype(dtype)
    return fv, tex, np.array(hit)


CROWDS = {"1024+1": [1024, 1], "1+1024+1": [1, 1024, 1], "1024+1024+5": [1024, 1024, 5], "1000+30+1000": [1000, 30, 1000]}


def crowd_all(S, dtype=np.float64, seed=0, F=65535):
    """F faces, every one on tile (0, 0): for F = 65535, 64 consumes of 2048 faces (the last of 2047)."""
    fv, tex, _ = crowd([WINDOW] * (F // WINDOW) + [F % WINDOW], S, dtype, seed, T2=1)
    return fv, tex


# tile-list lengths on one tile for the default path: either side of the LCAP segment and of k_raster_fwd4's FWD4_CAP
# list, and every face of a narrow mesh
LIST_LENGTHS = [LCAP - 1, LCAP, LCAP + 1, FWD4_CAP - 1, FWD4_CAP, FWD4_CAP + 1, 65535]


def edge_targets(S, fast=False):
    """Pixel indices where the edge scene puts box edges: raster ends and the 15 | 16 tile boundary; fast adds the
    31 | 32 boundary of k_raster_fwd4's tiles and the 63 | 64 boundary of the coarse bins."""
    return sorted({i for i in (0, 15, 16, S - 1) + ((31, 32, CB - 1, CB) if fast else ()) if 0 <= i < S})


def edge_vertices(c, r, side, dtype):
    """Vertex coordinates whose box edge (min - r for side -1, max + r for side +1, monotone in the vertex) is pixel centre c
    and the nearest values the edge can take either side of it: one ulp of c, or one step of the vertex where that is
    coarser.  Where no vertex puts the edge exactly on c (its value lies between two steps), only the two neighbours."""
    c = dtype(c)
    up = lambda v: np.nextafter(v, dtype(np.inf)).astype(dtype)     # noqa: E731
    dn = lambda v: np.nextafter(v, dtype(-np.inf)).astype(dtype)    # noqa: E731
    e = lambda v: dtype(v + side * r)                               # noqa: E731
    v = dtype(c - side * r)
    while e(v) > c:
        v = dn(v)
    while e(up(v)) <= c:
        v = up(v)
    if e(v) != c:
        return [v, up(v)]
    below = v
    while e(below) == c:
        below = dn(below)
    return [below, v, up(v)]


EDGE_DEPTH = 1.5


def edges(S, dtype=np.float64, seed=0, T2=4, fast=False):
    """Faces whose cull-box edge lies on a pixel centre, or at the nearest value either side of it (edge_vertices), for
    each of the four box sides at every edge_targets(S, fast) index.  Each face has an edge 3 pixels long on its box side,
    centred on a row (column) in the middle of the raster, and its third vertex EDGE_DEPTH = 1.5 away from that edge into
    the raster.  A pixel centre a box radius r outside the edge then has barycentric r / 1.5 against the third vertex,
    well inside the barycentric distance cut-off r^2 (edge_pixels_alive): the box tests alone decide it.  Returns fv,
    tex and [F, 3] (side 0..3, target index, edge below / on / above the centre: -1 / 0 / +1)."""
    rng = np.random.default_rng(seed)
    r = cull_radius(dtype)
    px = 2.0 / S
    mid = pixel_centre(S // 2, S, np.float64)
    faces, meta = [], []
    for side in range(4):   # xlo, xhi, ylo, yhi
        sign = -1 if side % 2 == 0 else 1
        for i in edge_targets(S, fast):
            c = pixel_centre(i, S, dtype)
            for v in edge_vertices(c, r, sign, dtype):
                d = int(np.sign(dtype(v + sign * r) - c))
                v = float(v)
                inner = v - sign * EDGE_DEPTH
                z = 2.0 + 0.25 * len(faces) % 1.0
                a, b = mid - 1.5 * px, mid + 1.5 * px
                if side < 2:
                    tri = [v, a, z, v, b, z, inner, mid, z]
                else:
                    tri = [a, v, z, b, v, z, mid, inner, z]
                faces.append(tri)
                meta.append((side, i, d))
    fv = np.array(faces, dtype)[None]
    tex = rng.uniform(0, 1, size=(1, fv.shape[1], T2, 3)).astype(dtype)
    return fv, tex, np.array(meta)


COVER = [-5.0, -4.0, 3.0, 6.0, -5.0, 4.0, 0.5, 7.0, 5.0]


def big(dtype=np.float64, seed=0, T2=9, nan=False):
    """A face covering the raster and reaching past it on every side, four faces whose boxes lie entirely off each side,
    one small face in the middle, and, with nan, a face with a NaN vertex (a NaN box)."""
    rng = np.random.default_rng(seed)
    faces = [COVER,
             [-1.6, -0.2, 2.0, -1.1, -0.3, 2.0, -1.3, 0.3, 2.0],    # left
             [1.1, -0.2, 2.0, 1.6, -0.3, 2.0, 1.3, 0.3, 2.0],       # right
             [-0.2, 1.1, 2.0, 0.3, 1.2, 2.0, 0.0, 1.6, 2.0],        # top
             [-0.2, -1.1, 2.0, 0.3, -1.2, 2.0, 0.0, -1.6, 2.0],     # bottom
             [-0.3, -0.25, 2.5, 0.35, -0.2, 3.5, 0.05, 0.4, 2.0]]   # middle
    if nan:
        faces.append([-0.5, -0.5, 3.0, 0.5, np.nan, 3.0, 0.0, 0.5, 3.0])
    fv = np.array(faces, np.float64)[None].astype(dtype)
    tex = rng.uniform(0, 1, size=(1, fv.shape[1], T2, 3)).astype(dtype)
    return fv, tex


def records(S, extra, dtype=np.float32, seed=0, T2=4):
    """The covering face, then `extra` faces of one pixel each in tile (0, 0) (crowd's faces): tile (0, 0) saves
    min(16, S)^2 + extra records (tile_records), for S >= 16 32 x 8 in the covering face's eight full 32-record blocks
    and one more block of one record per extra face."""
    fv, _, hit = crowd([extra], S, np.float64, seed)
    fv = np.concatenate([np.array(COVER, np.float64)[None, None], fv if extra else fv[:, :0]], 1)
    tex = np.random.default_rng(seed).uniform(0, 1, size=(1, fv.shape[1], T2, 3))
    return fv.astype(dtype), tex.astype(dtype)


def window_crossing(dtype=np.float32, seed=0, extra=4):
    """F = FACE_WINDOW + extra faces, on screen only at indices ON = 0, FACE_WINDOW - 1, FACE_WINDOW, F - 1 (returned),
    every other far off it: the recompute fallback's second face window holds the last two."""
    F = FACE_WINDOW + extra
    on = np.array([0, FACE_WINDOW - 1, FACE_WINDOW, F - 1])
    fv = np.tile(OFF, (F, 1))
    fv[on] = [[-0.6 + 0.3 * j, -0.5, 3.0 + j, 0.7, -0.4 + 0.2 * j, 4.0 + j, -0.1 * j, 0.8, 5.0 - j * 0.3] for j in range(len(on))]
    tex = np.full((1, F, 4, 3), 0.5)
    tex[0, on] = np.random.default_rng(seed).uniform(0, 1, size=(len(on), 4, 3))
    return fv[None].astype(dtype), tex.astype(dtype), on


def many_images(B=65535, seed=7, dtype=np.float64):
    """B renders of the covering face and one small face moved sideways per render; textures [B, 2, 1, 3]."""
    rng = np.random.default_rng(seed)
    fv = np.repeat(np.array([[COVER, [-0.6, -0.5, 2.0, 0.7, -0.4, 2.5, -0.1, 0.8, 3.0]]]), B, 0)
    fv[:, 1, [0, 3, 6]] += rng.uniform(-0.8, 0.8, size=(B, 1))
    tex = rng.uniform(0, 1, size=(B, 2, 1, 3))
    return fv.astype(dtype), tex.astype(dtype)


def textured(T2, dtype=np.float64, seed=0):
    """The covering face and a smaller one over the middle with T2 texels per face.  Texels at index R^2 and above
    (R = isqrt(T2)) are never sampled: they hold NaN, so a read of one shows in the images and its gradient must stay 0."""
    rng = np.random.default_rng(seed)
    fv = np.array([COVER, [-0.6, -0.5, 2.0, 0.7, -0.4, 2.5, -0.1, 0.8, 3.0]], np.float64)[None].astype(dtype)
    tex = rng.uniform(0, 1, size=(1, 2, T2, 3))
    R = math.isqrt(T2)
    tex[:, :, R * R:] = np.nan
    return fv, tex.astype(dtype)


def planes(dtype=np.float64, seed=0):
    """For near = 3, far = 6 (returned): faces that both planes cut (corners from z = 1 to 8), and faces of constant
    z = 4 (a power of two, so most covered pixels have depth exactly 4) and z = 6 = far."""
    rng = np.random.default_rng(seed)
    faces = [[-0.9, -0.8, 1.0, 0.8, -0.9, 8.0, 0.0, 0.9, 4.5],
             [-0.7, 0.6, 7.5, 0.9, 0.2, 1.5, -0.2, -0.9, 3.0],
             [-0.95, -0.95, 4.0, 0.1, -0.95, 4.0, -0.95, 0.1, 4.0],
             [0.95, 0.95, 6.0, -0.1, 0.95, 6.0, 0.95, -0.1, 6.0],
             [-0.5, -0.3, 3.0, 0.6, -0.2, 3.0, 0.0, 0.7, 3.0]]
    fv = np.array(faces, np.float64)[None].astype(dtype)
    tex = rng.uniform(0, 1, size=(1, fv.shape[1], 4, 3)).astype(dtype)
    return fv, tex, 3.0, 6.0


def shared(B, G, textype, dtype=np.float64, seed=0):
    """B renders of a few faces in different positions, G texture groups (textures [G, F, T2, 3])."""
    rng = np.random.default_rng(seed)
    F = 6
    base = np.array([COVER] + [[-0.6, -0.5, 2.0, 0.7, -0.4, 2.5, -0.1, 0.8, 3.0]] * (F - 1), np.float64)
    fv = np.repeat(base[None], B, 0)
    fv[:, 1:, [0, 3, 6]] += rng.uniform(-0.4, 0.4, size=(B, F - 1, 1))
    fv[:, 1:, [1, 4, 7]] += rng.uniform(-0.4, 0.4, size=(B, F - 1, 1))
    T2 = 3 if textype == "vertex" else 4
    tex = rng.uniform(0, 1, size=(G, F, T2, 3))
    return fv.astype(dtype), tex.astype(dtype)


def barycentric_alive(fv, xp, yp, sigma_val=KW["sigma_val"], dist_eps=KW["dist_eps"]):
    """Whether the barycentric distance keeps the pair (kernel.cu:156-159, :374-377, evaluated in double): the smallest
    barycentric m gives dis = +-m^2, and the pair is culled when -dis >= thr."""
    thr = float(np.float32(math.log(1.0 / dist_eps - 1.0)) * np.float32(sigma_val))
    x0, y0, _, x1, y1, _, x2, y2, _ = np.asarray(fv, np.float64)
    det = x2 * (y0 - y1) + x0 * (y1 - y2) + x1 * (y2 - y0)
    w0 = ((y1 - y2) * xp + (x2 - x1) * yp + (x1 * y2 - x2 * y1)) / det
    w1 = ((y2 - y0) * xp + (x0 - x2) * yp + (x2 * y0 - x0 * y2)) / det
    w2 = ((y0 - y1) * xp + (x1 - x0) * yp + (x0 * y1 - x1 * y0)) / det
    m = np.minimum(np.minimum(w0, w1), w2)
    dis = np.where(m > 0, m * m, -(m * m))
    return -dis < thr


def edge_pixels_alive(fv, side, i, S, dtype):
    """Pixels on the target column (sides 0, 1) or row (sides 2, 3) of an edge face, inside its box along the other axis,
    that the barycentric distance cut-off keeps: for these the box tests decide whether the pair is evaluated."""
    box = boxes(np.asarray(fv)[None], dtype)[0]
    c = float(pixel_centre(i, S, dtype))
    o = pixel_centre(np.arange(S), S, dtype)
    lo, hi = (box[2], box[3]) if side < 2 else (box[0], box[1])
    o = o[(o >= lo) & (o <= hi)].astype(np.float64)
    xp, yp = (np.full_like(o, c), o) if side < 2 else (o, np.full_like(o, c))
    return int(barycentric_alive(fv, xp, yp).sum())
