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


# ---------------------------------------------------------------------------------------------------------------------
# scenes of the visibility range tests (test_raster_visibility_range_gpu.py / _cpu.py): umr_raster_visibility's hard
# z-buffer, its planes (k_raster_fwd3<2>) and its visible-face bytes (k_visible_faces, which scans a face's pixel box
# per 64 x 64 bin: the tight vertex box + 2 pixels, or the whole cull box for a thin face, R_FLG bit 4).  Every scene
# returns face_vertices [B, F, 9] and a dict of its claims for the CPU checks.
# ---------------------------------------------------------------------------------------------------------------------
INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1
FAR_FACTORS = [0.5, 1.0, 2.0, 1e3]
WIDE_DRAWN = 5e7
FAR_BEHIND = [-0.3, -0.25, 2.0, 0.35, -0.2, 2.5, 0.05, 0.4, 2.0]   # a small nearer face in the middle of every far render


def bin_index(v, S, side):
    """k_visible_faces' pixel index of box coordinate v before the bin offset: floor (side -1) or ceil (+1) of
    (v S + S - 1) / 2 in float32, -2 / +2 pixels, as int64 (no saturation)."""
    e = ((np.float32(v) * np.float32(S) + np.float32(S - 1)) * np.float32(0.5)).astype(np.float32)
    return int(np.floor(e)) - 2 if side < 0 else int(np.ceil(e)) + 2


def crosses_int32(v, S, side):
    """Whether the unclamped index of box coordinate v leaves the int32 range at some bin of an S-pixel raster (the
    conversion saturates, or the margin or the bin offset x0 <= S - 1 wraps)."""
    i = bin_index(v, S, side)
    return i - (S - 1) < INT32_MIN if side < 0 else i > INT32_MAX


def far_faces(S, factors=FAR_FACTORS, z=5.0):
    """Faces covering the raster whose box reaches X = factor * 2^32 / S off it.
    thin: a sliver from a vertex X away on one side (axis x or y, side -1 low or +1 high) to an edge 1.5 off the other
          side; its smallest angle is about 1 / X, so it takes the whole-cull-box scan.  It covers the band between
          -0.5 and 0.5 across the raster.
    wide: a right triangle with its right angle on a corner (+-1.5, +-1.5) of the raster's surround and legs X long
          along x and y (the box reaches X off one x side and one y side; a triangle this wide reaching off one side
          only would be thin).  It covers the whole raster.
    One face per render, behind FAR_BEHIND and in front of an off-screen face (face F - 1 = 2 is then marked only by
    a background pixel).  Returns fv [B, 3, 9] and meta: (kind, axis, side, factor, X) per render.
    Which of them the z-buffer draws (oracle B): every thin one; the wide ones while X < WIDE_DRAWN (between 3.4e7 and
    6.7e7).  Past it the X^2 terms of the float32 barycentric inverse swamp the pixel terms and no pixel centre tests
    inside.  At S = 2048 the wide faces of factors 1/2 and 1 are not thin either (X^6, the product k_prep's bit-4 test
    forms, stays finite): they take the tight vertex box."""
    renders, meta = [], []
    for fac in factors:
        X = float(np.float32(fac * 2.0 ** 32 / S))
        for axis in (0, 1):
            for side in (-1, 1):
                v = [[side * X, -0.5], [-side * 1.5, -0.5], [-side * 1.5, 0.5 + 1e-3]]
                v = [p[::-1] if axis else p for p in v]
                renders.append([sum(([x, y, z] for x, y in v), []), FAR_BEHIND, list(OFF)])
                meta.append(("thin", axis, side, fac, X))
        for cx in (-1.5, 1.5):
            for cy in (-1.5, 1.5):
                v = [[cx, cy], [-np.sign(cx) * X, cy], [cx, -np.sign(cy) * X]]
                renders.append([sum(([x, y, z] for x, y in v), []), FAR_BEHIND, list(OFF)])
                meta.append(("wide", "x%+d y%+d" % (-np.sign(cx), -np.sign(cy)), 0, fac, X))
    return np.array(renders, np.float32), meta


def huge_faces(z=5.0):
    """Vertices at 1e15 and 1e20 and at +-inf, in far_faces' layout: the thin faces at 1e15 and 1e20 are drawn; the
    wide ones are not (at 1e15 as far_faces' past WIDE_DRAWN; at 1e20 x y overflows float32 and the barycentric inverse
    is not finite), nor is a face with an infinite vertex."""
    renders, meta = [], []
    for X in (1e15, 1e20):
        for kind, v in (("wide", [[-1.5, -1.5], [X, -1.5], [-1.5, X]]), ("thin", [[-X, -0.5], [1.5, -0.5], [1.5, 0.5]])):
            renders.append([sum(([x, y, z] for x, y in v), []), FAR_BEHIND, list(OFF)])
            meta.append((kind, X))
    for v in ([[-np.inf, -0.5], [1.5, -0.5], [1.5, 0.5]], [[-1.5, -1.5], [np.inf, -1.5], [-1.5, np.inf]],
              [[-np.inf, -1.5], [np.inf, -1.5], [0.0, 1.5]]):
        renders.append([sum(([x, y, z] for x, y in v), []), FAR_BEHIND, list(OFF)])
        meta.append(("inf", np.inf))
    return np.array(renders, np.float32), meta


THIN_CUT = np.float32(1e-6)


def thin_flag(f):
    """k_prep's bit 4 (raster.cu), restated in float32 for one face [9]: the sine of the smallest angle below ~1e-3."""
    x0, y0, _, x1, y1, _, x2, y2, _ = np.asarray(f, np.float32)
    l01 = (x1 - x0) * (x1 - x0) + (y1 - y0) * (y1 - y0)
    l02 = (x2 - x0) * (x2 - x0) + (y2 - y0) * (y2 - y0)
    l12 = (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1)
    lmin = np.fmin(np.fmin(l01, l02), l12)
    with np.errstate(all="ignore"):
        prod2 = (l01 * l02 * l12) / np.fmax(lmin, np.float32(1e-30))
        draw = x2 * (y0 - y1) + x0 * (y1 - y2) + x1 * (y2 - y0)
        return not bool(draw * draw >= THIN_CUT * prod2)


def _sliver(S, row, x_lo, x_hi, z, place=lambda f: f):
    """A right-angled sliver along pixel row `row` from x_lo to x_hi whose far corner's height crosses the bit-4 cut:
    (thin, not thin), the two adjacent float32 heights of that corner either side of the cut (a height of about
    1e-3 of its length).  Its base lies 1 % of that height below the row's centres, so it covers the row from about
    1 % of its length past its sharp end to its right-angled end."""
    xa, xb = np.float32(x_lo), np.float32(x_hi)
    yc = float(pixel_centre(S - 1 - row, S, np.float32))
    y0 = np.float32(yc - 1e-5 * (float(xb) - float(xa)))
    face = lambda y2: place(np.array([xa, y0, z, xb, y0, z, xb, y2, z], np.float32).reshape(3, 3)).reshape(9)   # noqa: E731
    lo, hi = np.float32(y0 + 1e-5 * (xb - xa)), np.float32(y0 + 0.01 * (xb - xa))   # thin at lo, not thin at hi
    assert thin_flag(face(lo)) and not thin_flag(face(hi))
    while np.nextafter(lo, hi) != hi:
        mid = np.float32((np.float64(lo) + np.float64(hi)) / 2)
        if mid == lo or mid == hi:
            mid = np.nextafter(lo, hi)
        lo, hi = (mid, hi) if thin_flag(face(mid)) else (lo, mid)
    return face(lo), face(hi)


def thin_switch(S):
    """Sliver pairs either side of k_prep's bit-4 cut, each sliver on a row of its own: along rows S/4 and S/4 + 2,
    mirrored in x along rows 3S/4 and 3S/4 + 2, and the four transposed (columns, behind the rows).  Each spans most of
    the raster (S >= 8).  Returns fv [1, 8, 9], the expected bit 4 per face."""
    px = 2.0 / S
    lo, hi = float(pixel_centre(1, S, np.float64)) - 0.25 * px, float(pixel_centre(S - 2, S, np.float64)) + 0.25 * px
    mirror = lambda f: f * np.float32([-1, 1, 1])           # noqa: E731
    transpose = lambda f: f[:, [1, 0, 2]]                     # noqa: E731
    faces, thin = [], []
    for k, (row, place) in enumerate(((S // 4, lambda f: f), ((3 * S) // 4, mirror), (S // 4, transpose),
                                      ((3 * S) // 4, lambda f: transpose(mirror(f))))):
        for t in range(2):   # the thin sliver on one row, the other on the row after next
            faces.append(_sliver(S, row + 2 * t, lo, hi, 2.0 + k, place)[t])
            thin.append(t == 0)
    return np.array(faces, np.float32)[None], np.array(thin)


def depth_order(S, seed=0):
    """Depth ties and near-ties, one render each:
    repeat   one face four times, between other faces: the lowest index wins everywhere;
    ulp      two overlapping constant-depth faces one float ulp apart, in both index orders;
    edge     two faces sharing an edge along a pixel-centre column (a barycentric exactly 0 there: fragment() decides)
             at the same depth, and a third sharing an edge along a pixel-centre row;
    centres  a face whose vertices are pixel centres, over one whose vertices are too."""
    rng = np.random.default_rng(seed)
    c = lambda i: float(pixel_centre(i, S, np.float32))   # noqa: E731
    rnd = rng.uniform(-0.9, 0.9, size=(2, 9)) * np.array([1, 1, 0] * 3) + np.array([0, 0, 3.0] * 3)
    tri = [-0.6, -0.5, 2.0, 0.7, -0.4, 2.5, -0.1, 0.8, 3.0]
    z = np.float32(2.0)
    zn = float(np.nextafter(z, np.float32(0)))
    flat = lambda zz: [-0.8, -0.7, zz, 0.75, -0.6, zz, 0.1, 0.85, zz]   # noqa: E731
    e = lambda k: c((k * S) // 8)   # noqa: E731
    m, a, b = c(S // 2), c(S // 4), c((3 * S) // 4)
    renders = {
        "repeat": [rnd[0], tri, tri, rnd[1], tri, tri],
        "ulp": [flat(2.0), flat(zn), OFF, OFF, OFF, OFF],
        "ulp reversed": [flat(zn), flat(2.0), OFF, OFF, OFF, OFF],
        # a diamond split along the column of e(2) (faces 0, 1) and one split along the row of e(6) (faces 2, 3)
        "edge": [[e(2), e(1), 2.0, e(2), e(3), 2.0, e(1), e(2), 2.0], [e(2), e(3), 2.0, e(2), e(1), 2.0, e(3), e(2), 2.0],
                 [e(5), e(6), 2.0, e(7), e(6), 2.0, e(6), e(7), 2.0], [e(7), e(6), 2.0, e(5), e(6), 2.0, e(6), e(5), 2.0],
                 OFF, OFF],
        "centres": [[a, a, 2.0, b, a, 2.0, m, b, 2.0], [c(1), c(1), 3.0, c(S - 2), c(1), 3.0, c(1), c(S - 2), 3.0],
                    OFF, OFF, OFF, OFF],
    }
    return np.array(list(renders.values()), np.float32), list(renders)


def zero_depths():
    """For near = 0: a face with a vertex at depth +0 and the same face with that vertex at -0 (every pixel of either
    has depth exactly +0 or -0: the clipped barycentric of that vertex is at least 1e-5), in both index orders, then an
    off-screen face.  The strict '<' of the z-buffer treats +0 and -0 as one depth: the lower index wins."""
    base = [-0.7, -0.6, 0.0, 0.8, -0.5, 2.0, 0.0, 0.75, 3.0]
    pos, neg = list(base), list(base)
    neg[2] = -0.0
    return np.array([[pos, neg, OFF], [neg, pos, OFF]], np.float32)


def negative_depths():
    """For near = -5, far = 5: faces at negative depths over faces at positive depths and one cut by near."""
    faces = [[-0.8, -0.7, 2.0, 0.75, -0.6, 2.5, 0.1, 0.85, 3.0],
             [-0.5, -0.4, -1.0, 0.6, -0.3, -1.5, 0.0, 0.6, -2.0],
             [-0.2, -0.9, -3.0, 0.9, 0.1, -0.5, -0.6, 0.5, -1.2],
             [-0.9, 0.2, -8.0, 0.2, 0.3, -2.0, -0.4, 0.9, -6.0],
             OFF]
    return np.array([faces], np.float32)


def depth_cut():
    """For far = 1e9: a constant-depth face at 1e7 (the z-buffer's initial depth_min) over one at the float below it,
    and the same pair the other way round in index."""
    z0, z1 = 1e7, float(np.nextafter(np.float32(1e7), np.float32(0)))
    a = [-0.8, -0.7, z0, 0.75, -0.6, z0, 0.1, 0.85, z0]
    b = [-0.6, -0.8, z1, 0.85, -0.5, z1, -0.1, 0.7, z1]
    return np.array([[a, b, OFF], [b, a, OFF]], np.float32)


def front_back(seed=0, F=12):
    """fill_back = False: front faces (even indices) and back faces (odd) interleaved and overlapping, the back faces
    nearer."""
    rng = np.random.default_rng(seed)
    faces = []
    for i in range(F):
        cx, cy = rng.uniform(-0.5, 0.5, size=2)
        r = rng.uniform(0.2, 0.5)
        v = [[cx - r, cy - r], [cx + r, cy - 0.5 * r], [cx, cy + r]]
        if i % 2 == 0:   # even faces front (k_prep's bit 3), odd ones back
            v = [v[0], v[2], v[1]]
        z = 2.0 + (0.0 if i % 2 else 1.0) + 0.01 * i
        faces.append(sum(([x, y, z] for x, y in v), []))
    fv = np.array(faces, np.float32)[None]
    return fv


def small(F, seed=0):
    """F = 1 or 2 faces (face 0 is then the background's marker too, or face 1)."""
    rng = np.random.default_rng(seed)
    base = np.array([[-0.6, -0.5, 2.0, 0.7, -0.4, 2.5, -0.1, 0.8, 3.0], [-0.9, -0.2, 2.2, 0.3, -0.9, 2.2, 0.5, 0.6, 4.0]])
    fv = base[:F] + rng.uniform(-0.05, 0.05, size=(F, 9)) * np.array([1, 1, 0] * 3)
    return fv[None].astype(np.float32)
