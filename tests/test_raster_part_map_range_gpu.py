"""The 4-channel part-map render (color_channels = 4: textures [G, F, T2, 4], images [B, 5, ...]) across its accepted input
range, through the float32 C entry points, against oracle B.

This is the render part_matching_loss draws every training step (loss_utils.part_matching_loss, its packed branch): one
raster call for the four part maps.  It runs on kernels of its own: k_raster_fwd3<1, 4, IdxT> (and the deterministic
k_raster_fwd3<1, 4, IdxT, true>) forward, whatever tile_mode says; k_raster_bwd2<1, false, 16, 4, ...> streaming the
saved pairs; k_raster_bwd_pairs(_list)<1, false, 4> recomputing the tiles left unsaved or, without a pair buffer, every
tile; k_raster_bwd_det<float, 1, false, 4> on the deterministic path.  There is no texel gradient (part maps are
constants).

Oracle B renders 3 channels, so the reference is composed from two of its renders (raster_range_harness.oracle4): A of
channels 0-2 on the background (b0, b1, b2), B of channels (3, 0, 1) on (bg3, b0, b1).  Each scene runs on the paths of
test_raster_fast_range_gpu (PATHS: a pair buffer with room for every tile at tile_mode 16 and 32, one leaving some tiles
unsaved, none, the deterministic path), once as is and once behind 65537 off-screen faces (the 32-bit face-index
kernels).  Besides the oracle gates, per path:
  - colour planes 0-2, alpha, aggrs (and the anti-aliased raster's planes) are bitwise the 3-channel kernels' render of
    A on the same path, plane 3 bitwise their render of B's plane 0 (the same arithmetic per channel, background
    included);
  - tile_mode 32 gives the planes and pair-buffer header of tile_mode 16 (the 4-channel render always uses 16x16 tiles);
  - deterministic: a second call gives the same bits, vertex gradient and p2f included, and so does soft_rasterize with
    a length-4 background_color under torch.use_deterministic_algorithms(True).

The default path's p2f and vertex gradient are float atomic sums, so across calls they agree to the gates, not bitwise.
Guard bands and gates are raster_range_harness.py's.  Each case prints its target and its worst error / bound ratio."""
import math

import numpy as np
import pytest
import torch

import raster_range_scenes as rs
from raster_range_harness import (DEV, KW, c_render, compare, oracle4, oracle_eps,
                                  oracle_on_the_kernel_grid)  # noqa: F401 (an autouse fixture)
from umr_b200 import raster, synth
from umr_b200.nnutils import loss_utils
from util import rel_report

pytestmark = pytest.mark.gpu
SIZES = [(1, False), (2, False), (17, False), (31, False), (33, False), (9, True), (17, True), (33, True)]
PATHS = ["full16", "full32", "partial", "none", "det"]
PAD = 65537          # off-screen faces put in front for the 32-bit face-index run
TEXEL_BITS = 23      # texel-index bits of the 4-channel pair record, at either tile_mode
BG = tuple(float(np.float32(c)) for c in (0.1, 0.7, 0.3))


def four(tex, seed=0):
    """tex [G, F, T2, 3] with a fourth channel: uniform, NaN where channel 0 is (rs.textured's unsampled texels)."""
    t = np.asarray(tex, np.float32)
    x = np.random.default_rng(seed + 1000).uniform(0, 1, size=t.shape[:3] + (1,)).astype(np.float32)
    x[np.isnan(t[..., :1])] = np.nan
    return np.concatenate([t, x], -1)


def _bits(a, b, what):
    assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), what


def _fit(B, S, run):
    """Blocks of a pair buffer with room for every tile: doubled until the forward leaves no tile unsaved."""
    blocks = B * ((S + 15) // 16) ** 2 * 16 + 64
    while True:
        out = run(blocks)
        if out["pairs"] is None or out["pairs"][1] == 0:
            return blocks, out
        blocks = 2 * max(blocks, out["pairs"][0])


def _sub(out, on):
    """The outputs of the on-screen faces `on` (ascending); every other face's p2f and vertex gradient must be 0."""
    res = {k: (v[:, on] if k in ("p2f", "grad_faces") else v) for k, v in out.items()
           if k not in ("t_bwd", "pairs") and v is not None}
    off = np.ones(out["p2f"].shape[1], bool)
    off[on] = False
    for k in ("p2f", "grad_faces"):
        if out.get(k) is not None:
            assert not out[k][:, off].any(), "%s of an off-screen face" % k
    return res


def _three_channel(cpath, fv, tex, isz, aa, k):
    """The 3-channel kernels' forward of A (channels 0-2 on (b0, b1, b2)) and of B (channels 3, 0, 1 on (bg3, b0, b1)) on
    the same path, 16x16 tiles, no pair buffer."""
    b0, b1, b2 = k["background_color"]
    ka, kb = dict(k, background_color=(b0, b1, b2)), dict(k, background_color=(k["background_extra"], b0, b1))
    a = c_render(cpath, fv, np.ascontiguousarray(tex[..., 0:3]), isz, aa, None, ka, tile=16)
    b = c_render(cpath, fv, np.ascontiguousarray(tex[..., [3, 0, 1]]), isz, aa, None, kb, tile=16)
    return a, b


def _planes_are_three_channel(got, a, b, aa, what):
    for name in ("images", "colors") if aa else ("images",):
        x = got[name]
        _bits(x[:, 0:3], a[name][:, 0:3], "%s: %s planes 0-2 are not the 3-channel render's" % (what, name))
        _bits(x[:, 4], a[name][:, 3], "%s: %s alpha is not the 3-channel render's" % (what, name))
        _bits(x[:, 3], b[name][:, 0], "%s: %s plane 3 is not the 3-channel render's plane 0 of B" % (what, name))
    _bits(got["aggrs"], a["aggrs"], "%s: aggrs are not the 3-channel render's" % what)


def autograd_render(fv, tex, isz, aa, g, k):
    """soft_rasterize with a length-4 background_color under torch.use_deterministic_algorithms(True)."""
    kk = {n: v for n, v in k.items() if n not in ("background_color", "background_extra")}
    bg = tuple(k["background_color"]) + (k["background_extra"],)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        tfv = torch.from_numpy(np.ascontiguousarray(fv)).to(DEV).requires_grad_(True)
        ttex = torch.from_numpy(np.ascontiguousarray(tex)).to(DEV)
        img, p2f, aggr = raster.soft_rasterize(tfv, ttex, isz, background_color=bg, anti_aliasing=aa, **dict(KW, **kk))
        img.backward(torch.from_numpy(np.ascontiguousarray(g)).to(DEV))
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(old)
    return dict(images=img.detach().cpu().numpy(), aggrs=aggr.cpu().numpy(), p2f=p2f.cpu().numpy(),
                grad_faces=tfv.grad.cpu().numpy().reshape(fv.shape[0], -1, 9))


def run_scene(fv, tex, isz, aa, what, feature, loose=False, on=None, wide=True, kw=None, seed=0, rtol=1e-4,
              paths=PATHS, blocks_want=None, autograd=True):
    """Every path of `paths` on one scene (and, with wide, again behind PAD off-screen faces) against oracle4, with the
    bitwise invariants of the module docstring.  on: the faces oracle B renders (the rest must stay off screen);
    blocks_want: the host-restated block cursor of the 16x16-tile forward.  Returns the worst error / bound ratio and
    the pair-buffer header of each path that ran."""
    fv, tex = np.ascontiguousarray(fv, np.float32), np.ascontiguousarray(tex, np.float32)
    B, F = fv.shape[:2]
    T2 = tex.shape[2]
    S = isz * (2 if aa else 1)
    on = np.arange(F) if on is None else np.asarray(on)
    g = np.random.default_rng(seed).uniform(-1, 1, size=(B, 5, isz, isz)).astype(np.float32)
    k = dict(dict(eps=oracle_eps(KW["gamma_val"]), background_color=(0.0, 0.0, 0.0), background_extra=0.0), **(kw or {}))
    ref = oracle4(fv[:, on], tex[:, on], isz, aa, g, k)
    worst, headers = 0.0, {}
    for P in ((0, PAD) if wide and F <= 65535 else (0,)):
        if P:
            pv = np.concatenate([np.broadcast_to(rs.OFF.astype(np.float32), (B, P, 9)), fv], 1)
            pt = np.concatenate([np.full((tex.shape[0], P) + tex.shape[2:], 0.5, np.float32), tex], 1)
        else:
            pv, pt = fv, tex
        idx = on + P
        tag = "%s%s" % (what, " F=%d" % pv.shape[1] if P or F > 65535 else "")
        three, full, wanted = {}, {}, None
        for path in paths:
            cpath = "det" if path == "det" else "default"
            tile = 32 if path == "full32" else 16
            pw = "%s %s" % (tag, path)

            def run(blocks, tile=tile):
                return c_render(cpath, pv, pt, isz, aa, g, k, grads=(True, False), nc=4, blocks=blocks, tile=tile)
            if path.startswith("full"):
                _, got = _fit(B, S, run)
                if T2 > 1 << TEXEL_BITS:   # the texel index does not fit the record: every tile recomputed
                    assert got["pairs"] is None, "%s: pair buffer used past the texel field %s" % (pw, got["pairs"])
                else:
                    assert got["pairs"] is not None and got["pairs"][1] == 0, "%s: pairs %s" % (pw, got["pairs"])
                full[path] = got
                if path == "full16":
                    wanted = got["pairs"][0] if got["pairs"] is not None else None
                    if blocks_want is not None:
                        assert wanted == blocks_want, "%s: %s blocks wanted, the host restatement says %d" % (pw, wanted, blocks_want)
                elif "full16" in full:
                    a16 = full["full16"]
                    assert got["pairs"] == a16["pairs"], "%s: header %s, tile_mode 16 %s" % (pw, got["pairs"], a16["pairs"])
                    for name in ("images", "colors", "aggrs"):
                        if got.get(name) is not None:
                            _bits(got[name], a16[name], "%s: %s differ from tile_mode 16" % (pw, name))
            elif path == "partial":
                if wanted is None or wanted // 3 < 4:   # below 4 blocks a buffer is no buffer
                    print("%s: unreachable (%s blocks wanted)" % (pw, wanted))
                    continue
                got = run(wanted // 3)
                assert got["pairs"][1] > 0, "%s: every tile saved %s" % (pw, got["pairs"])
            else:
                got = run(0)
                assert got["pairs"] is None
            headers[path] = got["pairs"]
            w = compare(cpath, _sub(got, idx), ref, "softmax", pw, rtol, loose)
            if cpath not in three:
                three[cpath] = _three_channel(cpath, pv, pt, isz, aa, k)
            _planes_are_three_channel(got, *three[cpath], aa, pw)
            if path == "det":
                again = run(0)
                for name in ("images", "colors", "aggrs", "p2f", "grad_faces"):
                    if got.get(name) is not None:
                        _bits(got[name], again[name], "%s: %s differs in a second call" % (pw, name))
                if autograd and not P:
                    auto = autograd_render(pv, pt, isz, aa, g, k)
                    for name in ("images", "aggrs", "p2f", "grad_faces"):
                        _bits(auto[name], got[name], "%s: soft_rasterize %s is not the C call's" % (pw, name))
            worst = max(worst, w)
            print("%s: %s; pairs %s; worst error/bound %.3g" % (pw, feature, got["pairs"], w))
    return worst, headers


def _sz(isz, aa):
    return "IS=%d aa" % isz if aa else "S=%d" % isz


def _union_outside_tiles(fv, S):
    """16x16 tiles outside the union of an image's cull boxes (the forward's empty-tile path), summed over images."""
    n = 0
    nt = (S + 15) // 16
    for img in fv:
        box = rs.boxes(img, np.float32)
        u = np.array([[np.nanmin(box[:, 0]), np.nanmax(box[:, 1]), np.nanmin(box[:, 2]), np.nanmax(box[:, 3])]], np.float32)
        n += sum(not bool(rs.tile_hits(u, S, tx, ty, np.float32)[0]) for ty in range(nt) for tx in range(nt))
    return n


# ---------------------------------------------------------------------------------------------------------------------
# the recompute kernels' shared memory: face counts either side of the 48 KB default
# ---------------------------------------------------------------------------------------------------------------------
FACE_COUNTS = [1280, 1543, 1544, 2048, 2049, 5120, 65535, 65536]


def _sparse(F, seed=0):
    """F faces, four of them on screen (indices 0, F // 3, F // 2 and F - 1, returned), every other one off it."""
    on = np.unique([0, F // 3, F // 2, F - 1])
    fv = np.tile(rs.OFF, (F, 1))
    fv[on] = [[-0.6 + 0.3 * j, -0.5, 3.0 + j, 0.7, -0.4 + 0.2 * j, 4.0 + j, -0.1 * j, 0.8, 5.0 - j * 0.3] for j in range(len(on))]
    tex = np.full((1, F, 4, 4), 0.5)
    tex[0, on] = np.random.default_rng(seed).uniform(0, 1, size=(len(on), 4, 4))
    return fv[None].astype(np.float32), tex.astype(np.float32), on


@pytest.mark.parametrize("buffer", [True, False])
@pytest.mark.parametrize("F", FACE_COUNTS)
def test_face_counts_across_the_shared_memory_default(F, buffer):
    """The default backward at F faces, with a pair buffer (the streamed backward, then k_raster_bwd_pairs_list over no
    or some unsaved tiles) and without (k_raster_bwd_pairs): their dynamic shared memory, 8192 + 16 min(F, 2048) +
    round16(2 min(F, 65536)) bytes beside 13184 static, passes the 48 KB a kernel gets without the opt-in from 1544 faces."""
    fv, tex, on = _sparse(F, seed=F)
    dyn = 8192 + 16 * min(F, 2048) + ((2 * min(F, 65536) + 15) & ~15)
    run_scene(fv, tex, 17, True, "F=%d" % F, "%d B dynamic shared memory, faces %s on screen" % (dyn, on.tolist()), on=on,
              wide=False, paths=["full16", "partial"] if buffer else ["none"])


# ---------------------------------------------------------------------------------------------------------------------
# sizes, box edges, saved records, covering faces
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("isz,aa", SIZES)
def test_edges(isz, aa):
    """Box edges on pixel centres and one step beside them at the raster ends and the 15 | 16, 31 | 32 and 63 | 64
    boundaries."""
    S = isz * (2 if aa else 1)
    fv, tex, meta = rs.edges(S, np.float32, seed=S, fast=True)
    run_scene(fv, four(tex, S), isz, aa, "edges %s" % _sz(isz, aa),
              "%d box sides on a pixel centre, %d one step beside" % ((meta[:, 2] == 0).sum(), (meta[:, 2] != 0).sum()),
              blocks_want=rs.fwd3_blocks_wanted(fv, S))


@pytest.mark.parametrize("isz,aa", SIZES)
def test_big_boxes(isz, aa):
    """Boxes over and off the raster, and a face with a NaN vertex (the box of its finite coordinates)."""
    for nan in (False, True):
        fv, tex = rs.big(np.float32, seed=isz, nan=nan)
        run_scene(fv, four(tex, isz), isz, aa, "big%s %s" % (" + NaN box" if nan else "", _sz(isz, aa)),
                  "%d faces" % fv.shape[1], loose=True, wide=not nan)


@pytest.mark.parametrize("isz,aa", [(17, False), (33, False), (17, True), (33, True)])
@pytest.mark.parametrize("extra", [0, 1, 2])
def test_saved_records(extra, isz, aa):
    """Tile (0, 0) saves 32 x 8 records in eight full blocks of the covering face, + extra blocks of one record."""
    S = isz * (2 if aa else 1)
    fv, tex = rs.records(S, extra)
    run_scene(fv, four(tex, S + extra), isz, aa, "records %s +%d" % (_sz(isz, aa), extra),
              "tile (0, 0) saves %d records" % rs.tile_records(fv[0], S)[0, 0], loose=True,
              blocks_want=rs.fwd3_blocks_wanted(fv, S))


# ---------------------------------------------------------------------------------------------------------------------
# crowded tile lists and the recompute fallback's face window
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("isz,aa", [(17, False), (17, True)])
@pytest.mark.parametrize("name", sorted(rs.CROWDS))
def test_crowds(name, isz, aa):
    S = isz * (2 if aa else 1)
    fv, tex, hit = rs.crowd(rs.CROWDS[name], S, np.float32, seed=len(name) + S)
    segs = rs.fwd3_segments(rs.boxes(fv[0], np.float32), S)
    run_scene(fv, four(tex, S), isz, aa, "crowd %s %s" % (name, _sz(isz, aa)),
              "%d faces on tile (0, 0), segments %s" % (len(hit), [c for c, _ in segs]),
              blocks_want=rs.fwd3_blocks_wanted(fv, S))


def test_crowd_of_65535_faces():
    """65535 faces of one pixel each on tile (0, 0): 128 LCAP segments, every face its own pair block."""
    fv, tex = rs.crowd_all(34, np.float32, seed=34)
    run_scene(fv, four(tex, 34), 17, True, "65535 faces in one tile IS=17 aa", "%d faces" % fv.shape[1], wide=False,
              blocks_want=rs.fwd3_blocks_wanted(fv, 34))


def test_recompute_crosses_the_face_window():
    """F = 65540: the recompute fallback lists faces 0 and 65535 in its first face window, 65536 and 65539 in its second."""
    fv, tex, on = rs.window_crossing()
    for isz, aa in ((17, True), (33, False)):
        run_scene(fv, four(tex, isz), isz, aa, "window crossing %s" % _sz(isz, aa), "faces %s on screen" % on.tolist(),
                  on=on, wide=False)


# ---------------------------------------------------------------------------------------------------------------------
# far-off, huge and infinite vertices
# ---------------------------------------------------------------------------------------------------------------------
def _textures(fv, T2=4, seed=0):
    return np.random.default_rng(seed).uniform(0, 1, size=fv.shape[:2] + (T2, 4)).astype(np.float32)


@pytest.mark.parametrize("isz,aa", [(64, False), (32, True)])
def test_far_off_boxes(isz, aa):
    """Faces covering the raster whose box reaches 1/2, 1, 2 and 1000 x 2^32 / S off it (rs.far_faces)."""
    S = isz * (2 if aa else 1)
    fv, meta = rs.far_faces(S)
    run_scene(fv, _textures(fv, seed=S), isz, aa, "far-off boxes %s" % _sz(isz, aa), "%d renders" % len(meta), loose=True)


def test_huge_and_infinite_vertices():
    """Vertices at 1e15 and 1e20 and at +-inf (rs.huge_faces)."""
    fv, meta = rs.huge_faces()
    for isz, aa in ((64, False), (33, True)):
        run_scene(fv, _textures(fv, seed=isz), isz, aa, "huge vertices %s" % _sz(isz, aa), "%d renders" % len(meta),
                  loose=True)


# ---------------------------------------------------------------------------------------------------------------------
# the fourth channel's background
# ---------------------------------------------------------------------------------------------------------------------
def _corner_scene(seed=0):
    """Three faces in the upper-left quarter of the raster: the tiles beyond their union box take the forward's empty-tile
    path, the tiles their boxes reach are partly covered."""
    rng = np.random.default_rng(seed)
    fv = np.array([[-0.9, 0.1, 2.0, -0.2, 0.15, 2.5, -0.6, 0.85, 3.0],
                   [-0.7, 0.3, 2.2, -0.1, 0.5, 2.2, -0.4, 0.05, 4.0],
                   [-0.95, 0.6, 3.0, -0.5, 0.6, 3.0, -0.75, 0.95, 3.0]], np.float32)[None]
    return fv, rng.uniform(0, 1, size=(1, 3, 4, 4)).astype(np.float32)


@pytest.mark.parametrize("isz,aa", [(33, False), (32, True), (17, True)])
@pytest.mark.parametrize("extra", [0.0, 0.37, -1.5])
def test_background_extra(extra, isz, aa):
    """background_extra (bg3) in {0, 0.37, -1.5} beside background_color (0.1, 0.7, 0.3), on empty and partly covered
    16x16 tiles; IS = 32 anti-aliased stores the empty tiles with 128-bit stores.  On empty tiles plane 3 comes from bg3
    alone: bitwise the 3-channel render of B's plane 0 (checked on every plane, every path)."""
    S = isz * (2 if aa else 1)
    fv, tex = _corner_scene(seed=S)
    empty = _union_outside_tiles(fv, S)
    assert empty > 0 and empty < ((S + 15) // 16) ** 2
    bg3 = float(np.float32(extra))
    run_scene(fv, tex, isz, aa, "bg3 %g %s" % (bg3, _sz(isz, aa)),
              "%d of %d tiles empty" % (empty, ((S + 15) // 16) ** 2), kw=dict(background_color=BG, background_extra=bg3))
    # covering faces, anti-aliased and not: every tile partly covered, bg3 only where the soft colours mix it in
    fv, tex = rs.big(np.float32, seed=S)
    run_scene(fv, four(tex, S), isz, aa, "bg3 %g big %s" % (bg3, _sz(isz, aa)), "covering face", loose=True,
              kw=dict(background_color=BG, background_extra=bg3))


# ---------------------------------------------------------------------------------------------------------------------
# textures
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T2", [1, 5, 36])
def test_textures(T2):
    fv, tex = rs.textured(T2, np.float32, seed=T2)
    for isz, aa in ((17, True), (33, False)):
        run_scene(fv, four(tex, T2), isz, aa, "T2=%d %s" % (T2, _sz(isz, aa)), "R^2 %d" % math.isqrt(T2) ** 2, loose=True)


@pytest.mark.parametrize("R", [2896, 2897])
def test_texel_field_edge(R):
    """T2 = R^2 either side of the pair record's 2^23 texel indices: 2896^2 saves pairs at tile_mode 16 and 32, 2897^2
    recomputes every tile.  F = 2, B = 1 (about 134 MB of texture per face)."""
    fv, tex = rs.textured(R * R, np.float32, seed=R)
    tex = four(tex, R)
    _, headers = run_scene(fv, tex, 9, True, "T2=%d^2 IS=9 aa" % R, "T2 %d vs 2^23 = %d" % (R * R, 1 << TEXEL_BITS),
                           loose=True, wide=False, autograd=False)
    fits = R * R <= 1 << TEXEL_BITS
    assert (headers["full16"] is not None) == fits and (headers["full32"] is not None) == fits, headers


@pytest.mark.parametrize("G", [1, 2, 8])
def test_shared_textures(G):
    """8 renders over G textures (G = 1: part_matching_loss's batch-shared layout).  The deterministic render of each is
    bitwise the render with the textures expanded to [8, ...]."""
    fv, tex = rs.shared(8, G, "surface", np.float32, seed=G)
    tex = four(tex, G)
    run_scene(fv, tex, 17, True, "shared G=%d" % G, "%d images per texture" % (8 // G), loose=True)
    g = np.random.default_rng(G).uniform(-1, 1, size=(8, 5, 17, 17)).astype(np.float32)
    k = dict(eps=oracle_eps(KW["gamma_val"]), background_color=BG, background_extra=0.25)
    shared = c_render("det", fv, tex, 17, True, g, k, grads=(True, False), nc=4)
    expanded = c_render("det", fv, np.repeat(tex, 8 // G, 0), 17, True, g, k, grads=(True, False), nc=4)
    for name in ("images", "colors", "aggrs", "p2f", "grad_faces"):
        _bits(shared[name], expanded[name], "shared G=%d: %s differs from the expanded textures'" % (G, name))


def test_65535_images():
    """B = 65535, the forward's gridDim.z and the backward's gridDim.y limit, F = 2, IS = 1 anti-aliased."""
    fv, tex = rs.many_images(65535, seed=7, dtype=np.float32)
    run_scene(fv, four(tex, 7), 1, True, "B=65535", "65535 images", loose=True, wide=False)


# ---------------------------------------------------------------------------------------------------------------------
# Python level
# ---------------------------------------------------------------------------------------------------------------------
def _loss_step(one_hot, verts, faces, cams, segs, IS, T, packed):
    m = loss_utils.part_matching_loss(None, None, 0, im_size=IS, batch_size=verts.shape[0], tex_size=T,
                                      stex_one_hot=one_hot).to(DEV)
    m.pack_parts = packed
    vv, cc = verts.clone().requires_grad_(True), cams.clone().requires_grad_(True)
    loss, projs = m(vv, faces, cc, segs)
    gv, gc = torch.autograd.grad(loss, (vv, cc))
    torch.cuda.synchronize()
    return loss.detach(), [p.detach() for p in projs], gv, gc


def test_part_matching_loss_on_5120_faces():
    """part_matching_loss on the 5120-face icosphere: the packed branch (one 4-channel render, its default backward)
    against four 3-channel renders -- part maps bitwise, the loss and the vertex and camera gradients within the gates
    of test_part_head_gpu.test_module_branches."""
    B, IS, T = 2, 32, 2
    rng = np.random.default_rng(5)
    v, f = synth.icosphere(4)
    assert f.shape[0] == 5120
    part = rng.integers(0, 5, size=(f.shape[0], T * T))
    one_hot = torch.zeros(1, f.shape[0], T * T, 5)
    one_hot.scatter_(3, torch.from_numpy(part)[None, :, :, None], 1.0)
    verts = torch.from_numpy(synth.bird_like(v, rng, B)).to(DEV)
    faces = torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1).to(DEV)
    cams = torch.from_numpy(synth.cameras(rng, B)).to(DEV)
    segs = torch.rand(B, 5, IS, IS, generator=torch.Generator().manual_seed(5)).to(DEV)
    packed = _loss_step(one_hot, verts, faces, cams, segs, IS, T, True)
    four_renders = _loss_step(one_hot, verts, faces, cams, segs, IS, T, False)
    for k, (a, b) in enumerate(zip(packed[1], four_renders[1])):
        assert torch.equal(a, b), "part map %d differs between the branches" % k
    assert abs(float(packed[0]) - float(four_renders[0])) <= 1e-6 * max(1.0, abs(float(four_renders[0])))
    for name, a, b in (("d/dverts", packed[2], four_renders[2]), ("d/dcams", packed[3], four_renders[3])):
        a, b = a.double().cpu().numpy(), b.double().cpu().numpy()
        ok, msg = rel_report(name, a, b, 1e-3, 1e-5 * float(np.abs(b).max()) + 1e-300)
        print(msg)
        assert ok and np.isfinite(a).all() and np.abs(b).max() > 0, msg


def test_four_channel_vertex_textures_are_refused():
    """Vertex textures render 3 channels: a [B, F, 3, 4] vertex texture would be read with a stride of 3."""
    fv = torch.from_numpy(rs.small(2)).to(DEV)
    tex = torch.rand(1, 2, 3, 4, device=DEV)
    with pytest.raises(ValueError, match="vertex textures take 3 colour channels"):
        raster.soft_rasterize(fv, tex, 16, texture_type="vertex")
    img, _, _ = raster.soft_rasterize(fv, tex[..., :3].contiguous(), 16, texture_type="vertex")
    assert img.shape == (1, 4, 16, 16)
