"""The default float32 rasteriser (umr_raster_forward / umr_raster_backward), its split backward
(umr_raster_backward_split(_deterministic)) and the silhouette render (umr_raster_*_silhouette(_deterministic)) across
their accepted input range, through their C entry points, against CPU oracle B in float32.

This is the path of every training step: k_prep, k_bin_coarse, k_raster_fwd3 / k_raster_fwd4 saving pair records, and
k_raster_bwd2 streaming them, with k_raster_bwd_pairs(_list) recomputing the tiles the pair buffer could not hold.  Each
scene runs on these paths (PATHS): a pair buffer with room for every tile at tile_mode 16 and 32, a pair buffer that
leaves some tiles unsaved (k_raster_bwd2 and k_raster_bwd_pairs_list), none (k_raster_bwd_pairs), and the deterministic
path; and each again with 65537 off-screen faces in front of its own, so the 32-bit face-index kernels run with every
on-screen face index above 65535.  The pair buffer's header after each forward asserts the state reached.

Per scene, path and colour mode (softmax, hard), one set of inputs is checked against oracle B:
  full        every plane, p2f, grad_faces and grad_textures, all four adjoints non-zero;
  split       grad_faces against oracle B's with the colour adjoints zeroed, grad_textures against oracle B's;
  silhouette  alpha (and the anti-aliased raster's alpha) and grad_faces against oracle B's alpha-only gradient; alpha
              bitwise the full render's on the same path, and the same pair-buffer header.
On the deterministic path the split and silhouette calls are bitwise equal to a second call and to the deterministic
full backward with zero colour adjoints (the texel gradient: to the texture-only call).

The scenes are raster_range_scenes.py's, with the fast path's own boundaries: tile lists of LCAP +- 1, FWD4_CAP +- 1 and
65535 faces on one tile, box edges on the 31 | 32 and 63 | 64 (coarse bin) pixel centres, tiles saving 32 k and
32 k + 1 records, a face window crossed by the recompute fallback, B = 65535 and IS = 1024.  Guard bands and gates are
raster_range_harness.py's.  Each case prints its target count and its worst error / bound ratio."""
import math

import numpy as np
import pytest

import raster_range_scenes as rs
from raster_range_harness import (KW, c_render, c_silhouette, compare, oracle, oracle_eps,
                                  oracle_on_the_kernel_grid)  # noqa: F401 (an autouse fixture)

pytestmark = pytest.mark.gpu
SIZES = [(1, False), (2, False), (17, False), (31, False), (33, False), (9, True), (17, True), (33, True)]
PATHS = ["full16", "full32", "partial", "none", "det"]
PAD = 65537   # off-screen faces put in front for the 32-bit face-index run


def _fit(B, isz, aa, S, tile, run):
    """Blocks of a pair buffer with room for every tile: doubled until the forward leaves no tile unsaved for want of
    room (k_raster_fwd4's windowed path saves no pairs whatever the room)."""
    blocks = B * ((S + 15) // 16) ** 2 * 16 + 64
    while True:
        out = run(blocks, tile)
        if out["pairs"] is None or out["pairs"][1] == 0 or out["pairs"][0] <= blocks:
            return blocks, out
        blocks = 2 * max(blocks, out["pairs"][0])


def _sub(out, on, rgb):
    """The outputs of the on-screen faces `on` (ascending), face ids of the hard plane mapped to oracle B's."""
    res = {k: (v[:, on] if k in ("p2f", "grad_faces", "grad_tex") else v) for k, v in out.items()
           if k not in ("t_bwd", "pairs") and v is not None}
    if "aggrs" in res and rgb == "hard":
        res["aggrs"] = res["aggrs"].copy()
        ids = res["aggrs"][:, 1]
        assert np.isin(ids[ids >= 0], on).all(), "an off-screen face won a pixel"
        res["aggrs"][:, 1] = np.where(ids >= 0, np.searchsorted(on, np.maximum(ids, 0)), ids)
    off = np.ones(out["p2f"].shape[1] if "p2f" in out else out["grad_faces"].shape[1], bool)
    off[on] = False
    for k in ("p2f", "grad_faces", "grad_tex"):
        if out.get(k) is not None:
            assert not out[k][:, off].any(), "%s of an off-screen face" % k
    return res


def _alpha_only(g):
    ga = np.zeros_like(g)
    ga[:, 3] = g[:, 3]
    return ga


def _bits(a, b, what):
    assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), what


def _nan_subset(got, ref, what):
    """A NaN vertex: oracle B forms the colour terms of the vertex gradient with zero adjoints too (0 x NaN), which the
    float32 kernels do not take (DESIGN.md §9); the split and silhouette gradients may be NaN only where oracle B's is."""
    assert not (np.isnan(got) & ~np.isnan(ref)).any(), what


def _same_pairs(a, b, what):
    """The same blocks wanted; with a partial buffer, which tiles win the room is a race, so only that some lost it."""
    assert (a is None) == (b is None) and (a is None or (a[0] == b[0] and (a[1] == 0) == (b[1] == 0))), "%s: %s %s" % (what, a, b)


def run_scene(fv, tex, isz, aa, what, feature, loose=False, on=None, wide=True, rgbs=("softmax", "hard"), blocks_want=None,
              kw=None, seed=0, fwd4_slow=False, rtol=1e-4, nan=False):
    """Every path of PATHS on one scene (and, with wide, again behind PAD off-screen faces) against oracle B.  on: the
    faces oracle B renders (the rest must stay off screen); blocks_want: the host-restated block cursor of the
    16x16-tile forward; fwd4_slow: a coarse list longer than FWD4_CAP, whose 32x32 tiles save no pairs; rtol: the planes'
    relative gate; nan: a scene with a NaN vertex (_nan_subset)."""
    fv, tex = fv.astype(np.float32), tex.astype(np.float32)
    B, F = fv.shape[:2]
    S = isz * (2 if aa else 1)
    on = np.arange(F) if on is None else on
    g = np.random.default_rng(seed).uniform(-1, 1, size=(B, 4, isz, isz)).astype(np.float32)
    ga = _alpha_only(g)
    worst, states = 0.0, {}
    for rgb in rgbs:
        k = dict(dict(aggr_func_rgb=rgb, eps=oracle_eps(KW["gamma_val"])), **(kw or {}))
        ref = oracle("det", fv[:, on], tex[:, on], isz, aa, g, k, alpha_only=True)
        ref_split = dict(grad_faces=ref["grad_faces_alpha"], grad_tex=ref["grad_tex"], grad_tex_abs=ref["grad_tex_abs"])
        ref_sil = dict(images=ref["images"][:, 3], colors=ref["colors"][:, 3] if aa else None, grad_faces=ref["grad_faces_alpha"])
        for P in ((0, PAD) if wide and F <= 65535 else (0,)):
            if P:
                pv = np.concatenate([np.broadcast_to(rs.OFF.astype(np.float32), (B, P, 9)), fv], 1)
                pt = np.concatenate([np.full((tex.shape[0], P) + tex.shape[2:], 0.5, np.float32), tex], 1)
            else:
                pv, pt = fv, tex
            idx = on + P
            tag = "%s %s%s" % (what, rgb, " F=%d" % pv.shape[1] if P or F > 65535 else "")
            wanted = None
            for path in PATHS:
                cpath = "det" if path == "det" else "default"
                tile = 32 if path == "full32" else 16
                run = lambda blocks, tile, gg=g, **a: c_render(cpath, pv, pt, isz, aa, gg, k, blocks=blocks, tile=tile, **a)  # noqa: E731
                blocks = 0
                if path.startswith("full"):
                    blocks, got = _fit(B, isz, aa, S, tile, run)
                    # the pair record's texel field holds 2^21 texels at 32x32 tiles: past that the buffer is not used
                    assert got["pairs"] is not None or (tile == 32 and pt.shape[2] > 1 << 21), "%s: pair buffer unused" % tag
                    assert got["pairs"] is None or (got["pairs"][1] > 0) == (tile == 32 and fwd4_slow), \
                        "%s %s: unsaved tiles %s" % (tag, path, got["pairs"])
                    if path == "full16":
                        wanted = got["pairs"][0]
                        if blocks_want is not None:
                            assert wanted == blocks_want, "%s: %d blocks wanted, the host restatement says %d" % (tag, wanted, blocks_want)
                elif path == "partial":
                    blocks = wanted // 3
                    if blocks < 4:   # a buffer below 4 blocks is no buffer: the state needs a render of 12 blocks or more
                        print("%s partial: unreachable (%d blocks wanted)" % (tag, wanted))
                        continue
                    got = run(blocks, tile)
                    assert got["pairs"][1] > 0, "%s partial: every tile saved %s" % (tag, got["pairs"])
                else:
                    got = run(0, tile)
                    assert got["pairs"] is None
                states[path] = states.get(path, 0) + 1
                pw = "%s %s" % (tag, path)
                w = compare(cpath, _sub(got, idx, rgb), ref, rgb, pw + " full", rtol, loose)
                sp = run(blocks, tile, split=True)
                _same_pairs(sp["pairs"], got["pairs"], pw + " split")
                if nan:
                    _nan_subset(sp["grad_faces"][:, idx], ref_split["grad_faces"], pw + " split")
                    w = max(w, compare(cpath, dict(grad_tex=sp["grad_tex"][:, idx]), ref_split, rgb, pw + " split", rtol, loose))
                else:
                    w = max(w, compare(cpath, _sub(sp, idx, rgb), ref_split, rgb, pw + " split", rtol, loose))
                sil = c_silhouette(cpath, pv, isz, aa, g[:, 3], k, blocks=blocks, tile=tile)
                if got["pairs"] is None and sil["pairs"] is not None:   # the texel field limit does not bind an alpha-only render
                    assert tile == 32 and sil["pairs"][1] == 0, "%s silhouette %s" % (pw, sil["pairs"])
                else:
                    _same_pairs(sil["pairs"], got["pairs"], pw + " silhouette")
                _bits(sil["alpha"], got["images"][:, 3], pw + ": silhouette alpha is not the full render's")
                if aa:
                    _bits(sil["alpha_hi"], got["colors"][:, 3], pw + ": silhouette raster alpha is not the full render's")
                sil_c = dict(images=sil["alpha"], colors=sil.get("alpha_hi"), grad_faces=sil["grad_faces"][:, idx])
                assert not sil["grad_faces"][:, np.setdiff1d(np.arange(pv.shape[1]), idx)].any()
                if nan:
                    _nan_subset(sil_c.pop("grad_faces"), ref_sil["grad_faces"], pw + " silhouette")
                w = max(w, compare(cpath, sil_c, ref_sil, "softmax", pw + " silhouette", rtol, loose))
                if path == "det":
                    _bits(sp["grad_faces"], run(0, 0, split=True)["grad_faces"], pw + ": split second call")
                    _bits(sil["grad_faces"], c_silhouette(cpath, pv, isz, aa, g[:, 3], k)["grad_faces"], pw + ": silhouette second call")
                    zero = run(0, 0, gg=ga)
                    _bits(sp["grad_faces"], zero["grad_faces"], pw + ": split vertex gradient is not the alpha-only one")
                    _bits(sil["grad_faces"], zero["grad_faces"], pw + ": silhouette gradient is not the alpha-only one")
                    _bits(sp["grad_tex"], run(0, 0, grads=(False, True))["grad_tex"], pw + ": split texel gradient")
                worst = max(worst, w)
                print("%s: %s; pairs %s; worst error/bound %.3g" % (pw, feature, got["pairs"], w))
    return worst, states


def _sz(isz, aa):
    return "IS=%d aa" % isz if aa else "S=%d" % isz


# ---------------------------------------------------------------------------------------------------------------------
# the fast path's own boundaries
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", rs.LIST_LENGTHS)
def test_tile_list_lengths(n):
    """n faces of one pixel each on tile (0, 0): k_raster_fwd3's list crosses (or ends on) an LCAP segment,
    k_raster_fwd4's an FWD4_CAP list; every face is its own pair block."""
    for isz, aa in ((17, True),) if n == 65535 else ((17, False), (17, True)):
        S = isz * (2 if aa else 1)
        fv, tex = rs.crowd_all(S, np.float32, seed=n + S, F=n)
        box = rs.boxes(fv[0], np.float32)
        seg = rs.fwd3_segments(box, S)
        assert sum(c for c, _ in seg) == n
        run_scene(fv, tex, isz, aa, "list of %d %s" % (n, _sz(isz, aa)),
                  "segments %s, fwd4 list %d vs FWD4_CAP %d" % ([c for c, _ in seg], n, rs.FWD4_CAP),
                  blocks_want=rs.fwd3_blocks_wanted(fv, S), rgbs=("softmax", "hard") if n < 65535 else ("softmax",),
                  wide=n < 65535, fwd4_slow=n > rs.FWD4_CAP)


@pytest.mark.parametrize("isz,aa", SIZES)
def test_edges(isz, aa):
    """Box edges on pixel centres and one step beside them at the raster ends and the 15 | 16, 31 | 32 and 63 | 64
    boundaries (the last two: k_raster_fwd4's tile and the coarse bin; the faces reaching 1.5 into the raster from a
    63 | 64 edge straddle two bins)."""
    S = isz * (2 if aa else 1)
    fv, tex, meta = rs.edges(S, np.float32, seed=S, fast=True)
    box = rs.boxes(fv[0], np.float32)
    straddle = sum(bool(rs.tile_hits(box[f:f + 1], S, 0, 0, np.float32, rs.CB)[0]) and
                   bool(rs.tile_hits(box[f:f + 1], S, 1, 0, np.float32, rs.CB)[0] or rs.tile_hits(box[f:f + 1], S, 0, 1, np.float32, rs.CB)[0])
                   for f in range(fv.shape[1])) if S > rs.CB else 0
    run_scene(fv, tex, isz, aa, "edges %s" % _sz(isz, aa),
              "%d box sides on a pixel centre, %d one step beside, %d boxes over two coarse bins"
              % ((meta[:, 2] == 0).sum(), (meta[:, 2] != 0).sum(), straddle), blocks_want=rs.fwd3_blocks_wanted(fv, S))


@pytest.mark.parametrize("isz,aa", [(17, False), (33, False), (17, True), (33, True)])
@pytest.mark.parametrize("extra", [0, 1, 2])
def test_saved_records(extra, isz, aa):
    """Tile (0, 0) saves 32 x 8 records in eight full blocks of the covering face, + extra blocks of one record."""
    S = isz * (2 if aa else 1)
    fv, tex = rs.records(S, extra)
    recs = rs.tile_records(fv[0], S)
    assert recs[0, 0] == 32 * 8 + extra
    run_scene(fv, tex, isz, aa, "records %s +%d" % (_sz(isz, aa), extra), "tile (0, 0) saves %d records" % recs[0, 0],
              loose=True, blocks_want=rs.fwd3_blocks_wanted(fv, S))


def test_recompute_crosses_the_face_window():
    """F = 65540: the recompute fallback lists faces 0 and 65535 in its first face window, 65536 and 65539 in its second."""
    fv, tex, on = rs.window_crossing()
    for isz, aa in ((17, True), (33, False)):
        run_scene(fv, tex, isz, aa, "window crossing %s" % _sz(isz, aa), "faces %s on screen" % on.tolist(), on=on, wide=False)


# ---------------------------------------------------------------------------------------------------------------------
# the range scenes of the gather tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("isz,aa", SIZES)
def test_big_boxes(isz, aa):
    """Boxes over and off the raster, and a face with a NaN vertex (the box of its finite coordinates)."""
    for nan in (False, True):
        fv, tex = rs.big(np.float32, seed=isz, nan=nan)
        run_scene(fv, tex, isz, aa, "big%s %s" % (" + NaN box" if nan else "", _sz(isz, aa)), "%d faces" % fv.shape[1],
                  loose=True, wide=not nan, nan=nan)


@pytest.mark.parametrize("T2", [1, 5, 36, 1449 ** 2])
def test_textures(T2):
    fv, tex = rs.textured(T2, np.float32, seed=T2 % 1000)
    R = math.isqrt(T2)
    for isz, aa in ((17, True), (33, False)):
        run_scene(fv, tex, isz, aa, "T2=%d %s" % (T2, _sz(isz, aa)), "T2 %d, R^2 %d" % (T2, R * R), loose=True,
                  wide=T2 < 10000)


@pytest.mark.parametrize("G", [1, 2, 8])
def test_shared_textures(G):
    fv, tex = rs.shared(8, G, "surface", np.float32, seed=G)
    run_scene(fv, tex, 17, True, "shared G=%d" % G, "%d images per texture" % (8 // G), loose=True)


def test_planes_and_scalars():
    fv, tex, near, far = rs.planes(np.float32)
    bg = tuple(float(np.float32(c)) for c in (0.1, 0.7, 0.3))
    for isz, aa in ((33, False), (17, True)):
        run_scene(fv, tex, isz, aa, "planes %s" % _sz(isz, aa), "near %g far %g" % (near, far), loose=True,
                  kw=dict(near=near, far=far, background_color=bg))


def test_65535_images():
    """B = 65535, the forward's gridDim.z and the backward's gridDim.y limit, F = 2, IS = 1 anti-aliased."""
    fv, tex = rs.many_images(65535, seed=7, dtype=np.float32)
    run_scene(fv, tex, 1, True, "B=65535", "65535 images", loose=True, wide=False)


def test_one_tile_list_walks_four_million_pixels():
    """IS = 1024 anti-aliased (S = 2048): 16384 tiles, every one listing the covering face."""
    fv, tex = rs.big(np.float32, seed=5)
    # the float32 oracle sums a face's 4M p2f and texel terms one after another (relative error up to 4M ulps), as in
    # test_raster_gather_range_gpu's IS = 1024 case
    run_scene(fv, tex, 1024, True, "IS=1024 aa", "%d pixels" % (2048 * 2048), loose=True, wide=False, rgbs=("softmax",),
              rtol=1e-3)


# ---------------------------------------------------------------------------------------------------------------------
# the NaN box, with the reference's own CUDA kernels as arbiter
# ---------------------------------------------------------------------------------------------------------------------
def _ref_module():
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "soft_rasterize_ref_nofma.so")
    if not os.path.exists(path):
        return None
    spec = importlib.util.spec_from_file_location("soft_rasterize_ref_nofma", path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


_REF = _ref_module()


def _ref_forward(fv, tex, S, rgb, eps):
    """The reference's forward kernel (-fmad=false build) on device buffers of fv's dtype (float, or double: its
    AT_DISPATCH_FLOATING_TYPES instantiation), the kernels' grid."""
    import torch
    dt = torch.float64 if fv.dtype == np.float64 else torch.float32
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dt)  # noqa: E731
    B, Fn = fv.shape[:2]
    z = lambda *s: torch.zeros(*s, device="cuda", dtype=dt)  # noqa: E731
    faces_info, aggrs, p2f, p2f_sum = z(B, Fn, 27), z(B, 2, S, S), z(B, Fn, 2), z(B, Fn, 2)
    colors = z(B, 4, S, S)
    colors[:, 3] = 1.0
    grid = t(rs.kernel_grid(S, fv.dtype.type))
    args = (1.0, 100.0, eps, KW["sigma_val"], 2, float(np.log(1.0 / KW["dist_eps"] - 1.0)), KW["gamma_val"],
            1 if rgb == "softmax" else 0, 2, 0, True)
    _REF.forward_soft_rasterize(t(fv), t(tex), faces_info, aggrs, grid, p2f, p2f_sum, colors, S, *args)
    torch.cuda.synchronize()
    return dict(colors=colors.cpu().numpy(), aggrs=aggrs.cpu().numpy())


def _planes_bit_exact(got, ref, what):
    for name in ("colors", "aggrs"):
        a, b = got[name], ref[name]
        na, nb = np.isnan(a), np.isnan(b)
        assert np.array_equal(na, nb), "%s %s: %d NaN vs the reference's %d" % (what, name, na.sum(), nb.sum())
        _bits(a[~na], b[~nb], "%s %s: not bit-exact" % (what, name))


@pytest.mark.skipif(_REF is None, reason="oracle/_ref/soft_rasterize_ref_nofma.so not built")
@pytest.mark.parametrize("isz,aa", [(17, False), (33, False), (9, True), (17, True)])
def test_nan_box_against_the_reference_kernels(isz, aa):
    """A face with a NaN vertex (raster_range_scenes.big(nan=True)): the float32 default and deterministic forwards
    against the reference's float kernels, the float64 forward against its double kernels -- every pixel plane bit-exact,
    NaN positions included."""
    S = isz * (2 if aa else 1)
    eps = oracle_eps(KW["gamma_val"])
    for rgb in ("softmax", "hard"):
        kw = dict(aggr_func_rgb=rgb, eps=eps)
        for path, dt in (("default", np.float32), ("det", np.float32), ("f64", np.float64)):
            fv, tex = rs.big(dt, seed=isz, nan=True)
            got = c_render(path, fv, tex, isz, aa, None, kw)
            if not aa:
                got["colors"] = got["images"]
            ref = _ref_forward(fv, tex, S, rgb, eps)
            orc = oracle(path, fv, tex, isz, aa, None, kw)
            print("NaN box %s %s %s: NaN pixels (all planes) ours %d, reference %d, oracle B %d"
                  % (path, _sz(isz, aa), rgb, np.isnan(got["colors"]).sum() + np.isnan(got["aggrs"]).sum(),
                     np.isnan(ref["colors"]).sum() + np.isnan(ref["aggrs"]).sum(),
                     np.isnan(orc["colors"]).sum() + np.isnan(orc["aggrs"]).sum()))
            _planes_bit_exact(got, ref, "NaN box %s %s %s" % (path, _sz(isz, aa), rgb))

