"""The hard visibility render (umr_raster_visibility) across its accepted input range, through its C entry point,
against CPU oracle B, the hard-mode umr_raster_forward and, where they were built, the reference's own CUDA kernels.

MultiTextureLoss runs this render on every training step and keeps only which faces win a pixel.  Its three output
combinations take different kernels:
  planes  aggrs_info only: k_raster_fwd3<2> writes (depth_min, float(face_index_min)) per raster pixel;
  bytes   visible_faces only: k_visible_faces, face-parallel, one CTA per 64 x 64 bin, a pixel box per face and packed
          (depth bits << 32 | face) keys kept by atomicMin;
  both    k_raster_fwd3<2> writing the planes and the bytes.
Each scene runs all three, with 16-bit face indices and again behind PAD = 65537 off-screen faces (32-bit indices,
ids mapped back), and the planes 16-byte aligned (vectorised stores at anti-aliased S % 8 == 0) and 4 bytes past a
boundary (scalar stores).  face_vertices, the planes, the bytes and the workspace sit between guard bands; the bytes
start non-zero, so the call must clear them.

Checks:
  planes  bit-exact (NaN positions included) against oracle B's hard-mode aggrs_info, the hard-mode umr_raster_forward
          on the same inputs and, when oracle/_ref/soft_rasterize_ref_nofma.so exists, the reference's kernels;
  bytes   exactly the ids of oracle B's face-index plane, with the background's -1 marking face F - 1, from both kernels
          that write bytes; a second call bitwise equal;
  texcycle on some scenes, the TexCycle loss from the bytes has the bits of the loss from the plane.

Scenes: the range scenes (coarse-bin box edges, crowded tile lists, the NaN box, a face window crossed, B = 65535,
IS = 1024 anti-aliased, needles and coincident corners), and raster_range_scenes' visibility scenes: boxes reaching
past the int32 range of k_visible_faces' pixel index, the thin-face switch, depth ties, zero and negative depths, the
initial depth cut, near > far, single-sided rendering and small shapes."""
import ctypes

import numpy as np
import pytest
import torch

import raster_range_scenes as rs
from raster_range_harness import (NULL, Banded, BandedBytes, Workspace, _stream, c_render, oracle,
                                  oracle_on_the_kernel_grid, params)  # noqa: F401 (an autouse fixture)
from test_raster_fast_range_gpu import _REF
from umr_b200 import _lib
from util import scene

pytestmark = pytest.mark.gpu
PAD = 65537        # off-screen faces put in front for the 32-bit face-index run
PAD_MAX_B = 64     # renders of at most this many images also run behind PAD


def c_visibility(fv, isz, aa, kw, planes, faces, skew=0):
    """umr_raster_visibility with guard bands; returns (planes [B, 2, S, S] or None, bytes [B, F] or None)."""
    lib = _lib.load()
    B, F = fv.shape[:2]
    S = isz * (2 if aa else 1)
    p = params(B, F, 1, isz, aa, kw)
    fvb = Banded(np.float32, array=fv)
    ws = Workspace(lib.umr_raster_workspace_bytes(B, F, isz, 1 if aa else 0))
    aggrs = Banded(np.float32, (B, 2, S, S), skew=skew) if planes else None
    vis = BandedBytes((B, F)) if faces else None
    _lib.check(lib.umr_raster_visibility(fvb.ptr(), aggrs.ptr() if planes else NULL, vis.ptr() if faces else NULL,
                                         ctypes.byref(p), ws.ptr(), _stream()), "umr_raster_visibility")
    torch.cuda.synchronize()
    fvb.check("face_vertices", False)
    ws.check()
    out = [None, None]
    if planes:
        aggrs.check("aggrs_info", True)
        out[0] = aggrs.numpy()
    if faces:
        vis.check("visible_faces")
        out[1] = vis.numpy()
    return out


def _ref_planes(fv, S, kw):
    """The reference's forward kernel (-fmad=false build) in hard mode: aggrs_info."""
    B, F = fv.shape[:2]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to("cuda", torch.float32)  # noqa: E731
    z = lambda *s: torch.zeros(*s, device="cuda", dtype=torch.float32)  # noqa: E731
    faces_info, aggrs, p2f, p2f_sum, colors = z(B, F, 27), z(B, 2, S, S), z(B, F, 2), z(B, F, 2), z(B, 4, S, S)
    colors[:, 3] = 1.0
    k = dict(dict(rs.KW, near=1.0, far=100.0, fill_back=True), **kw)
    args = (k["near"], k["far"], 1e-3, k["sigma_val"], 2, float(np.log(1.0 / k["dist_eps"] - 1.0)), k["gamma_val"], 0, 2, 0,
            bool(k["fill_back"]))
    _REF.forward_soft_rasterize(t(fv), z(B, F, 1, 3), faces_info, aggrs, t(rs.kernel_grid(S, np.float32)), p2f, p2f_sum,
                                colors, S, *args)
    torch.cuda.synchronize()
    return aggrs.cpu().numpy()


def _bits(a, b, what):
    na, nb = np.isnan(a), np.isnan(b)
    assert np.array_equal(na, nb), "%s: NaN at %d vs %d elements" % (what, na.sum(), nb.sum())
    diff = np.flatnonzero(a.view(np.int32) != b.view(np.int32))
    assert diff.size == 0, "%s: %d elements differ, first at %s: %r vs %r" % (
        what, diff.size, np.unravel_index(diff[0], a.shape), a.flat[diff[0]], b.flat[diff[0]])


def expected_bytes(ids, F):
    """[B, F] bytes of the ids in face-index planes [B, S, S]: -1 (background) marks face F - 1."""
    B = ids.shape[0]
    want = np.zeros((B, F), np.uint8)
    for b in range(B):
        u = np.unique(ids[b]).astype(np.int64)
        want[b, np.where(u < 0, F - 1, u)] = 1
    return want


def _unpad(planes, P):
    """Face ids of a render behind P off-screen faces mapped back to the scene's."""
    out = planes.copy()
    ids = out[:, 1]
    assert not ((ids >= 0) & (ids < P)).any(), "an off-screen face won a pixel"
    out[:, 1] = np.where(ids >= 0, ids - P, ids)
    return out


def _texcycle(planes, vis, F, seed=0):
    """The deterministic TexCycle loss from the face-index plane and from the bytes (bits of each)."""
    lib = _lib.load()
    B = planes.shape[0]
    rng = np.random.default_rng(seed)
    T2 = 4
    flow = torch.from_numpy(rng.uniform(-1, 1, size=(B, F, T2, 2)).astype(np.float32)).cuda()
    prob = torch.from_numpy(rng.uniform(-1, 1, size=(B, F, 2)).astype(np.float32)).cuda()
    ws = torch.empty(lib.umr_texcycle_workspace_bytes_deterministic(B, F), dtype=torch.uint8, device="cuda")
    out = []
    for ids, v in ((torch.from_numpy(np.ascontiguousarray(planes[:, 1])).cuda(), torch.empty(B, F, dtype=torch.uint8, device="cuda")),
                   (None, torch.from_numpy(vis).cuda())):
        loss = torch.empty(1, device="cuda")
        P = int(planes.shape[2] * planes.shape[3])
        _lib.check(lib.umr_texcycle_forward_deterministic(
            flow.data_ptr(), prob.data_ptr(), ids.data_ptr() if ids is not None else None, v.data_ptr(), loss.data_ptr(),
            B, F, T2, P if ids is not None else 0, ws.data_ptr(), _stream()), "umr_texcycle_forward_deterministic")
        torch.cuda.synchronize()
        out.append((loss.cpu().numpy().view(np.int32)[0], v.cpu().numpy()))
    return out


def run_vis(fv, isz, aa, what, kw=None, wide=True, consumer=False, expect=None, ref_skip=()):
    """Every output combination of umr_raster_visibility on one scene (and, with wide, behind PAD off-screen faces)
    against oracle B, the hard-mode forward and the reference's kernels (except on the images ref_skip).
    expect(ids [B, S, S], want [B, F]): the scene's own assertions on oracle B's answer.  Returns oracle B's planes."""
    fv = np.ascontiguousarray(fv, np.float32)
    B, F = fv.shape[:2]
    S = isz * (2 if aa else 1)
    k = dict(dict(aggr_func_rgb="hard", eps=1e-3), **(kw or {}))
    tex = np.zeros((B, F, 1, 3), np.float32)
    orc = oracle("det", fv, tex, isz, aa, None, k)["aggrs"]
    want = expected_bytes(orc[:, 1], F)
    if expect is not None:
        expect(orc[:, 1], want)
    if _REF is not None:
        keep = [b for b in range(B) if b not in ref_skip]
        _bits(_ref_planes(fv[keep], S, {n: k[n] for n in ("near", "far", "fill_back") if n in k}), orc[keep],
              "%s: the reference's kernels against oracle B" % what)
    pads = (0, PAD) if wide and B <= PAD_MAX_B and F <= 65535 else (0,)
    for P in pads:
        tag = "%s%s" % (what, " F=%d" % (P + F) if P or F > 65535 else "")
        if P:
            pv = np.concatenate([np.broadcast_to(rs.OFF.astype(np.float32), (B, P, 9)), fv], 1)
        else:
            pv = fv
        unpad = (lambda a: _unpad(a, P)) if P else (lambda a: a)
        fwd = c_render("default", pv, np.zeros((B, P + F, 1, 3), np.float32), isz, aa, None, k)
        _bits(unpad(fwd["aggrs"]), orc, tag + ": hard-mode umr_raster_forward against oracle B")
        for skew in (0, 1):
            planes, _ = c_visibility(pv, isz, aa, k, True, False, skew)
            _bits(unpad(planes), orc, "%s planes (skew %d): against oracle B" % (tag, skew))
            both, vb = c_visibility(pv, isz, aa, k, True, True, skew)
            _bits(unpad(both), orc, "%s both (skew %d): planes against oracle B" % (tag, skew))
            assert not vb[:, :P].any(), "%s both: an off-screen face marked" % tag
            bad = np.argwhere(vb[:, P:] != want)
            assert bad.size == 0, "%s both (k_raster_fwd3<2>): %d bytes differ, first (image, face, got, want) %s" % (
                tag, len(bad), [(int(b), int(f), int(vb[b, P + f]), int(want[b, f])) for b, f in bad[:6]])
        _, vis = c_visibility(pv, isz, aa, k, False, True)
        assert not vis[:, :P].any(), "%s bytes: an off-screen face marked" % tag
        bad = np.argwhere(vis[:, P:] != want)
        assert bad.size == 0, "%s bytes (k_visible_faces): %d bytes differ, first (image, face, got, want) %s" % (
            tag, len(bad), [(int(b), int(f), int(vis[b, P + f]), int(want[b, f])) for b, f in bad[:6]])
        _, again = c_visibility(pv, isz, aa, k, False, True)
        assert again.tobytes() == vis.tobytes(), "%s bytes: a second call differs" % tag
        if consumer and not P:
            (l_plane, v_plane), (l_bytes, _) = _texcycle(orc, vis, F)
            assert v_plane.tobytes() == vis.tobytes(), "%s: TexCycle's bytes from the plane differ" % tag
            assert l_plane == l_bytes, "%s: TexCycle loss from the bytes is not the loss from the plane" % tag
        print("%s: %d of %d faces visible, %d background images; planes, bytes and both agree" % (
            tag, int(want.sum()), B * F, int((orc[:, 1] < 0).any(axis=(1, 2)).sum())))
    return orc


def _sz(isz, aa):
    return "IS=%d aa" % isz if aa else "S=%d" % isz


# ---------------------------------------------------------------------------------------------------------------------
# k_visible_faces' pixel box: boxes past the int32 range of its index, and the thin-face switch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("isz,aa", [(64, False), (1024, True)])
def test_far_off_boxes(isz, aa):
    """Faces covering the raster whose box reaches 1/2, 1, 2 and 1000 x 2^32 / S off it, thin (one side at a time)
    and wide (an x and a y side, the tight-box scan at S = 2048 up to factor 1): every face drawn wins the pixels
    oracle B gives it."""
    S = isz * (2 if aa else 1)
    fv, meta = rs.far_faces(S)
    if S > 1024:   # the four factors in turn: 8 images of 2048^2 each
        for fac in rs.FAR_FACTORS:
            sel = [i for i, m in enumerate(meta) if m[3] == fac]
            _far(fv[sel], [meta[i] for i in sel], isz, aa)
    else:
        _far(fv, meta, isz, aa)


def _far(fv, meta, isz, aa):
    def expect(ids, want):
        for i, m in enumerate(meta):
            assert bool(want[i, 0]) == (m[0] == "thin" or m[4] < rs.WIDE_DRAWN), "oracle B: far face %s drawn %s" % (
                m, bool(want[i, 0]))
    run_vis(fv, isz, aa, "far-off boxes %s factors %s" % (_sz(isz, aa), sorted({m[3] for m in meta})), expect=expect,
            consumer=True, ref_skip=_undrawn_wide(meta))


def _undrawn_wide(meta):
    """Renders of a wide face past WIDE_DRAWN.  Oracle B and the kernels draw none of it; the reference's kernels were
    seen to draw a few pixels of such a face (depth 5.0000005) in one run and none in another, so they are no arbiter
    there."""
    return tuple(i for i, m in enumerate(meta) if m[0] == "wide" and m[-1] >= rs.WIDE_DRAWN)


def test_huge_and_infinite_vertices():
    """Vertices at 1e15 and 1e20 (thin faces drawn, wide ones not: at 1e20 x y overflows float32) and +-inf (absent)."""
    fv, meta = rs.huge_faces()

    def expect(ids, want):
        for i, m in enumerate(meta):
            assert bool(want[i, 0]) == (m[0] == "thin"), "far face %s: oracle B draws it %s" % (m, bool(want[i, 0]))
    for isz, aa in ((64, False), (33, True)):
        run_vis(fv, isz, aa, "huge vertices %s" % _sz(isz, aa), expect=expect, ref_skip=_undrawn_wide(meta))


@pytest.mark.parametrize("isz,aa", [(64, False), (65, False), (63, True), (500, True)])
def test_thin_face_switch(isz, aa):
    """Sliver pairs whose smallest-angle sine lies one float step either side of k_prep's bit-4 cut, each over a row
    or column of pixels to near the far ends of its box."""
    S = isz * (2 if aa else 1)
    fv, thin = rs.thin_switch(S)

    def expect(ids, want):
        assert want[0].all(), "oracle B does not draw every sliver: %s" % want[0].tolist()
    run_vis(fv, isz, aa, "thin switch %s" % _sz(isz, aa), expect=expect)


# ---------------------------------------------------------------------------------------------------------------------
# depth order and depth range
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("isz,aa", [(64, False), (33, True)])
def test_depth_order(isz, aa):
    """Repeated faces, faces one float ulp apart in depth (both orders), shared edges through pixel centres, vertices on
    pixel centres."""
    S = isz * (2 if aa else 1)
    fv, names = rs.depth_order(S)

    def expect(ids, want):
        r = names.index("repeat")
        assert want[r, 1] and not want[r, [2, 4]].any(), "repeat: the lowest index of the copies must win"
        assert want[names.index("edge"), :4].all(), "edge: every half of both diamonds wins pixels"
    # the shared-edge render: on a pixel centre where k_prep's inverse gives a barycentric of exactly 0, the reference's
    # own kernels may round it otherwise (2 of 4356 plane elements at IS = 33 anti-aliased); oracle B states the
    # kernels' arithmetic and is the arbiter there
    run_vis(fv, isz, aa, "depth order %s" % _sz(isz, aa), expect=expect, consumer=True, ref_skip=(names.index("edge"),))


def test_zero_depths_at_near_zero():
    """near = 0: a face at depth +0 and the same face at -0, both orders: the lower index wins every pixel."""
    fv = rs.zero_depths()

    def expect(ids, want):
        assert want[:, 0].all() and not want[:, 1].any(), "oracle B: +0 and -0 are one depth, the lower index wins"
    for isz, aa in ((64, False), (33, True)):
        run_vis(fv, isz, aa, "+-0 %s" % _sz(isz, aa), kw=dict(near=0.0), expect=expect, consumer=True)


def test_negative_near():
    fv = rs.negative_depths()
    for isz, aa in ((64, False), (33, True)):
        run_vis(fv, isz, aa, "near -5 %s" % _sz(isz, aa), kw=dict(near=-5.0, far=5.0))


def test_initial_depth_cut():
    """far = 1e9: depth 1e7 does not beat the z-buffer's initial depth_min, the float below it does."""
    fv = rs.depth_cut()
    for isz, aa in ((64, False), (33, True)):
        run_vis(fv, isz, aa, "depth cut %s" % _sz(isz, aa), kw=dict(far=1e9))


def test_near_above_far():
    """near > far: no pair passes the depth test, every pixel is background and only face F - 1 is marked."""
    fv, _ = rs.big(np.float32, seed=3)

    def expect(ids, want):
        assert (ids < 0).all() and want[0].tolist() == [0] * (fv.shape[1] - 1) + [1]
    for isz, aa in ((17, False), (33, True)):
        run_vis(fv, isz, aa, "near > far %s" % _sz(isz, aa), kw=dict(near=5.0, far=2.0), expect=expect)


def test_single_sided():
    """fill_back = False: back faces never win, however near."""
    fv = rs.front_back(seed=4)
    for isz, aa in ((64, False), (33, True)):
        run_vis(fv, isz, aa, "single-sided %s" % _sz(isz, aa), kw=dict(fill_back=False), consumer=True)


# ---------------------------------------------------------------------------------------------------------------------
# small shapes and the range scenes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F", [1, 2])
def test_one_and_two_faces(F):
    fv = rs.small(F, seed=F)
    for isz, aa in ((1, False), (17, False), (9, True)):
        run_vis(fv, isz, aa, "F=%d %s" % (F, _sz(isz, aa)))


@pytest.mark.parametrize("S", [1, 63, 65, 127, 1000])
def test_partial_bins(S):
    fv, _ = scene(2, 2, 1, seed=S)
    run_vis(fv, S, False, "mesh S=%d" % S, consumer=S < 1000)


def test_65535_images_at_s2():
    fv, _ = rs.many_images(65535, seed=9, dtype=np.float32)
    run_vis(fv, 1, True, "B=65535 IS=1 aa", wide=False)


@pytest.mark.parametrize("isz,aa", [(17, False), (33, False), (17, True), (33, True), (64, False)])
def test_edges(isz, aa):
    """Box edges on pixel centres and one step beside them, at the 63 | 64 coarse-bin boundary among others."""
    S = isz * (2 if aa else 1)
    fv, _, _ = rs.edges(S, np.float32, seed=S, fast=True)
    run_vis(fv, isz, aa, "edges %s" % _sz(isz, aa))


@pytest.mark.parametrize("n", rs.LIST_LENGTHS)
def test_tile_list_lengths(n):
    """n one-pixel faces on tile (0, 0), every fifth a repeat of an earlier one: the face counter hands them out."""
    fv, _ = rs.crowd_all(34, np.float32, seed=n, F=n)
    run_vis(fv, 17, True, "list of %d" % n, wide=n < 65535)


def test_nan_box():
    for nan in (False, True):
        fv, _ = rs.big(np.float32, seed=2, nan=nan)
        for isz, aa in ((17, False), (33, True), (64, False)):
            run_vis(fv, isz, aa, "big%s %s" % (" + NaN" if nan else "", _sz(isz, aa)))


def test_face_window_crossing():
    fv, _, on = rs.window_crossing()
    run_vis(fv, 17, True, "window crossing", wide=False)


def test_raster_of_2048():
    """IS = 1024 anti-aliased: 32 x 32 bins of k_visible_faces, 16-byte-aligned vectorised plane stores."""
    fv, _ = rs.big(np.float32, seed=5)
    run_vis(fv, 1024, True, "IS=1024 aa big", wide=False)
    fv, _ = scene(2, 3, 1, seed=11)
    run_vis(fv, 1024, True, "IS=1024 aa mesh", wide=False, consumer=True)


@pytest.mark.parametrize("B,subdiv,isz,aa", [(2, 3, 64, True), (1, 2, 37, True), (2, 2, 48, False)])
def test_needles_and_coincident_corners(B, subdiv, isz, aa):
    """Every 7th face a needle, every 21st a triangle with two coincident corners (both take the whole-cull-box scan)."""
    fv, _ = scene(B, subdiv, 1, seed=3 + isz)
    fv = fv.copy().reshape(B, -1, 3, 3)
    t = np.float32(1e-6)
    fv[:, ::7, 2, :2] = (fv[:, ::7, 0, :2] + fv[:, ::7, 1, :2]) * np.float32(0.5) + t
    fv[:, ::21, 2] = fv[:, ::21, 1]
    run_vis(np.ascontiguousarray(fv.reshape(B, -1, 9)), isz, aa, "slivers B=%d %s" % (B, _sz(isz, aa)), consumer=True)
