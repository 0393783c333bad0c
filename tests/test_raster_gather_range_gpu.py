"""The float64 rasteriser (umr_raster_*_f64) and the deterministic float32 one (umr_raster_*_deterministic) across their
accepted input range, through their C entry points, against CPU oracle B (float64 for the first, float32 for the second).

Both run the face-parallel gather backward (one warp per face walks its cull box; texel gradients combined with
__match_any_sync) and fixed-point p2f; the float64 forward lists each tile's faces in 1024-face windows.  The scenes of
raster_range_scenes.py reach what the feature scenes of test_raster_f64_gpu / test_deterministic_gpu do not: tile lists
consumed mid-scan, box edges on pixel centres, S = 1 and 2, odd anti-aliased sizes, T2 up to 1449^2 and non-square T2,
shared textures over 8 images, planes that cut faces, B = 65535 and F = 2^24.

The harness (guard bands, prefilled outputs, oracle B, the gates) is raster_range_harness.py.  Each case prints the
count of what it targets and its worst error / bound ratio."""
import math

import numpy as np
import pytest
import torch

import raster_range_scenes as rs
from raster_range_harness import (DEV, KW, TDT, _bits_equal, c_render, compare, oracle, oracle_eps,
                                  oracle_on_the_kernel_grid)  # noqa: F401 (an autouse fixture)
from umr_b200 import _lib, raster

pytestmark = pytest.mark.gpu
SIZES = [(1, False), (2, False), (17, False), (31, False), (33, False), (9, True), (17, True), (33, True)]
PATHS = ["f64", "det"]


def autograd_render(path, fv, tex, isz, aa, g, kw):
    """The same render through raster.soft_rasterize (float64 inputs, or float32 under deterministic algorithms)."""
    dt = TDT[np.float64 if path == "f64" else np.float32]
    k = dict(KW, **kw)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(path == "det")
    try:
        tfv = torch.from_numpy(np.ascontiguousarray(fv)).to(DEV, dt).requires_grad_(g is not None)
        ttex = torch.from_numpy(np.ascontiguousarray(tex)).to(DEV, dt).requires_grad_(g is not None)
        img, p2f, aggr = raster.soft_rasterize(tfv, ttex, isz, anti_aliasing=aa, **k)
        if g is not None:
            img.backward(torch.from_numpy(np.asarray(g)).to(DEV, dt))
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(old)
    out = dict(images=img.detach().cpu().numpy(), aggrs=aggr.cpu().numpy(), p2f=p2f.cpu().numpy())
    if g is not None:
        out["grad_faces"] = tfv.grad.cpu().numpy().reshape(fv.shape[0], -1, 9)
        out["grad_tex"] = ttex.grad.cpu().numpy()
    return out


def run_case(path, fv, tex, isz, aa, kw, what, feature, seed=0, reproduce=True, split=False, rtol=1e-4, loose=False,
             face_floor_shared=False):
    """C-ABI render with guards vs oracle B, twice (bitwise equal), and vs soft_rasterize (bitwise equal)."""
    dt = np.float64 if path == "f64" else np.float32
    fv, tex = fv.astype(dt), tex.astype(dt)
    B = fv.shape[0]
    g = np.random.default_rng(seed).uniform(-1, 1, size=(B, 4, isz, isz)).astype(dt)
    got = c_render(path, fv, tex, isz, aa, g, kw)
    ref = oracle(path, fv, tex, isz, aa, g, kw)
    worst = compare(path, got, ref, kw.get("aggr_func_rgb", "softmax"), what, rtol, loose, face_floor_shared)
    if reproduce:
        _bits_equal(got, c_render(path, fv, tex, isz, aa, g, kw), "%s %s second call" % (path, what))
        auto = autograd_render(path, fv, tex, isz, aa, g, kw)
        _bits_equal(auto, got, "%s %s soft_rasterize" % (path, what))
    if split:
        geo = c_render(path, fv, tex, isz, aa, g, kw, grads=(True, False))
        tx = c_render(path, fv, tex, isz, aa, g, kw, grads=(False, True))
        assert geo["grad_faces"].tobytes() == got["grad_faces"].tobytes() and "grad_tex" not in geo
        assert tx["grad_tex"].tobytes() == got["grad_tex"].tobytes() and "grad_faces" not in tx
    print("%s %s: %s; worst error/bound %.3g" % (path, what, feature, worst))
    return got, ref


def _sz(isz, aa):
    return "IS=%d aa" % isz if aa else "S=%d" % isz


# ---------------------------------------------------------------------------------------------------------------------
# crowds: tile lists consumed mid-scan
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("isz,aa", SIZES)
@pytest.mark.parametrize("name", sorted(rs.CROWDS))
def test_crowd(name, isz, aa, path):
    S = isz * (2 if aa else 1)
    dt = np.float64 if path == "f64" else np.float32
    fv, tex, hit = rs.crowd(rs.CROWDS[name], S, dt, seed=len(name) + S)
    counts = rs.window_hits(rs.boxes(fv[0], dt), S, dt)
    assert counts == rs.CROWDS[name]
    for rgb in ("softmax", "hard"):
        kw = dict(aggr_func_rgb=rgb, eps=oracle_eps(KW["gamma_val"]))
        got, _ = run_case(path, fv, tex, isz, aa, kw, "crowd %s %s %s" % (name, _sz(isz, aa), rgb),
                          "consumes at n = %s" % rs.consumes(counts), reproduce=rgb == "softmax")
        if rgb == "hard":   # the listed faces win pixels, and ties went to the lower index (bit-exact face-id plane above)
            ids = got["aggrs"][:, 1]
            assert np.isin(ids[ids >= 0], hit).all() and (ids >= 0).any()


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("isz,aa", [(1, False), (17, True)])
def test_crowd_of_65535_faces(isz, aa, path):
    S = isz * (2 if aa else 1)
    dt = np.float64 if path == "f64" else np.float32
    fv, tex = rs.crowd_all(S, dt, seed=S)
    counts = rs.window_hits(rs.boxes(fv[0], dt), S, dt)
    for rgb in ("softmax", "hard"):
        kw = dict(aggr_func_rgb=rgb, eps=oracle_eps(KW["gamma_val"]))
        run_case(path, fv, tex, isz, aa, kw, "65535 faces in one tile %s %s" % (_sz(isz, aa), rgb),
                 "%d consumes" % len(rs.consumes(counts)), reproduce=False)


# ---------------------------------------------------------------------------------------------------------------------
# box edges on pixel centres, boxes over and off the raster
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("isz,aa", SIZES)
def test_edges(isz, aa, path):
    """Barycentric distance keeps the pixels on each box edge alive (raster_range_scenes.edge_pixels_alive), so the
    forward's tile and pixel box tests and the backward's spans decide them; euclidean (where the edge pixel sits at the
    distance cut-off) and hard as well.  This case found the backward spans dropping pixel 0 when a box's upper edge
    lies exactly on its centre and rounding puts the edge's index just below 0 (det_span / box_span)."""
    S = isz * (2 if aa else 1)
    dt = np.float64 if path == "f64" else np.float32
    fv, tex, meta = rs.edges(S, dt, seed=S)
    for dist, rgb in (("barycentric", "softmax"), ("euclidean", "softmax"), ("barycentric", "hard")):
        kw = dict(dist_func=dist, aggr_func_rgb=rgb, eps=oracle_eps(KW["gamma_val"]))
        run_case(path, fv, tex, isz, aa, kw, "edges %s %s %s" % (_sz(isz, aa), dist, rgb),
                 "%d box sides on a pixel centre, %d one step beside" % ((meta[:, 2] == 0).sum(), (meta[:, 2] != 0).sum()),
                 reproduce=dist == "euclidean")


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("isz,aa", SIZES)
def test_big_boxes(isz, aa, path):
    dt = np.float64 if path == "f64" else np.float32
    for nan in (False, True):
        fv, tex = rs.big(dt, seed=isz, nan=nan)
        for rgb in ("softmax", "hard"):
            kw = dict(aggr_func_rgb=rgb, eps=oracle_eps(KW["gamma_val"]))
            got, _ = run_case(path, fv, tex, isz, aa, kw, "big%s %s %s" % (" + NaN box" if nan else "", _sz(isz, aa), rgb),
                              "%d faces" % fv.shape[1], reproduce=not nan, split=not nan and rgb == "softmax", loose=True)
            if not nan:
                assert np.abs(got["grad_tex"][0, :1]).max() > 0 or (isz == 1 and rgb == "hard")  # covering face reached
                assert not np.abs(got["grad_faces"][0, 1:5]).any()          # the off-raster faces have no pixel


# ---------------------------------------------------------------------------------------------------------------------
# textures
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("T2", [1, 2, 3, 5, 8, 36, 1449 ** 2])
def test_textures(T2, path):
    """T2 = 1: every lane of a warp on one texel; 1449^2: every lane on its own; non-square T2: NaN in the texels at
    index R^2 and above, which must never be read (no NaN in the images) and keep a zero gradient."""
    dt = np.float64 if path == "f64" else np.float32
    R = math.isqrt(T2)
    fv, tex = rs.textured(T2, dt, seed=T2 % 1000)
    for isz, aa in ((17, True), (33, False)):
        S = isz * (2 if aa else 1)
        seg = rs.texels_per_segment(fv[0, 0].astype(np.float64), S, T2)
        for rgb in ("softmax", "hard"):
            kw = dict(aggr_func_rgb=rgb, eps=oracle_eps(KW["gamma_val"]))
            got, _ = run_case(path, fv, tex, isz, aa, kw, "T2=%d %s %s" % (T2, _sz(isz, aa), rgb),
                              "distinct texels per 32-lane segment %d..%d" % (min(d for _, d in seg), max(d for _, d in seg)),
                              reproduce=rgb == "softmax" and T2 < 10000, split=rgb == "softmax" and T2 == 1, loose=True)
            assert not np.isnan(got["images"]).any()
            assert not got["grad_tex"][:, :, R * R:].any()
            assert np.abs(got["grad_tex"][:, :, :R * R]).max() > 0


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("textype", ["surface", "vertex"])
@pytest.mark.parametrize("G", [1, 2, 8])
def test_shared_textures(G, textype, path):
    """B = 8 renders, G texture groups: one backward warp walks B / G images in turn."""
    fv, tex = rs.shared(8, G, textype, seed=G)
    for rgb in ("softmax", "hard"):
        kw = dict(aggr_func_rgb=rgb, texture_type=textype, eps=oracle_eps(KW["gamma_val"]))
        run_case(path, fv, tex, 17, True, kw, "shared G=%d %s %s" % (G, textype, rgb), "%d images per warp" % (8 // G),
                 reproduce=rgb == "softmax", split=rgb == "softmax", loose=True)


# ---------------------------------------------------------------------------------------------------------------------
# planes and scalars
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", PATHS)
def test_planes_and_scalars(path):
    """near = 3 and far = 6 cut faces; faces of constant depth 4 and 6 put covered pixels exactly on a depth and on the far
    plane; a background inexact in float (the kernels take it as float, so the oracle is handed the same floats) and a
    non-dyadic eps."""
    dt = np.float64 if path == "f64" else np.float32
    fv, tex, near, far = rs.planes(dt)
    bg = tuple(float(np.float32(c)) for c in (0.1, 0.7, 0.3))
    for isz, aa in ((33, False), (17, True)):
        for rgb in ("softmax", "hard"):
            kw = dict(aggr_func_rgb=rgb, near=near, far=far, background_color=bg, eps=oracle_eps(KW["gamma_val"]))
            got, ref = run_case(path, fv, tex, isz, aa, kw, "planes %s %s" % (_sz(isz, aa), rgb), "", reproduce=rgb == "softmax",
                                loose=True)
            if rgb == "hard":
                on_far = int((ref["aggrs"][:, 0] == far).sum())
                assert on_far > 0 and int((ref["aggrs"][:, 0] == 4.0).sum()) > 0
                print("  %d pixels at depth exactly far = %g" % (on_far, far))


# ---------------------------------------------------------------------------------------------------------------------
# limits
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", PATHS)
def test_65535_images(path):
    """B = 65535, the forward's gridDim.z and the backward's gridDim.y limit, F = 2, IS = 1 anti-aliased."""
    fv, tex = rs.many_images(65535, seed=7)
    for rgb in ("softmax", "hard"):
        kw = dict(aggr_func_rgb=rgb, eps=oracle_eps(KW["gamma_val"]))
        got, _ = run_case(path, fv, tex, 1, True, kw, "B=65535 %s" % rgb, "65535 images", reproduce=False, loose=True,
                          face_floor_shared=True)
        assert np.abs(got["grad_tex"][-1]).max() > 0 and (rgb == "hard" or np.abs(got["grad_faces"][-1]).max() > 0)


@pytest.mark.parametrize("path", PATHS)
def test_max_faces(path):
    """F = 2^24: six faces on screen (indices 0, 1023, 1024, 2^23, F - 2, F - 1), every other far off it.  Only the
    on-screen faces go to the oracle (re-indexed); every other face must get p2f = 0 and a zero gradient."""
    F = raster_max_faces()
    dt = np.float64 if path == "f64" else np.float32
    lib = _lib.load()
    ws = (lib.umr_raster_workspace_bytes_f64 if path == "f64" else lib.umr_raster_workspace_bytes_deterministic)(1, F, 8, 1)
    it = np.dtype(dt).itemsize
    need = ws + F * it * (9 + 3 + 2 + 9 + 3)   # workspace, then vertices, textures, p2f and the two gradients
    free = torch.cuda.mem_get_info()[0]
    if free < 2 * need:
        pytest.skip("F = 2^24 needs %.1f GB of device memory (twice the %.1f GB computed), %.1f GB free"
                    % (2 * need / 2 ** 30, need / 2 ** 30, free / 2 ** 30))
    on = np.array([0, 1023, 1024, 1 << 23, F - 2, F - 1])
    rng = np.random.default_rng(3)
    fv = np.empty((1, F, 9), dt)
    fv[:] = rs.OFF.astype(dt)
    small = np.array([[-0.6 + 0.1 * j, -0.5, 3.0 + j, 0.7, -0.4 + 0.05 * j, 4.0 + j, -0.1 * j, 0.8, 5.0 - j * 0.3]
                      for j in range(len(on))])
    fv[0, on] = small
    tex = np.full((1, F, 1, 3), 0.5, dt)
    tex[0, on] = rng.uniform(0, 1, size=(len(on), 1, 3))
    isz = 8
    g = rng.uniform(-1, 1, size=(1, 4, isz, isz)).astype(dt)
    for rgb in ("softmax", "hard"):
        kw = dict(aggr_func_rgb=rgb, eps=oracle_eps(KW["gamma_val"]))
        got = c_render(path, fv, tex, isz, True, g, kw)
        ref = oracle(path, fv[:, on], tex[:, on], isz, True, g, kw)
        if rgb == "hard":   # re-index the oracle's face ids
            ids = ref["aggrs"][:, 1]
            ref["aggrs"][:, 1] = np.where(ids >= 0, on[np.maximum(ids, 0).astype(np.int64)], ids)
        sub = {k: (v[:, on] if k in ("p2f", "grad_faces", "grad_tex") else v) for k, v in got.items() if k != "t_bwd"}
        worst = compare(path, sub, ref, rgb, "F=2^24 %s" % rgb)
        off = np.ones(F, bool)
        off[on] = False
        assert not got["p2f"][0, off].any() and not got["grad_faces"][0, off].any() and not got["grad_tex"][0, off].any()
        assert np.abs(got["grad_faces"][0, F - 1]).max() > 0
        print("%s F=2^24 %s: %d faces on screen; worst error/bound %.3g" % (path, rgb, len(on), worst))


def raster_max_faces():
    return 1 << 24   # UMR_RASTER_MAX_FACES


@pytest.mark.parametrize("path", PATHS)
def test_one_warp_walks_four_million_pixels(path):
    """IS = 1024 anti-aliased (S = 2048) with the raster-covering face: one backward warp walks 4M pixels."""
    fv, tex = rs.big(np.float64, seed=5)
    kw = dict(eps=oracle_eps(KW["gamma_val"]))
    # the float32 oracle sums a face's 4M p2f and texel terms one after another (relative error up to 4M ulps)
    got, _ = run_case(path, fv, tex, 1024, True, kw, "IS=1024 aa", "%d pixels in the covering face's walk" % (2048 * 2048),
                      reproduce=False, rtol=1e-3, loose=True)
    print("%s IS=1024 aa: backward %.1f ms (one call, host clock around a synchronised launch)" % (path, 1e3 * got["t_bwd"]))


def test_part_map_on_the_deterministic_path():
    """4 colour channels (UMR's part maps): each colour plane equals the 3-channel render of that channel."""
    fv, _ = rs.big(np.float32, seed=2)
    rng = np.random.default_rng(4)
    tex4 = rng.uniform(0, 1, size=(1, fv.shape[1], 4, 4)).astype(np.float32)
    kw = dict(background_color=(0.0, 0.0, 0.0, 0.0), eps=oracle_eps(KW["gamma_val"]))
    got = c_render("det", fv, tex4, 17, True, None, dict(kw, background_extra=0.0), nc=4)
    again = c_render("det", fv, tex4, 17, True, None, dict(kw, background_extra=0.0), nc=4)
    _bits_equal(got, again, "part map second call")
    kw3 = dict(eps=kw["eps"])
    a = oracle("det", fv, tex4[..., :3], 17, True, None, kw3)
    b = oracle("det", fv, tex4[..., [3, 0, 1]], 17, True, None, kw3)
    ref = dict(images=np.concatenate([a["images"][:, :3], b["images"][:, :1], a["images"][:, 3:]], 1), aggrs=a["aggrs"],
               p2f=a["p2f"])
    worst = compare("det", {k: got[k] for k in ("images", "aggrs", "p2f")}, ref, "softmax", "part map", loose=True)
    print("det part map IS=17 aa: 4 channels; worst error/bound %.3g" % worst)


def test_one_pixel_on_the_default_path():
    """S = 1 on the default float32 path: the grid is (-1, -1), so p2f is finite."""
    fv, tex = rs.big(np.float32, seed=1)
    g = np.random.default_rng(0).uniform(-1, 1, size=(1, 4, 1, 1)).astype(np.float32)
    kw = dict(eps=1e-3)
    tfv = torch.from_numpy(fv).to(DEV).requires_grad_(True)
    ttex = torch.from_numpy(tex).to(DEV).requires_grad_(True)
    img, p2f, aggr = raster.soft_rasterize(tfv, ttex, 1, **dict(KW, **kw))
    img.backward(torch.from_numpy(g).to(DEV))
    got = dict(images=img.detach().cpu().numpy(), aggrs=aggr.cpu().numpy(), p2f=p2f.cpu().numpy(),
               grad_faces=tfv.grad.cpu().numpy().reshape(1, -1, 9), grad_tex=ttex.grad.cpu().numpy())
    assert np.isfinite(got["p2f"]).all() and (got["p2f"][0, 0] == -1).all()
    ref = oracle("det", fv, tex, 1, False, g, kw)
    worst = compare("det", got, ref, "softmax", "default path S=1", loose=True)
    print("default S=1: p2f of the covering face %s; worst error/bound %.3g" % (got["p2f"][0, 0], worst))


@pytest.mark.parametrize("isz,aa", [(17, True), (33, False)])
def test_f64_inputs_at_an_element_offset(isz, aa):
    """float64 views at an odd element offset (8-byte aligned, not 16): every read of a caller buffer in raster_f64.cu is
    scalar, so the render is bitwise the aligned one."""
    fv, tex = rs.big(np.float64, seed=9)
    g = np.random.default_rng(1).uniform(-1, 1, size=(1, 4, isz, isz))
    kw = dict(KW, eps=1e-3)

    def run(offset):
        def at(a):
            t = torch.empty(a.size + offset, dtype=torch.float64, device=DEV)
            v = t[offset:].view(a.shape)
            v.copy_(torch.from_numpy(a))
            return v
        tfv, ttex, tg = at(fv).requires_grad_(True), at(tex).requires_grad_(True), at(g)
        assert tfv.data_ptr() % 16 == 8 * (offset % 2)
        img, p2f, aggr = raster.soft_rasterize(tfv, ttex, isz, anti_aliasing=aa, **kw)
        img.backward(tg)
        torch.cuda.synchronize()
        return [x.detach().cpu().numpy().tobytes() for x in (img, p2f, aggr, tfv.grad, ttex.grad)]
    assert run(1) == run(0)
