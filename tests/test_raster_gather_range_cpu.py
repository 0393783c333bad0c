"""The range scenes of test_raster_gather_range_gpu.py have the properties they claim (no GPU): per-window tile-list hit
counts and consume points, box edges exactly on (or one ulp beside) pixel centres, lanes per texel, the S = 1 grid, the
float64 and deterministic workspace formulas, and the size refusals of both entry-point families."""
import ctypes
import math

import numpy as np
import pytest

import softras
import raster_range_scenes as rs
from umr_b200 import _lib

SIZES = [1, 2, 17, 31, 33, 18, 34, 66]   # raster sides: S, and 2 * IS for the anti-aliased IS = 9, 17, 33
DTYPES = [np.float64, np.float32]
UMR_ERR_TOO_LARGE = -3


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("S", SIZES)
@pytest.mark.parametrize("name", sorted(rs.CROWDS))
def test_crowd_window_hits(name, S, dtype):
    counts = rs.CROWDS[name]
    fv, _, hit = rs.crowd(counts, S, dtype)
    box = rs.boxes(fv[0], dtype)
    assert rs.window_hits(box, S, dtype) == counts
    assert np.array_equal(np.flatnonzero(rs.tile_hits(box, S, 0, 0, dtype)), hit)
    tiles = (S + 15) // 16
    for tx in range(tiles):   # the crowd lists in tile (0, 0) only
        for ty in range(tiles):
            if tx or ty:
                assert not rs.tile_hits(box, S, tx, ty, dtype).any()
    # every scan branch: a continue, a consume before the last window, a window after a consume, a full list
    want = {"1024+1": [1025], "1+1024+1": [1025, 1], "1024+1024+5": [2048, 5], "1000+30+1000": [1030, 1000]}
    assert rs.consumes(counts) == want[name]
    # exact depth ties: repeated faces at different indices (some in different windows)
    _, inv, cnt = np.unique(fv[0, hit], axis=0, return_inverse=True, return_counts=True)
    assert (cnt > 1).sum() >= 10


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("S", [1, 34])
def test_crowd_of_65535_faces_in_one_tile(S, dtype):
    fv, _ = rs.crowd_all(S, dtype)
    assert fv.shape[1] == 65535
    h = rs.window_hits(rs.boxes(fv[0], dtype), S, dtype)
    assert h == [1024] * 63 + [1023]
    assert rs.consumes(h) == [2048] * 31 + [2047]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("S", SIZES)
def test_edges_lie_on_pixel_centres(S, dtype):
    fv, _, meta = rs.edges(S, dtype)
    box = rs.boxes(fv[0], dtype)
    r = rs.cull_radius(dtype)
    assert box.dtype == dtype
    groups = {}
    for f, (side, i, d) in enumerate(meta):
        c = rs.pixel_centre(i, S, dtype)
        e = box[f, side]
        assert np.sign(e - c) == d, (f, side, i, d)
        groups.setdefault((side, i), set()).add(d)
        # the nearest value the edge can take on its side: one vertex step towards the centre crosses or reaches it
        coord = fv[0, f, (side // 2)::3]
        v = coord.min() if side % 2 == 0 else coord.max()
        sign = -1 if side % 2 == 0 else 1
        if d:
            back = np.nextafter(v, dtype(-np.inf) if d > 0 else dtype(np.inf))
            assert np.sign(dtype(back + sign * r) - c) != d
            assert abs(e - c) <= 2 * max(np.spacing(abs(c)), np.spacing(abs(v)))
    # raster columns / rows 0 and S - 1, and the tile boundary 15 | 16 where the raster has one: every side of every
    # target has an edge just below and just above the centre; the raster's end pixels have one exactly on it, and so
    # have most tile-boundary pixels (a centre nearer 0 than r can lie between two steps of the vertex)
    assert {i for _, i in groups} == set(rs.edge_targets(S))
    assert len(groups) == 4 * len(rs.edge_targets(S)) and all({-1, 1} <= g for g in groups.values())
    assert all(0 in g for (_, i), g in groups.items() if i in (0, S - 1))
    exact = sum(0 in g for g in groups.values())
    assert exact >= 0.5 * len(groups)
    # the box decides: the pixel on (or one step beside) every edge survives the barycentric distance cut-off
    alive = [rs.edge_pixels_alive(fv[0, f], side, i, S, dtype) for f, (side, i, _) in enumerate(meta)]
    assert min(alive) >= 1, alive
    print("S=%d %s: %d of %d box sides exactly on a pixel centre" % (S, np.dtype(dtype).name, exact, len(groups)))


def test_pixel_centres_of_the_two_precisions():
    for S in SIZES:
        c64, c32 = rs.pixel_centre(np.arange(S), S, np.float64), rs.pixel_centre(np.arange(S), S, np.float32)
        assert np.array_equal(c64.astype(np.float32), c32)   # one float division of exact integers = the rounded double


def test_big_scene_boxes():
    box = rs.boxes(rs.big(nan=True)[0][0], np.float64)
    assert (box[0, [0, 2]] < -1).all() and (box[0, [1, 3]] > 1).all()   # covers the raster, reaches past every side
    assert box[1, 1] < -1 and box[2, 0] > 1 and box[3, 2] > 1 and box[4, 3] < -1    # off the left, right, top, bottom
    assert np.isfinite(box[6]).all() and box[6, 2] < -0.5 and box[6, 3] > 0.5   # the NaN face: its finite coordinates' box


@pytest.mark.parametrize("S", [17, 33, 66])
def test_lanes_per_texel(S):
    fv, _ = rs.textured(1)
    assert all(d == 1 for _, d in rs.texels_per_segment(fv[0, 0], S, 1))                 # a whole warp on one texel
    fv, _ = rs.textured(1449 ** 2)
    assert all(d == n for n, d in rs.texels_per_segment(fv[0, 0], S, 1449 ** 2))         # every lane on its own texel
    assert max(n for n, _ in rs.texels_per_segment(fv[0, 0], S, 1449 ** 2)) == min(32, S)


@pytest.mark.parametrize("T2", [2, 3, 5, 8])
def test_non_square_textures_hold_nan_past_r_squared(T2):
    _, tex = rs.textured(T2)
    R = math.isqrt(T2)
    assert np.isnan(tex[:, :, R * R:]).all() and np.isfinite(tex[:, :, :R * R]).all()


def test_plane_scene():
    fv, _, near, far = rs.planes()
    z = fv[0, :, 2::3]
    assert (z.min(1) < near).any() and (z.max(1) > far).any()
    assert (z == 4.0).all(1).any() and (z == far).all(1).any()


def test_grid_at_one_pixel_is_minus_one():
    """torch 1.1's affine_grid takes linspace(-1, 1, 1) = [-1] (torch >= 1.3 returns 0 there)."""
    for g in (softras.standard_grid(1), softras.standard_grid(1, np.float64), rs.kernel_grid(1), rs.kernel_grid(1, np.float32)):
        assert g.shape == (1, 1, 2) and (g == -1).all()
    assert np.array_equal(rs.kernel_grid(2), np.array([[[-1, -1], [1, -1]], [[-1, 1], [1, 1]]], np.float64))
    assert np.array_equal(softras.standard_grid(2), rs.kernel_grid(2, np.float32))


def _a(x):
    return (x + 255) // 256 * 256


@pytest.mark.parametrize("B,F,isz,aa", [(1, 1, 1, 0), (3, 7, 9, 1), (16, 1280, 256, 1), (65535, 2, 1, 1), (1, 1 << 24, 8, 1)])
def test_workspace_formulas(lib, B, F, isz, aa):
    n = B * F
    f64 = lib.umr_raster_workspace_bytes_f64(B, F, isz, aa)
    assert f64 == _a(n * 256) + _a(n * 32) + _a(n * 152)      # record, box, p2f limbs: 440 B per (image, face)
    assert n * 440 <= f64 < n * 440 + 3 * 256
    det = lib.umr_raster_workspace_bytes_deterministic(B, F, isz, aa)
    assert det == lib.umr_raster_workspace_bytes(B, F, isz, aa) + _a(n * 104)
    if (B, F) == (1, 1 << 24):
        assert abs(f64 / 2 ** 30 - 6.875) < 1e-3   # 7.4 GB


def _params(B, F, isz, aa):
    p = _lib.UmrRasterParams()
    p.batch_size, p.num_faces, p.texture_size, p.image_size, p.anti_aliasing = B, F, 1, isz, aa
    p.near_plane, p.far_plane, p.eps, p.sigma_val, p.gamma_val, p.dist_eps = 1.0, 100.0, 1e-3, 1e-5, 1e-4, 9.0
    p.func_id_dist, p.func_id_rgb, p.func_id_alpha, p.texture_sample_type, p.double_side = 2, 1, 2, 0, 1
    return p


@pytest.mark.parametrize("B,F,isz,aa", [(65536, 2, 1, 1), (1, 2, 65535 * 16 + 1, 0), (1, 2, 65535 * 8 + 1, 1),
                                        (1, (1 << 24) + 1, 8, 0)])
def test_size_refusals_without_buffers(lib, B, F, isz, aa):
    """The size checks come before the pointer checks, so these calls are refused with NULL buffers."""
    p = ctypes.byref(_params(B, F, isz, aa))
    z = ctypes.c_void_p(0)
    for fn in (lib.umr_raster_forward_f64, lib.umr_raster_forward_deterministic):
        assert fn(z, z, z, z, z, z, p, z, z) == UMR_ERR_TOO_LARGE
    for fn in (lib.umr_raster_backward_f64, lib.umr_raster_backward_deterministic):
        assert fn(z, z, z, z, z, z, z, p, z, z) == UMR_ERR_TOO_LARGE
    ok = _params(65535, 2, 65535 * 8, 1)   # the largest accepted sizes pass the size checks (then refuse the NULLs)
    assert lib.umr_raster_forward_f64(z, z, z, z, z, z, ctypes.byref(ok), z, z) == -2
