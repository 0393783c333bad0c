"""Keypoint transfer without a GPU: the oracle against the reference's definitions, the entry points' refusals through
the .so, the Python argument checks, PCK, and which sampler calls `ops.bilinear_sample` issues for C > 4 channels."""
import contextlib
import ctypes
import os
import re
import types

import numpy as np
import pytest
import torch

import kp_transfer_oracle as ko
from umr_b200 import _lib, ops
from umr_b200.nnutils import kp_transfer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNSUPPORTED, BAD_ARG, TOO_LARGE = -1, -2, -3


# ---------------------------------------------------------------------------------------------------------------------
# oracle
# ---------------------------------------------------------------------------------------------------------------------
def heatmap_per_pixel(kp, sigma, S):
    """draw_labelmap pixel by pixel: (x, y) lies in the window [int(pt - 3 sigma), int(pt + 3 sigma + 1)) per axis (int
    truncates toward zero) and in the image -> gauss[y - ul1][x - ul0]; the whole map is zero when ul >= S or br < 0 on
    either axis."""
    pt = ko.heat_center(kp)
    ul = [int(pt[d] - np.float32(3 * sigma)) for d in range(2)]
    br = [int((pt[d] + np.float32(3 * sigma)) + np.float32(1)) for d in range(2)]
    g = ko.gauss_table(sigma).reshape(6 * sigma + 1, 6 * sigma + 1)
    img = np.zeros((S, S), np.float32)
    n = 6 * sigma + 1
    if ul[0] >= S or ul[1] >= S or br[0] < 0 or br[1] < 0:
        return img
    for y in range(S):
        for x in range(S):
            # the window is at most the table's n pixels wide (float32 rounding can make br - ul = n + 1)
            if ul[0] <= x < br[0] and ul[1] <= y < br[1] and x - ul[0] < n and y - ul[1] < n:
                img[y, x] = g[y - ul[1], x - ul[0]]
    return img


# (kp, sigma, S): centred, clipped at each border, negative pt whose truncation moves the window, all-zero maps
HEAT_CASES = [((0.0, 0.0), 3, 64), ((-0.95, 0.3), 3, 64), ((0.2, -1.0), 2, 48), ((-1.02, -1.03), 3, 64),
              ((-1.05, 0.0), 1, 32), ((-1.0 - 9.5 / 128, 0.0), 3, 64), ((-1.0 - 10.5 / 128, 0.0), 3, 64),
              ((-1.0 - 12.0 / 128, 0.5), 3, 64), ((-1.0 + 8.5 / 128, 0.0), 3, 64), ((-1.0 + 0.5 / 128, 0.2), 3, 64),
              ((-1.0 - 0.5 / 128, -1.0 - 0.5 / 128), 3, 64), ((0.0, -1.3), 3, 64), ((-0.5, -0.5), 7, 64), ((-0.51, -0.49), 7, 64),
              ((-1.0 + 62.5 / 128, 0.0), 3, 64), ((-1.0 + 63.0 / 128, 0.1), 3, 64), ((-1.0 + 64.0 / 128, 0.0), 3, 64),
              ((0.9, 0.9), 3, 255), ((1.0, 1.0), 3, 257), ((float("nan"), 0.0), 3, 32), ((5.0, 0.0), 3, 64),
              # float32 rounding makes br - ul = 6 sigma + 2 on one or both axes: the window is clamped to the table
              ((-0.06250006, 0.0), 3, 256), ((-0.06250006, -0.06250006), 3, 256), ((-5.96e-8, -5.96e-8), 3, 256),
              ((-5.96e-8, 0.3), 1, 256), ((-0.16406257450580597, -0.16406257450580597), 7, 255),
              ((-0.4218750596046448, 0.5781248807907104), 18, 257)]


@pytest.mark.parametrize("kp,sigma,S", HEAT_CASES)
def test_oracle_heatmap_is_draw_labelmap(kp, sigma, S):
    got = ko.heatmap(kp, sigma, S)
    if np.isnan(kp[0]):
        assert not got.any()   # the reference cannot draw it (int(nan)); the kernels and the oracle draw nothing
        return
    np.testing.assert_array_equal(got, heatmap_per_pixel(kp, sigma, S))


def test_heatmap_cases_cover_truncation_and_clipping():
    pts = [ko.heat_center(kp)[0] for kp, s, S in HEAT_CASES if not np.isnan(kp[0])]
    # pt in heat-map pixels; sigma = 3 for these
    assert any(-1 < p - 9 < 0 for p in pts)                  # pt - 3 sigma in (-1, 0): int() rounds up to 0
    assert any(-1 < p + 10 < 0 for p in pts)                 # br = int(pt + 10) = 0: drawn, but an empty window
    assert any(p + 10 <= -1 for p in pts)                    # br < 0: the all-zero map
    assert any(p - 9 <= -1 and p + 10 >= 1 for p in pts)     # clipped on the left
    maps = [ko.heatmap(kp, s, S) for kp, s, S in HEAT_CASES]
    assert sum(not m.any() for m in maps) >= 4


def _unclamped_width(kp, sigma):
    pt = ko.heat_center(kp)
    return [int((pt[d] + np.float32(3 * sigma)) + np.float32(1)) - int(pt[d] - np.float32(3 * sigma)) for d in range(2)]


def test_heatmap_cases_cover_windows_wider_than_the_table():
    widths = [_unclamped_width(kp, s) == [6 * s + 2] * 2 for kp, s, S in HEAT_CASES if not np.isnan(kp[0])]
    assert sum(widths) >= 3    # both axes one pixel too wide, so the last row would overrun the table
    for sigma in (1, 3, 7, 18):
        wide = ko.wide_window_keypoints(sigma, 256)
        assert wide and all(_unclamped_width((w, w), sigma) == [6 * sigma + 2] * 2 for w in wide)
        m = ko.heatmap((wide[0], wide[0]), sigma, 256)
        assert np.count_nonzero(m) == (6 * sigma + 1) ** 2   # the table once, nothing beyond it


def test_gauss_table_is_the_reference_gaussian():
    g = ko.gauss_table(3).reshape(19, 19)
    assert g[9, 9] == 1.0 and g.dtype == np.float32
    assert g[9, 12] == np.float32(np.exp(-0.5))


def test_p2face_is_the_mean_flow_inside_the_image():
    rng = np.random.default_rng(0)
    for S in (64, 255, 256, 257):
        flow = rng.uniform(-1, 1, (50, 9, 2)).astype(np.float32)
        np.testing.assert_allclose(ko.p2face(flow, S), flow.mean(axis=1), rtol=0, atol=4e-6)


@pytest.mark.parametrize("H,W", [(37, 41), (64, 64), (257, 255)])
def test_oracle_sample_is_grid_sample_align_corners(H, W):
    """The oracle's sampler on a random image against torch's own grid_sample(bilinear, zeros, align_corners=True) in
    float64 on the same float32 inputs: within the float32 rounding of the coordinate map and the four products."""
    rng = np.random.default_rng(H * W)
    img = rng.uniform(-1, 1, (3, H, W)).astype(np.float32)
    flow = rng.uniform(-1.2, 1.2, (500, 2)).astype(np.float32)
    flow[:4] = [[-1, -1], [1, 1], [-1, 1], [1, -1]]      # the corners, exactly
    want = torch.nn.functional.grid_sample(torch.from_numpy(img).double()[None], torch.from_numpy(flow).double()[None, None],
                                           mode="bilinear", padding_mode="zeros", align_corners=True)[0, :, 0].T.numpy()
    got = ko.sample(img, flow)
    np.testing.assert_allclose(got, want, rtol=0, atol=4 * max(H, W) * 2.0 ** -24 + 4e-7)
    np.testing.assert_array_equal(got[:4], img[:, [0, H - 1, H - 1, 0], [0, W - 1, 0, W - 1]].T)


def test_p2face_outside_the_image_is_pulled_to_zero():
    """zeros padding: a point past the border on either axis samples the grid at 0; within one pixel of it, less"""
    flow = np.array([[[1.5, 0.0]], [[-3.0, 0.2]], [[1.01, 0.5]]], np.float32)
    pf = ko.p2face(flow, 64)
    assert (pf[:2] == 0).all()
    assert 0 < pf[2, 0] < 1 and 0 < pf[2, 1] < 0.5


def test_oracle_flow_ties_and_empty_heat_maps():
    S = 64
    rng = np.random.default_rng(1)
    fs = rng.uniform(-1, 1, (1, 6, 4, 2)).astype(np.float32)
    fs[0, 4] = fs[0, 2]                                  # faces 2 and 4 tie exactly for every keypoint
    ft = rng.uniform(-1, 1, (1, 6, 4, 2)).astype(np.float32)
    centre = fs[0, 2].mean(axis=0)
    kps = np.array([[centre, [3.0, 3.0]]], np.float32)    # the second keypoint's heat map is all zero
    out, face, margin = ko.transfer_flow(kps, fs, ft, 3, S)
    assert face[0, 1] == 0 and margin[0, 1] == 0          # all-zero means: face 0
    np.testing.assert_array_equal(out[0, 1], ko.p2face(ft[0], S)[0])
    if face[0, 0] in (2, 4):
        assert face[0, 0] == 2 and margin[0, 0] == 0


def test_oracle_cam_nearest_and_empty_mask():
    S = 8
    grid = ko.grid_table(S)
    mask = np.zeros((2, S, S), np.float32)
    mask[0, 2, 5] = 0.25
    mask[0, 6, 1] = 1.0
    proj_src = np.array([[[0.0, 0.0], [0.9, 0.9]]] * 2, np.float32)
    proj_tgt = np.array([[[grid[5], grid[2]], [grid[1], grid[6]]]] * 2, np.float32)
    kps = np.array([[[0.1, 0.0], [0.8, 0.7]]] * 2, np.float32)
    out, margin = ko.transfer_cam(kps, proj_src, proj_tgt, mask, S)
    np.testing.assert_array_equal(out[0, 0], [grid[5], grid[2]])
    np.testing.assert_array_equal(out[0, 1], [grid[1], grid[6]])
    assert np.isnan(out[1]).all()


# ---------------------------------------------------------------------------------------------------------------------
# C ABI: declarations, exports and refusals (no GPU: a refusal comes before any device work)
# ---------------------------------------------------------------------------------------------------------------------
def test_header_declares_exactly_the_bound_symbols():
    src = open(os.path.join(ROOT, "include", "umr_kp_transfer.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = set(re.findall(r"\b(umr_[a-z0-9_]+)\s*\(", src))
    assert names == set(_lib.KP_EXPORTS)
    assert '#include "umr_kp_transfer.h"' in open(os.path.join(ROOT, "include", "umr_b200.h")).read()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(lib, n)


A = 256        # non-NULL, aligned
N0 = None      # NULL
ODD = 256 + 4  # float-aligned, not float2-aligned
ODD1 = 256 + 1  # not float-aligned

FLOW = "umr_kp_transfer_flow"
CAM = "umr_kp_transfer_cam"


def _flow(*, ptrs=(A,) * 6, P=2, K=15, F=8, T2=36, S=256, sigma=3):
    return (FLOW, tuple(ptrs) + (P, K, F, T2, S, sigma))


def _cam(*, ptrs=(A,) * 6, P=2, K=15, V=642, S=256):
    return (CAM, tuple(ptrs) + (P, K, V, S))


def _with(i, v):
    p = [A] * 6
    p[i] = v
    return tuple(p)


REFUSALS = (
    [(_flow(ptrs=_with(i, N0)), BAD_ARG) for i in range(6)]
    + [(_flow(ptrs=_with(i, ODD)), BAD_ARG) for i in (0, 1, 2, 5)]
    + [(_flow(ptrs=_with(i, ODD1)), BAD_ARG) for i in (3, 4)]
    + [(_flow(**{k: v}), BAD_ARG) for k in ("P", "K", "F", "T2", "S", "sigma") for v in (0, -1)]
    + [(_flow(sigma=19), TOO_LARGE), (_flow(P=2 ** 15, K=2 ** 15), TOO_LARGE), (_flow(F=2 ** 25, T2=36), TOO_LARGE)]
    + [(_cam(ptrs=_with(i, N0)), BAD_ARG) for i in range(6)]
    + [(_cam(ptrs=_with(i, ODD)), BAD_ARG) for i in (0, 1, 2, 5)]
    + [(_cam(ptrs=_with(i, ODD1)), BAD_ARG) for i in (3, 4)]
    + [(_cam(**{k: v}), BAD_ARG) for k in ("P", "K", "V", "S") for v in (0, -1)]
    + [(_cam(P=2 ** 15, K=2 ** 15), TOO_LARGE), (_cam(V=2 ** 30), TOO_LARGE), (_cam(S=32768), TOO_LARGE)]
)


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def test_every_entry_point_has_refusal_cases():
    assert {c[0][0] for c in REFUSALS} == set(_lib.KP_EXPORTS)


@pytest.mark.parametrize("case,code", REFUSALS, ids=["%s-%d" % (c[0][4:], i) for i, (c, _) in enumerate(REFUSALS)])
def test_refused_before_device_work(lib, case, code):
    name, args = case
    before = lib.umr_launch_count()
    assert getattr(lib, name)(*args, None) == code
    assert lib.umr_launch_count() == before


# ---------------------------------------------------------------------------------------------------------------------
# Python argument checks (before any device work)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def claims_cuda(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def test_cpu_tensors_are_refused():
    k, f = torch.zeros(2, 15, 3), torch.zeros(2, 8, 6, 6, 2)
    with pytest.raises(TypeError):
        kp_transfer.transfer_flow(k, f, f)
    with pytest.raises(TypeError):
        kp_transfer.transfer_cam(k, torch.zeros(1, 5, 3), torch.zeros(2, 7), torch.zeros(2, 7), torch.zeros(2, 8, 8), None)


def test_inputs_on_different_devices_are_refused(claims_cuda):
    k, f = torch.zeros(2, 15, 3), torch.zeros(2, 8, 36, 2)
    with pytest.raises(ValueError, match="one device"):
        kp_transfer.transfer_flow(k, f, f.to("meta"))
    with pytest.raises(ValueError, match="one device"):
        kp_transfer.transfer_cam(k, torch.zeros(1, 5, 3), torch.zeros(2, 7), torch.zeros(2, 7), torch.zeros(2, 8, 8, device="meta"),
                                 None)


@pytest.mark.parametrize("kps,fs,ft,kw", [
    ((2, 15), (2, 8, 6, 6, 2), (2, 8, 6, 6, 2), {}),            # keypoints without coordinates
    ((2, 15, 4), (2, 8, 6, 6, 2), (2, 8, 6, 6, 2), {}),
    ((2, 15, 3), (3, 8, 6, 6, 2), (3, 8, 6, 6, 2), {}),         # P differs
    ((2, 15, 3), (2, 8, 6, 6, 2), (2, 9, 6, 6, 2), {}),         # flows differ
    ((2, 15, 3), (2, 8, 6, 6, 3), (2, 8, 6, 6, 3), {}),
    ((2, 15, 3), (2, 8, 36, 2), (2, 8, 36, 2), {"sigma": 0}),
    ((2, 15, 3), (2, 8, 36, 2), (2, 8, 36, 2), {"sigma": 2.5}),
    ((2, 15, 3), (2, 8, 36, 2), (2, 8, 36, 2), {"image_size": 0}),
])
def test_flow_argument_checks(claims_cuda, kps, fs, ft, kw):
    with pytest.raises(ValueError):
        kp_transfer.transfer_flow(torch.zeros(kps), torch.zeros(fs), torch.zeros(ft), **kw)


@pytest.mark.parametrize("verts,cs,ct,mask", [
    ((1, 5, 3), (2, 7), (2, 7), (2, 8, 9)),        # mask not square
    ((1, 5, 3), (2, 7), (2, 7), (3, 8, 8)),        # P differs
    ((1, 5, 3), (2, 6), (2, 7), (2, 8, 8)),
    ((3, 5, 3), (2, 7), (2, 7), (2, 8, 8)),        # verts neither shared nor per pair
    ((1, 5, 2), (2, 7), (2, 7), (2, 8, 8)),
])
def test_cam_argument_checks(claims_cuda, verts, cs, ct, mask):
    with pytest.raises(ValueError):
        kp_transfer.transfer_cam(torch.zeros(2, 15, 3), torch.zeros(verts), torch.zeros(cs), torch.zeros(ct),
                                 torch.zeros(mask), None)


# ---------------------------------------------------------------------------------------------------------------------
# PCK (test_kp.py:254-258, 316-322)
# ---------------------------------------------------------------------------------------------------------------------
def test_pck_matches_the_reference_formula():
    rng = np.random.default_rng(2)
    pred = rng.uniform(-1, 1, (40, 15, 2)).astype(np.float32)
    gt = (pred + rng.normal(0, 0.1, pred.shape)).astype(np.float32)
    vis = (rng.uniform(size=(40, 15)) > 0.3).astype(np.float32)
    scale = (1 + 2 * 0.05) / 2.0
    err = np.sqrt(np.sum((pred - gt) * (pred - gt), axis=2)) * scale
    want = [((np.sum((err < t) * vis, axis=0)) / np.sum(vis, axis=0)).mean() for t in (0.1, 0.15)]
    got = kp_transfer.pck(torch.from_numpy(pred), torch.from_numpy(gt), torch.from_numpy(vis), scale)
    assert got == pytest.approx(want, abs=0) and len(got) == 2


def test_pck_threshold_is_strict_and_an_unseen_keypoint_gives_nan():
    pred = np.zeros((2, 2, 2), np.float32)
    gt = np.array([[[0.1, 0.0], [0.0, 0.0]], [[0.0, 0.0], [0.0, 0.0]]], np.float32)
    assert kp_transfer.pck(pred, gt, np.ones((2, 2)), 1.0, thresholds=(np.float32(0.1),))[0] == 0.75
    assert np.isnan(kp_transfer.pck(pred, gt, np.array([[1, 0], [1, 0]]), 1.0)[0])


# ---------------------------------------------------------------------------------------------------------------------
# sampler channel groups, on a fake library (the dispatch only: calls, channel counts and NULL pointers)
# ---------------------------------------------------------------------------------------------------------------------
class FakeLib(object):
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        argtypes = _lib.EXPORTS[name][1]

        def call(*args):
            assert len(args) == len(argtypes)
            for t, a in zip(argtypes, args):
                t.from_param(a)
            self.calls.append((name, args))
            return 0
        return call


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(torch.cuda, "device", lambda device: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: types.SimpleNamespace(cuda_stream=0))
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    return lib


def _calls(fake):
    """(symbol, channel count or None, NULL mask of the pointers) per call"""
    out = []
    for name, args in fake.calls:
        ints = [a for a in args if isinstance(a, int)]
        mask = "".join("1" if a.value else "0" for a in args[:-1] if isinstance(a, ctypes.c_void_p))   # not the stream
        out.append((name, ints[1] if "cells" not in name else None, mask))
    return out


def _run(C, dtype, image_grad=True):
    img = torch.rand(2, C, 5, 6, dtype=dtype).requires_grad_(image_grad)
    flow = torch.rand(2, 7, 2, dtype=dtype).requires_grad_(True)
    out = ops.bilinear_sample(img, flow)
    assert out.shape == (2, 7, C) and out.dtype == dtype
    out.sum().backward()
    assert flow.grad.shape == flow.shape
    if image_grad:
        assert img.grad.shape == img.shape
    return out


# the calls of today's code, C <= 4: one forward, one backward (after the cell table in deterministic / float64 mode)
@pytest.mark.parametrize("C", [1, 2, 3, 4])
@pytest.mark.parametrize("mode", ["f32", "det", "f64"])
def test_up_to_four_channels_issue_todays_calls(fake, C, mode):
    dtype = torch.float64 if mode == "f64" else torch.float32
    with _deterministic(mode == "det"):
        _run(C, dtype)
    sfx = {"f32": "", "det": "_deterministic", "f64": "_f64"}[mode]
    fsfx = "_f64" if mode == "f64" else ""
    want = [("umr_bilinear_sample_forward" + fsfx, C, "111")]
    if mode == "f32":
        want.append(("umr_bilinear_sample_backward", C, "11111"))
    else:
        want += [("umr_bilinear_sample_cells" + fsfx, None, "11"), ("umr_bilinear_sample_backward" + sfx, C, "1111111")]
    assert _calls(fake) == want


@pytest.mark.parametrize("C,groups", [(5, [4, 1]), (8, [4, 4]), (15, [4, 4, 4, 3])])
@pytest.mark.parametrize("mode", ["f32", "det", "f64"])
@pytest.mark.parametrize("image_grad", [True, False])
def test_more_channels_run_in_groups_of_four(fake, C, groups, mode, image_grad):
    dtype = torch.float64 if mode == "f64" else torch.float32
    with _deterministic(mode == "det"):
        _run(C, dtype, image_grad)
    sfx = {"f32": "", "det": "_deterministic", "f64": "_f64"}[mode]
    fsfx = "_f64" if mode == "f64" else ""
    gi = "1" if image_grad else "0"
    want = [("umr_bilinear_sample_forward" + fsfx, c, "111") for c in groups]
    if mode == "f32":
        want += [("umr_bilinear_sample_backward", c, "1111" + gi) for c in groups]
    else:
        if image_grad:   # one cell table for all groups: it depends on the flow only
            want.append(("umr_bilinear_sample_cells" + fsfx, None, "11"))
        want += [("umr_bilinear_sample_backward" + sfx, c, "1111" + gi + gi + gi) for c in groups]
    assert _calls(fake) == want


@contextlib.contextmanager
def _deterministic(on):
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(old)
