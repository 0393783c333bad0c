"""The float64 rasteriser (umr_raster_*_f64) and the deterministic float32 one (umr_raster_*_deterministic) across their
accepted input range, through their C entry points, against CPU oracle B (float64 for the first, float32 for the second).

Both run the face-parallel gather backward (one warp per face walks its cull box; texel gradients combined with
__match_any_sync) and fixed-point p2f; the float64 forward lists each tile's faces in 1024-face windows.  The scenes of
raster_range_scenes.py reach what the feature scenes of test_raster_f64_gpu / test_deterministic_gpu do not: tile lists
consumed mid-scan, box edges on pixel centres, S = 1 and 2, odd anti-aliased sizes, T2 up to 1449^2 and non-square T2,
shared textures over 8 images, planes that cut faces, B = 65535 and F = 2^24.

Every input sits between NaN guard bands and every output is prefilled with a NaN payload no kernel produces; after each
call the bands are compared bit for bit and every output element must have been written.  Buffers start on 256-byte
boundaries (the float32 kernels store float2 / float4).

Tolerances.  float64: hard depth, face-id and RGB planes bit-exact; planes and p2f RTOL 1e-11 with ATOL 1e-13; gradients
1e-11 relative with a floor of 1e-11 x the largest reference magnitude of that face's own 9 vertex components or texel
block (one scene excepted, see face_floor_shared below).  Deterministic: the gates of test_raster_modes_gpu (1e-4
relative, 1e-6 absolute on planes, gradients 1e-6 of the tensor's largest magnitude; hard depth / face-id planes
bit-exact), widened only for the scenes with a face covering the raster (DET_LOOSE below).  Each case prints the count of what it targets and its
worst error / bound ratio."""
import ctypes
import math
import time

import numpy as np
import pytest
import torch

import raster_range_scenes as rs
import softras
from umr_b200 import _lib, raster

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KW = rs.KW
RTOL64, ATOL64, GRTOL64 = 1e-11, 1e-13, 1e-11
# A face's vertex gradient sums D (1 - D) / sigma terms.  Where D lies within a few ulps of 1 (a band just inside the
# edge), 1 - D is rounding noise that one ulp of exp (CUDA's against glibc's) changes completely.  A face whose few
# pixels all fall in that band has a vertex gradient made of that noise: the 65535 renders of 2 x 2 pixels do, and only
# there is the float64 floor of a face's vertex gradient 1e-11 of the larger of its own largest component and 1e-2 of
# the tensor's largest (face_floor_shared); everywhere else it is the face's own.  Texel gradients carry no 1 - D.
# In float32 the band is 2^29 times wider: scenes with a face covering the raster put thousands of pixels in it, and
# only those scenes (LOOSE) hold deterministic vertex gradients to 5e-5 of the tensor's largest with a relative
# tolerance of 2e-3 and p2f to 2e-6 absolute; the crowd and edge scenes keep test_raster_modes_gpu's gates.
GRAD_FACE_FLOOR = 1e-2
DET_STRICT = dict(grad_faces_atol=1e-6, grad_faces_rtol=1e-4, p2f_atol=1e-6)
DET_LOOSE = dict(grad_faces_atol=5e-5, grad_faces_rtol=2e-3, p2f_atol=2e-6)
GUARD = 256                                     # bytes of each band
BITS = {np.float64: (torch.int64, 0x7FF4DEAD0000F111, 0x7FF4DEAD0000A5A5),   # (int view, output fill, guard)
        np.float32: (torch.int32, 0x7FA0F111, 0x7FA0A5A5)}
TDT = {np.float64: torch.float64, np.float32: torch.float32}
SIZES = [(1, False), (2, False), (17, False), (31, False), (33, False), (9, True), (17, True), (33, True)]
PATHS = ["f64", "det"]


@pytest.fixture(autouse=True)
def _oracle_on_the_kernel_grid(monkeypatch):
    # oracle B is handed the kernels' own float32 grid (see raster_range_scenes.kernel_grid), in both precisions
    monkeypatch.setattr(softras, "standard_grid", rs.kernel_grid)


_EPS = {}


def oracle_eps(gamma):
    """An eps for which the device's expf(eps / gamma) (the softmax seed, a float expression) equals glibc's: at others
    they may differ by a float ulp, which is not a property of the kernels.  Not a dyadic value."""
    if gamma not in _EPS:
        libm = ctypes.CDLL("libm.so.6")
        libm.expf.restype, libm.expf.argtypes = ctypes.c_float, [ctypes.c_float]
        for eps in (1e-3, 2e-3, 5e-4, 1.5e-3, 3e-3, 7e-4, 1e-4):
            q = np.float32(eps) / np.float32(gamma)
            if float(torch.exp(torch.tensor(float(q), dtype=torch.float32, device=DEV))) == libm.expf(float(q)):
                _EPS[gamma] = eps
                break
        else:
            raise AssertionError("no eps found")
    return _EPS[gamma]


# ---------------------------------------------------------------------------------------------------------------------
# guarded buffers
# ---------------------------------------------------------------------------------------------------------------------
class Banded(object):
    """A device buffer [guard | body | guard]; the body is a copy of `array` or, for an output, the fill payload."""

    def __init__(self, dtype, shape=None, array=None):
        self.dtype = dtype
        it, fill, guard = BITS[dtype]
        self.shape = tuple(array.shape if array is not None else shape)
        self.n = int(np.prod(self.shape))
        self.g = GUARD // np.dtype(dtype).itemsize
        self.raw = torch.full((self.n + 2 * self.g,), guard, dtype=it, device=DEV)
        self.body = self.raw[self.g:self.g + self.n]
        if array is not None:
            src = np.ascontiguousarray(array, dtype).reshape(-1)
            self.body.copy_(torch.from_numpy(src.view(np.int64 if dtype == np.float64 else np.int32)))
        else:
            self.body.fill_(fill)
        assert self.ptr().value % 256 == 0

    def ptr(self):
        return ctypes.c_void_p(self.body.data_ptr())

    def tensor(self):
        return self.body.view(TDT[self.dtype]).view(self.shape)

    def check(self, what, output):
        it, fill, guard = BITS[self.dtype]
        assert bool((self.raw[:self.g] == guard).all()) and bool((self.raw[self.g + self.n:] == guard).all()), \
            "%s: a guard band was written" % what
        if output:
            left = int((self.body == fill).sum())
            assert left == 0, "%s: %d of %d elements not written" % (what, left, self.n)

    def numpy(self):
        return self.tensor().cpu().numpy()


class Workspace(object):
    def __init__(self, nbytes):
        self.nbytes = nbytes
        self.raw = torch.full((nbytes + GUARD,), 0xA5, dtype=torch.uint8, device=DEV)
        assert self.raw.data_ptr() % 256 == 0

    def ptr(self):
        return ctypes.c_void_p(self.raw.data_ptr())

    def check(self):
        assert bool((self.raw[self.nbytes:] == 0xA5).all()), "the workspace's guard was written"


NULL = ctypes.c_void_p(0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---------------------------------------------------------------------------------------------------------------------
# one render through the C entry points
# ---------------------------------------------------------------------------------------------------------------------
def params(B, F, T2, isz, aa, kw, group=1, nc=3):
    k = dict(dict(KW, background_color=(0.0, 0.0, 0.0), near=1.0, far=100.0, fill_back=True, eps=1e-3, dist_func="euclidean",
                  aggr_func_rgb="softmax", aggr_func_alpha="prod", texture_type="surface"), **kw)
    p = raster.make_params(B, F, T2, isz, aa, k["background_color"], k["near"], k["far"], k["fill_back"], k["eps"],
                           k["sigma_val"], k["dist_func"], k["dist_eps"], k["gamma_val"], k["aggr_func_rgb"],
                           k["aggr_func_alpha"], k["texture_type"])
    p.shared_textures = group if group > 1 else 0
    p.color_channels = nc
    if nc == 4:
        p.background_extra = float(k.get("background_extra", 0.0))
    return p


def c_render(path, fv, tex, isz, aa, g, kw, grads=(True, True), nc=3):
    """Forward and (g not None) backward of `path` with guard bands; returns numpy outputs."""
    lib = _lib.load()
    dt = np.float64 if path == "f64" else np.float32
    sfx = "_f64" if path == "f64" else "_deterministic"
    B, F = fv.shape[:2]
    T2, G = tex.shape[2], tex.shape[0]
    S = isz * (2 if aa else 1)
    p = params(B, F, T2, isz, aa, kw, B // G, nc)
    NPL = nc + 1
    fvb, texb = Banded(dt, array=fv), Banded(dt, array=tex)
    ws = Workspace(getattr(lib, "umr_raster_workspace_bytes" + sfx)(B, F, isz, 1 if aa else 0))
    images = Banded(dt, (B, NPL, isz, isz))
    colors = Banded(dt, (B, NPL, S, S)) if aa else None
    aggrs, p2f = Banded(dt, (B, 2, S, S)), Banded(dt, (B, F, 2))
    st = _stream()
    _lib.check(getattr(lib, "umr_raster_forward" + sfx)(fvb.ptr(), texb.ptr(), images.ptr(), colors.ptr() if aa else NULL,
                                                        aggrs.ptr(), p2f.ptr(), ctypes.byref(p), ws.ptr(), st),
               "umr_raster_forward" + sfx)
    out = {}
    outs = [("images", images), ("aggrs", aggrs), ("p2f", p2f)] + ([("colors", colors)] if aa else [])
    t_bwd = None
    if g is not None:
        gb = Banded(dt, array=g)
        gf = Banded(dt, (B, F, 9)) if grads[0] else None
        gt = Banded(dt, tex.shape) if grads[1] else None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _lib.check(getattr(lib, "umr_raster_backward" + sfx)(fvb.ptr(), texb.ptr(), (colors if aa else images).ptr(),
                                                             aggrs.ptr(), gb.ptr(), gf.ptr() if gf else NULL,
                                                             gt.ptr() if gt else NULL, ctypes.byref(p), ws.ptr(), st),
                   "umr_raster_backward" + sfx)
        torch.cuda.synchronize()
        t_bwd = time.perf_counter() - t0
        outs += [("grad_faces", gf), ("grad_tex", gt)]
        gb.check("grad_images", False)
    torch.cuda.synchronize()
    for name, b in outs:
        if b is not None:
            b.check("%s %s" % (path, name), True)
            out[name] = b.numpy()
    fvb.check("face_vertices", False)
    texb.check("textures", False)
    ws.check()
    out["t_bwd"] = t_bwd
    return out


def oracle(path, fv, tex, isz, aa, g, kw, dt=None):
    """oracle B in the path's precision (or dt); textures [G, ...] are expanded to the B renders and their gradient summed
    back."""
    dt = dt or (np.float64 if path == "f64" else np.float32)
    k = dict(KW, **kw)
    k.pop("background_extra", None)
    B, G = fv.shape[0], tex.shape[0]
    S = isz * (2 if aa else 1)
    cfg = softras.RasterCfg(S, **k)
    texe = np.repeat(tex, B // G, axis=0)
    fwd = softras.forward(fv, texe, cfg, impl="B", dtype=dt)
    out = dict(images=softras.avg_pool2(fwd["soft_colors"]) if aa else fwd["soft_colors"], aggrs=fwd["aggrs_info"],
               p2f=fwd["p2f_info"], colors=fwd["soft_colors"])
    if g is not None:
        ghi = softras.avg_pool2_backward(np.asarray(g, dt)) if aa else np.asarray(g, dt)
        gf, gt = softras.backward(fwd, ghi, cfg, impl="B")
        out["grad_faces"], out["grad_tex"] = gf, gt.reshape(G, B // G, *tex.shape[1:]).sum(1)
    return out


def _ratio(got, ref, rtol, atol):
    """worst |got - ref| / (atol + rtol * max(|got|, |ref|)) over elements finite in both; NaN positions must match."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), "NaN positions differ: %d vs %d" % (np.isnan(got).sum(), np.isnan(ref).sum())
    fin = np.isfinite(got) & np.isfinite(ref)
    assert np.array_equal(got[~fin], ref[~fin], equal_nan=True)
    if not fin.any():
        return 0.0
    atol = np.broadcast_to(atol, got.shape)[fin]
    return float((np.abs(got[fin] - ref[fin]) / (atol + rtol * np.maximum(np.abs(got[fin]), np.abs(ref[fin])))).max())


def compare(path, got, ref, rgb, what, rtol=1e-4, loose=False, face_floor_shared=False):
    """Asserts the path's tolerances (rtol: the deterministic path's planes; loose: a scene with a face covering the
    raster; face_floor_shared: the float64 vertex-gradient floor takes 1e-2 of the tensor's largest as well); returns the
    worst error / bound ratio."""
    worst = {}
    det = DET_LOOSE if loose else DET_STRICT
    for name in ("images", "aggrs", "p2f", "colors", "grad_faces", "grad_tex"):
        if got.get(name) is None or ref.get(name) is None:
            continue
        b = np.asarray(ref[name], np.float64)
        if path == "f64":
            if name == "grad_tex":        # per face: its own texel block
                atol = GRTOL64 * np.nanmax(np.abs(b), axis=(-2, -1), keepdims=True, initial=0.0) + 1e-300
            elif name == "grad_faces":    # per face: its own 9 components
                face = np.nanmax(np.abs(b), axis=-1, keepdims=True, initial=0.0)
                if face_floor_shared:
                    face = np.maximum(face, GRAD_FACE_FLOOR * float(np.nanmax(np.abs(b), initial=0.0)))
                atol = GRTOL64 * face + 1e-300
            else:
                atol = ATOL64
            worst[name] = _ratio(got[name], b, GRTOL64 if name.startswith("grad") else RTOL64, atol)
        else:
            rel = det["grad_faces_atol"] if name == "grad_faces" else 1e-6
            atol = rel * float(np.nanmax(np.abs(b), initial=0.0)) + 1e-7 if name.startswith("grad") else det["p2f_atol"] if name == "p2f" else 1e-6
            worst[name] = _ratio(got[name], b, max(rtol, det["grad_faces_rtol"]) if name == "grad_faces" else rtol, atol)
    msg = "%s %s: worst error/bound %s" % (path, what, ", ".join("%s %.3g" % kv for kv in worst.items()))
    assert all(v <= 1.0 for v in worst.values()), msg
    if rgb == "hard":
        assert np.array_equal(got["aggrs"], ref["aggrs"]), "%s %s: hard depth / face-id planes not bit-exact" % (path, what)
        if path == "f64":
            assert np.array_equal(got["images"][:, :3], ref["images"][:, :3], equal_nan=True), "%s %s: hard RGB" % (path, what)
    return max(worst.values()) if worst else 0.0


def _bits_equal(a, b, what):
    for k in a:
        if k == "t_bwd" or a[k] is None:
            continue
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), "%s: %s differs bitwise" % (what, k)


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
    for nan in (False, True) if path == "f64" else (False,):
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
    rng = np.random.default_rng(7)
    B = 65535
    fv = np.repeat(np.array([[rs.COVER, [-0.6, -0.5, 2.0, 0.7, -0.4, 2.5, -0.1, 0.8, 3.0]]]), B, 0)
    fv[:, 1, [0, 3, 6]] += rng.uniform(-0.8, 0.8, size=(B, 1))
    tex = rng.uniform(0, 1, size=(B, 2, 1, 3))
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
