"""The harness of the rasteriser range tests (test_raster_gather_range_gpu.py, test_raster_fast_range_gpu.py,
test_raster_part_map_range_gpu.py): renders through the C entry points with every buffer between NaN guard bands, oracle
B on the same inputs (oracle4: the 4-channel part-map render composed from two of them), and the tolerance gates.

Every input sits between guard bands and every output is prefilled with a NaN payload no kernel produces; after each
call the bands are compared bit for bit and every output element must have been written.  Buffers start on 256-byte
boundaries (the float32 kernels store float2 / float4).  The caller-allocated pair buffer of the default float32 path
sits between byte guard bands too; its header (blocks wanted, tiles left unsaved) is returned with each forward.

Tolerances.  float64: hard depth, face-id and RGB planes bit-exact; planes and p2f RTOL 1e-11 with ATOL 1e-13; gradients
1e-11 relative with a floor of 1e-11 x the largest reference magnitude of that face's own 9 vertex components or texel
block (one scene excepted, see face_floor_shared below).  float32: the gates of test_raster_modes_gpu (1e-4 relative,
1e-6 absolute on planes, gradients 1e-6 of the tensor's largest magnitude; hard depth / face-id planes bit-exact),
widened only for the scenes with a face covering the raster (DET_LOOSE below)."""
import ctypes
import time

import numpy as np
import pytest
import torch

import raster_range_scenes as rs
import softras
from umr_b200 import _lib, raster

DEV = "cuda:0"
KW = rs.KW
RTOL64, ATOL64, GRTOL64 = 1e-11, 1e-13, 1e-11
# A face's vertex gradient sums D (1 - D) / sigma terms.  Where D lies within a few ulps of 1 (a band just inside the
# edge), 1 - D is rounding noise that one ulp of exp (CUDA's against glibc's) changes completely.  A face whose few
# pixels all fall in that band has a vertex gradient made of that noise: the 65535 renders of 2 x 2 pixels do, and only
# there is the float64 floor of a face's vertex gradient 1e-11 of the larger of its own largest component and 1e-2 of
# the tensor's largest (face_floor_shared); everywhere else it is the face's own.  Texel gradients carry no 1 - D.
# In float32 the band is 2^29 times wider: scenes with a face covering the raster put thousands of pixels in it, and
# only those scenes (LOOSE) hold float32 vertex gradients to 5e-5 of the tensor's largest with a relative
# tolerance of 2e-3 and p2f to 2e-6 absolute; the crowd and edge scenes keep test_raster_modes_gpu's gates.
GRAD_FACE_FLOOR = 1e-2
# A float32 texel gradient is a sum of one term per (pixel, face) pair that samples the texel, added by the kernels in
# the order their atomics land and by oracle B in pixel order.  Each addition rounds by at most half an ulp of the
# partial sum, and every partial sum is at most sum |term|, so the two results differ by a random walk of such
# roundings: about 2^-24 x sum |term| where the terms cancel.  Where they cancel, that exceeds the float32 floor below
# (1e-6 of the tensor's largest gradient), and the comparison would depend on the atomics' order: the float32 paths'
# texel gradients also get a per-texel floor of TEX_SUM_ULPS x 2^-24 x sum |term| (oracle B's texel gradient with
# absolute adjoints, "grad_tex_abs": every texel weight is >= 0).  A term dropped or added twice is larger than that.
TEX_SUM_ULPS = 8.0
DET_STRICT = dict(grad_faces_atol=1e-6, grad_faces_rtol=1e-4, p2f_atol=1e-6)
DET_LOOSE = dict(grad_faces_atol=5e-5, grad_faces_rtol=2e-3, p2f_atol=2e-6)
GUARD = 256                                     # bytes of each band
BITS = {np.float64: (torch.int64, 0x7FF4DEAD0000F111, 0x7FF4DEAD0000A5A5),   # (int view, output fill, guard)
        np.float32: (torch.int32, 0x7FA0F111, 0x7FA0A5A5)}
TDT = {np.float64: torch.float64, np.float32: torch.float32}
SUFFIX = {"f64": "_f64", "det": "_deterministic", "default": ""}


@pytest.fixture(autouse=True)
def oracle_on_the_kernel_grid(monkeypatch):
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
    """A device buffer [guard | body | guard]; the body is a copy of `array` or, for an output, the fill payload.
    skew: the body starts `skew` elements past a 256-byte boundary (the leading band grows by as much)."""

    def __init__(self, dtype, shape=None, array=None, skew=0):
        self.dtype = dtype
        it, fill, guard = BITS[dtype]
        self.shape = tuple(array.shape if array is not None else shape)
        self.n = int(np.prod(self.shape))
        self.g = GUARD // np.dtype(dtype).itemsize + skew
        self.raw = torch.full((self.n + 2 * self.g,), guard, dtype=it, device=DEV)
        self.body = self.raw[self.g:self.g + self.n]
        if array is not None:
            src = np.ascontiguousarray(array, dtype).reshape(-1)
            self.body.copy_(torch.from_numpy(src.view(np.int64 if dtype == np.float64 else np.int32)))
        else:
            self.body.fill_(fill)
        assert self.ptr().value % 256 == skew * np.dtype(dtype).itemsize

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


class BandedBytes(object):
    """A uint8 output [guard | body | guard] whose body starts filled with a non-zero byte: an output the call must
    clear before it marks anything."""
    FILL, GUARD_BYTE = 0x5A, 0xA5

    def __init__(self, shape):
        self.shape = tuple(shape)
        self.n = int(np.prod(self.shape))
        self.raw = torch.full((self.n + 2 * GUARD,), self.GUARD_BYTE, dtype=torch.uint8, device=DEV)
        self.body = self.raw[GUARD:GUARD + self.n]
        self.body.fill_(self.FILL)
        assert self.ptr().value % 256 == 0

    def ptr(self):
        return ctypes.c_void_p(self.body.data_ptr())

    def check(self, what):
        assert bool((self.raw[:GUARD] == self.GUARD_BYTE).all()) and bool((self.raw[GUARD + self.n:] == self.GUARD_BYTE).all()), \
            "%s: a guard band was written" % what

    def numpy(self):
        return self.body.view(self.shape).cpu().numpy()


class Workspace(object):
    """Scratch bytes [guard | body | guard] (the workspace, the pair buffer)."""

    def __init__(self, nbytes):
        self.nbytes = nbytes
        self.raw = torch.full((nbytes + 2 * GUARD,), 0xA5, dtype=torch.uint8, device=DEV)
        self.body = self.raw[GUARD:GUARD + nbytes]
        assert self.body.data_ptr() % 256 == 0

    def ptr(self):
        return ctypes.c_void_p(self.body.data_ptr())

    def check(self, what="the workspace"):
        assert bool((self.raw[:GUARD] == 0xA5).all()) and bool((self.raw[GUARD + self.nbytes:] == 0xA5).all()), \
            "%s: a guard band was written" % what

    def header(self):
        """The pair buffer's control words: (blocks wanted, tiles left unsaved), or None where the call left them
        untouched (a buffer the render does not use)."""
        if bool((self.body[:8] == 0xA5).all()):
            return None
        return tuple(int(x) for x in self.body[:8].view(torch.int32).cpu().tolist())


NULL = ctypes.c_void_p(0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def pair_buffer(B, isz, aa, blocks):
    """A pair buffer sized by umr_raster_pair_buffer_bytes for `blocks` blocks, or None for blocks = 0."""
    if not blocks:
        return None
    return Workspace(_lib.load().umr_raster_pair_buffer_bytes(B, isz, 1 if aa else 0, int(blocks)))


# ---------------------------------------------------------------------------------------------------------------------
# one render through the C entry points
# ---------------------------------------------------------------------------------------------------------------------
def params(B, F, T2, isz, aa, kw, group=1, nc=3, pairs=None, tile=0):
    k = dict(dict(KW, background_color=(0.0, 0.0, 0.0), near=1.0, far=100.0, fill_back=True, eps=1e-3, dist_func="euclidean",
                  aggr_func_rgb="softmax", aggr_func_alpha="prod", texture_type="surface"), **kw)
    p = raster.make_params(B, F, T2, isz, aa, k["background_color"], k["near"], k["far"], k["fill_back"], k["eps"],
                           k["sigma_val"], k["dist_func"], k["dist_eps"], k["gamma_val"], k["aggr_func_rgb"],
                           k["aggr_func_alpha"], k["texture_type"])
    p.shared_textures = group if group > 1 else 0
    p.color_channels = nc
    p.tile_mode = tile
    if pairs is not None:
        p.pair_buffer, p.pair_buffer_bytes = pairs.body.data_ptr(), pairs.nbytes
    if nc == 4:
        p.background_extra = float(k.get("background_extra", 0.0))
    return p


def c_render(path, fv, tex, isz, aa, g, kw, grads=(True, True), nc=3, blocks=0, tile=0, split=False):
    """Forward and (g not None) backward of `path` ("f64", "det" or "default"; blocks: the default path's pair buffer,
    tile: its tile_mode; split: the split backward) with guard bands; returns numpy outputs and the pair buffer's
    header after the forward ("pairs", None without a buffer)."""
    lib = _lib.load()
    dt = np.float64 if path == "f64" else np.float32
    sfx = SUFFIX[path]
    B, F = fv.shape[:2]
    T2, G = tex.shape[2], tex.shape[0]
    S = isz * (2 if aa else 1)
    pb = pair_buffer(B, isz, aa, blocks) if path == "default" else None
    p = params(B, F, T2, isz, aa, kw, B // G, nc, pb, tile)
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
    out = {"pairs": pb.header() if pb is not None else None}
    outs = [("images", images), ("aggrs", aggrs), ("p2f", p2f)] + ([("colors", colors)] if aa else [])
    t_bwd = None
    if g is not None:
        gb = Banded(dt, array=g)
        gf = Banded(dt, (B, F, 9)) if grads[0] else None
        gt = Banded(dt, tex.shape) if grads[1] else None
        bwd = "umr_raster_backward" + ("_split" if split else "") + sfx
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _lib.check(getattr(lib, bwd)(fvb.ptr(), texb.ptr(), (colors if aa else images).ptr(), aggrs.ptr(), gb.ptr(),
                                     gf.ptr() if gf else NULL, gt.ptr() if gt else NULL, ctypes.byref(p), ws.ptr(), st), bwd)
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
    if pb is not None:
        pb.check("the pair buffer")
    out["t_bwd"] = t_bwd
    return out


def c_silhouette(path, fv, isz, aa, g_alpha, kw, blocks=0, tile=0):
    """umr_raster_forward_silhouette(_deterministic) and (g_alpha [B, isz, isz] not None) the backward, float32, with
    guard bands; returns alpha, alpha_hi (anti-aliased only), grad_faces and the pair buffer's header."""
    lib = _lib.load()
    dt = np.float32
    sfx = SUFFIX[path]
    B, F = fv.shape[:2]
    S = isz * (2 if aa else 1)
    pb = pair_buffer(B, isz, aa, blocks) if path == "default" else None
    p = params(B, F, 1, isz, aa, kw, 1, 3, pb, tile)
    fvb = Banded(dt, array=fv)
    ws = Workspace(lib.umr_raster_workspace_bytes(B, F, isz, 1 if aa else 0))
    alpha = Banded(dt, (B, isz, isz))
    alpha_hi = Banded(dt, (B, S, S)) if aa else None
    st = _stream()
    _lib.check(getattr(lib, "umr_raster_forward_silhouette" + sfx)(fvb.ptr(), alpha.ptr(), alpha_hi.ptr() if aa else NULL,
                                                                   ctypes.byref(p), ws.ptr(), st),
               "umr_raster_forward_silhouette" + sfx)
    out = {"pairs": pb.header() if pb is not None else None}
    outs = [("alpha", alpha)] + ([("alpha_hi", alpha_hi)] if aa else [])
    if g_alpha is not None:
        gb = Banded(dt, array=g_alpha)
        gf = Banded(dt, (B, F, 9))
        _lib.check(getattr(lib, "umr_raster_backward_silhouette" + sfx)(fvb.ptr(), (alpha_hi if aa else alpha).ptr(), gb.ptr(),
                                                                        gf.ptr(), ctypes.byref(p), ws.ptr(), st),
                   "umr_raster_backward_silhouette" + sfx)
        outs.append(("grad_faces", gf))
        torch.cuda.synchronize()
        gb.check("grad_alpha", False)
    torch.cuda.synchronize()
    for name, b in outs:
        b.check("%s silhouette %s" % (path, name), True)
        out[name] = b.numpy()
    fvb.check("face_vertices", False)
    ws.check()
    if pb is not None:
        pb.check("the pair buffer")
    return out


def oracle(path, fv, tex, isz, aa, g, kw, dt=None, alpha_only=False, tex_abs=True):
    """oracle B in the path's precision (or dt); textures [G, ...] are expanded to the B renders and their gradient summed
    back.  alpha_only: also the vertex gradient with the colour adjoints zeroed ("grad_faces_alpha"); tex_abs: the float32
    texel gradient with absolute adjoints ("grad_tex_abs", the texel gates' floor)."""
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
        if dt == np.float32 and tex_abs:
            gta = softras.backward(fwd, np.abs(ghi), cfg, impl="B")[1]
            out["grad_tex_abs"] = np.abs(gta).reshape(G, B // G, *tex.shape[1:]).sum(1)
        if alpha_only:
            ga = np.zeros_like(ghi)
            ga[:, 3] = ghi[:, 3]
            out["grad_faces_alpha"] = softras.backward(fwd, ga, cfg, impl="B")[0]
    return out


def oracle4(fv, tex, isz, aa, g, kw):
    """The 4-channel part-map render (float32, textures [G, F, T2, 4], images [B, 5, ...], kw's background_color (b0, b1,
    b2) and background_extra bg3) composed from two 3-channel oracle B renders: A of channels 0-2 on (b0, b1, b2), and B of
    channels (3, 0, 1) on (bg3, b0, b1).  Colour planes 0-2, alpha, aggrs and p2f are A's, plane 3 is B's plane 0.  Colour
    channels do not interact in the rasteriser, so the vertex gradient is linear in the adjoint: A's for the adjoints of
    planes 0-2 and alpha plus B's for plane 3's adjoint alone.  There is no texel gradient (part maps are constants).
    Also returns the two renders ("A", "B")."""
    k = dict(kw)
    b0, b1, b2 = (float(c) for c in k.get("background_color", (0.0, 0.0, 0.0))[:3])
    bg3 = float(k.pop("background_extra", 0.0))
    ga = gb = None
    if g is not None:
        g = np.asarray(g, np.float32)
        ga = np.ascontiguousarray(g[:, [0, 1, 2, 4]])
        gb = np.zeros_like(ga)
        gb[:, 0] = g[:, 3]
    a = oracle("det", fv, tex[..., 0:3], isz, aa, ga, dict(k, background_color=(b0, b1, b2)), tex_abs=False)
    b = oracle("det", fv, tex[..., [3, 0, 1]], isz, aa, gb, dict(k, background_color=(bg3, b0, b1)), tex_abs=False)
    four = lambda x, y: np.concatenate([x[:, :3], y[:, :1], x[:, 3:]], 1)   # noqa: E731
    out = dict(images=four(a["images"], b["images"]), colors=four(a["colors"], b["colors"]), aggrs=a["aggrs"], p2f=a["p2f"],
               A=a, B=b)
    if g is not None:
        out["grad_faces"] = a["grad_faces"] + b["grad_faces"]
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
    """Asserts the path's tolerances (rtol: the float32 paths' planes; loose: a scene with a face covering the raster;
    face_floor_shared: the float64 vertex-gradient floor takes 1e-2 of the tensor's largest as well); returns the
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
            if name == "grad_tex" and ref.get("grad_tex_abs") is not None:   # rounding of a cancelling sum (TEX_SUM_ULPS)
                atol = np.fmax(atol, TEX_SUM_ULPS * 2.0 ** -24 * np.asarray(ref["grad_tex_abs"], np.float64))
            worst[name] = _ratio(got[name], b, max(rtol, det["grad_faces_rtol"]) if name == "grad_faces" else rtol, atol)
    msg = "%s %s: worst error/bound %s" % (path, what, ", ".join("%s %.3g" % kv for kv in worst.items()))
    assert all(v <= 1.0 for v in worst.values()), msg
    if rgb == "hard" and got.get("aggrs") is not None and ref.get("aggrs") is not None:
        assert np.array_equal(got["aggrs"], ref["aggrs"]), "%s %s: hard depth / face-id planes not bit-exact" % (path, what)
        if path == "f64":
            assert np.array_equal(got["images"][:, :3], ref["images"][:, :3], equal_nan=True), "%s %s: hard RGB" % (path, what)
    return max(worst.values()) if worst else 0.0


def _bits_equal(a, b, what):
    for k in a:
        if k in ("t_bwd", "pairs") or a[k] is None:
            continue
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), "%s: %s differs bitwise" % (what, k)
