"""Kernel launches of every raster C entry point and branch: umr_launch_count() counts each kernel launch once (memsets
and event records not at all), and the two profiling events of UmrRasterParams are recorded around the raster kernels.

Counts per call:
  forward (default and deterministic)    3 in UMR's configuration (k_prep, k_bin_coarse, forward), 2 in a generic mode,
                                         +1 (the p2f finalize) for a softmax render asked for p2f
  visibility                             3 (k_prep, k_bin_coarse, planes or bytes)
  backward / split                       2 in a generic mode or without a pair buffer (k_prep, recompute), 3 with one
                                         (k_prep, streamed backward, recompute of the unsaved tiles)
  deterministic backward / split         2 (k_prep, gather)
  silhouette forward                     3, both variants
  silhouette backward                    2, or 3 with a pair buffer; deterministic 2
  float64 forward                        2, +1 finalize for a softmax render asked for p2f
  float64 backward                       2
"""
import ctypes
import itertools

import numpy as np
import pytest
import torch

from umr_b200 import _lib, raster
from util import scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
B, IS = 2, 32
WIDE_F = 65537      # past the 16-bit face indices: the 32-bit index kernels
MODES = {"softmax": {}, "hard": dict(aggr_func_rgb="hard"), "generic softmax": dict(dist_func="barycentric"),
         "generic hard": dict(aggr_func_alpha="sum", aggr_func_rgb="hard")}


def _faces(F, dtype):
    """A seeded mesh in raster space; faces past its own 1280 are copies moved off the raster."""
    fv, _ = scene(B=B, subdiv=3, tex_res=2)
    if F > fv.shape[1]:
        extra = np.repeat(fv[:, :1], F - fv.shape[1], axis=1).copy()
        extra[..., 0::3] += 10.0
        fv = np.concatenate([fv, extra], axis=1)
    return torch.from_numpy(np.ascontiguousarray(fv[:, :F])).to(DEV, dtype)


def _zeros(*shape, dtype=torch.float32):
    return torch.zeros(*shape, dtype=dtype, device=DEV)


def _ptr(t):
    return None if t is None else t.data_ptr()


class Render(object):
    """Buffers and params of one render: F faces, nc colour channels, a pair buffer or none."""

    def __init__(self, F=1280, mode="softmax", nc=3, tile=0, pairs=False, dtype=torch.float32):
        lib = _lib.load()
        kw = dict(dict(B=B, F=F, T2=4, image_size=IS, anti_aliasing=False, background_color=(0, 0, 0), near=1, far=100,
                       fill_back=True, eps=1e-3, sigma_val=1e-4, dist_func="euclidean", dist_eps=1e-4, gamma_val=1e-4,
                       aggr_func_rgb="softmax", aggr_func_alpha="prod", texture_type="surface"), **MODES[mode])
        self.p = raster.make_params(**kw)
        self.p.tile_mode, self.p.color_channels = tile, nc
        self.F, self.dtype = F, dtype
        NPL = (4 if nc == 4 else 3) + 1
        self.fv = _faces(F, dtype)
        self.tex = torch.rand(B, F, 4, NPL - 1, device=DEV).to(dtype)
        self.images, self.aggrs = _zeros(B, NPL, IS, IS, dtype=dtype), _zeros(B, 2, IS, IS, dtype=dtype)
        self.p2f = _zeros(B, F, 2, dtype=dtype)
        self.grad_images = torch.rand(B, NPL, IS, IS, device=DEV).to(dtype)
        self.grad_faces, self.grad_tex = _zeros(B, F, 9, dtype=dtype), torch.zeros_like(self.tex)
        self.alpha, self.grad_alpha = _zeros(B, IS, IS), torch.rand(B, IS, IS, device=DEV)
        self.vis = torch.zeros(B, F, dtype=torch.uint8, device=DEV)
        nbytes = max(lib.umr_raster_workspace_bytes_deterministic(B, F, IS, 0), lib.umr_raster_workspace_bytes_f64(B, F, IS, 0))
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        self.pairs = None
        if pairs:
            n = lib.umr_raster_pair_buffer_bytes(B, IS, 0, 4096)
            self.pairs = torch.empty(n, dtype=torch.uint8, device=DEV)
            self.p.pair_buffer, self.p.pair_buffer_bytes = self.pairs.data_ptr(), n

    def call(self, name, *buffers):
        """Calls the entry point with fresh profiling events; returns its launch count after checking that both events
        were recorded, with device work between them."""
        lib = _lib.load()
        ev = [ctypes.c_void_p(), ctypes.c_void_p()]
        for e in ev:
            _lib.check(lib.umr_event_create(ctypes.byref(e)), "umr_event_create")
        self.p.ev_kernel_start, self.p.ev_kernel_stop = ev[0].value, ev[1].value
        try:
            torch.cuda.synchronize()
            n0 = lib.umr_launch_count()
            _lib.check(getattr(lib, name)(*[_ptr(b) for b in buffers], ctypes.byref(self.p), self.ws.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream), name)
            n = lib.umr_launch_count() - n0
            torch.cuda.synchronize()
            ms = ctypes.c_float()
            assert lib.umr_event_elapsed_ms(ev[0], ev[1], ctypes.byref(ms)) == 0, "%s: an event was not recorded" % name
            assert ms.value > 0, "%s: nothing ran between the events" % name
        finally:
            self.p.ev_kernel_start = self.p.ev_kernel_stop = None
            for e in ev:
                lib.umr_event_destroy(e)
        return n

    def forward(self, det=False, p2f=True):
        sfx = "_f64" if self.dtype == torch.float64 else "_deterministic" if det else ""
        return self.call("umr_raster_forward" + sfx, self.fv, self.tex, self.images, None, self.aggrs,
                         self.p2f if p2f else None)

    def backward(self, det=False, split=False, faces=True, tex=True):
        sfx = ("_split" if split else "") + ("_f64" if self.dtype == torch.float64 else "_deterministic" if det else "")
        return self.call("umr_raster_backward" + sfx, self.fv, self.tex, self.images, self.aggrs, self.grad_images,
                         self.grad_faces if faces else None, self.grad_tex if tex else None)


def _generic(mode):
    return mode.startswith("generic")


@pytest.mark.parametrize("wide", [False, True])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_forward(mode, wide):
    softmax = "softmax" in mode
    for det, p2f, tile, pairs in itertools.product([False, True], [False, True], [16, 32], [False, True]):
        r = Render(WIDE_F if wide else 1280, mode, tile=tile, pairs=pairs)
        want = (2 if _generic(mode) else 3) + (1 if softmax and p2f else 0)
        assert r.forward(det, p2f) == want, (det, p2f, tile, pairs)


@pytest.mark.parametrize("wide", [False, True])
def test_forward_four_channels(wide):
    for det, p2f, pairs in itertools.product([False, True], [False, True], [False, True]):
        r = Render(WIDE_F if wide else 1280, nc=4, tile=32, pairs=pairs)
        assert r.forward(det, p2f) == 3 + p2f, (det, p2f, pairs)


@pytest.mark.parametrize("wide", [False, True])
def test_visibility(wide):
    r = Render(WIDE_F if wide else 1280, "hard")
    for planes, faces in ((True, False), (False, True), (True, True)):
        assert r.call("umr_raster_visibility", r.fv, r.aggrs if planes else None, r.vis if faces else None) == 3


@pytest.mark.parametrize("wide", [False, True])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_backward(mode, wide):
    grads = [(True, True), (True, False)] + ([] if _generic(mode) else [(False, True)])
    for (faces, tex), tile, pairs in itertools.product(grads, [16, 32], [False, True]):
        r = Render(WIDE_F if wide else 1280, mode, tile=tile, pairs=pairs)
        r.forward()
        want = 3 if pairs and not _generic(mode) else 2
        assert r.backward(faces=faces, tex=tex) == want, (faces, tex, tile, pairs)
        assert r.backward(det=True, faces=faces, tex=tex) == 2, (faces, tex, tile, pairs)
        if not _generic(mode) and faces and tex:
            assert r.backward(split=True) == want, (tile, pairs)
            assert r.backward(det=True, split=True) == 2, (tile, pairs)
    if _generic(mode):  # the deterministic backward also takes a texture-only call in the generic modes
        r = Render(WIDE_F if wide else 1280, mode)
        r.forward()
        assert r.backward(det=True, faces=False) == 2


@pytest.mark.parametrize("wide", [False, True])
def test_backward_four_channels(wide):
    for pairs in (False, True):
        r = Render(WIDE_F if wide else 1280, nc=4, tile=32, pairs=pairs)
        r.forward()
        assert r.backward(tex=False) == (3 if pairs else 2), pairs
        assert r.backward(det=True, tex=False) == 2, pairs


@pytest.mark.parametrize("wide", [False, True])
def test_silhouette(wide):
    for tile, pairs in itertools.product([16, 32], [False, True]):
        r = Render(WIDE_F if wide else 1280, tile=tile, pairs=pairs)
        for det in (False, True):
            assert r.call("umr_raster_forward_silhouette" + ("_deterministic" if det else ""), r.fv, r.alpha, None) == 3
        r.call("umr_raster_forward_silhouette", r.fv, r.alpha, None)  # the pair records of the default backward
        assert r.call("umr_raster_backward_silhouette", r.fv, r.alpha, r.grad_alpha, r.grad_faces) == (3 if pairs else 2)
        assert r.call("umr_raster_backward_silhouette_deterministic", r.fv, r.alpha, r.grad_alpha, r.grad_faces) == 2


@pytest.mark.parametrize("mode", sorted(MODES))
def test_f64(mode):
    r = Render(1280, mode, dtype=torch.float64)
    for p2f in (False, True):
        assert r.forward(p2f=p2f) == 2 + (1 if "softmax" in mode and p2f else 0), p2f
    for faces, tex in ((True, True), (True, False), (False, True)):
        assert r.backward(faces=faces, tex=tex) == 2, (faces, tex)
