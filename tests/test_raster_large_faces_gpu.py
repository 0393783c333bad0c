"""GPU parity of meshes above 65535 faces, which take the 32-bit face-index instantiations of the raster kernels (wide
coarse-bin pool, 24-bit pair-block face field, tile lists consumed in 65536-face windows).  Same rules as
test_raster_modes_gpu.check: oracle B at 1e-4 relative, hard planes bit-exact; every pixel plane also bit-exact with the
reference's own CUDA kernels built with -fmad=false, which have no face limit."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from umr_b200 import _lib, raster, synth
from test_raster_modes_gpu import PAIR_BUFFERS, SOFT, UMR, _last_face_is_live, _mode_kw, check, gpu, oracle

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import ref_gpu_compare as rc  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_REF_NOFMA = rc.load("soft_rasterize_ref_nofma")
_ICO7 = {}


def _mesh(F, B=1, seed=0):
    """The F faces of a deformed icosphere(7) (327680 faces) ordered so that the highest indices are the near-side faces
    closest to the pixel centre (1/64, 1/64) of a 64-pixel raster: face F-1 covers that pixel, in front."""
    if "vf" not in _ICO7:
        _ICO7["vf"] = synth.icosphere(7)
    v, f = _ICO7["vf"]
    rng = np.random.default_rng(seed)
    fv = synth.raster_space_faces(synth.bird_like(v, rng, B), f, synth.cameras(rng, B))
    c = fv[0].reshape(-1, 3, 3).mean(axis=1)
    near = c[:, 2] < np.median(c[:, 2])
    order = np.lexsort((-np.hypot(c[:, 0] - 1 / 64, c[:, 1] - 1 / 64), near))
    fv = np.ascontiguousarray(fv[:, order[-F:]])
    tex = rng.uniform(0, 1, size=(B, F, 4, 3)).astype(np.float32)
    return fv, tex


def _vs_reference_planes(fv, tex, isz, got, rgb, **modes):
    """Pixel planes bit-exact with the reference's -fmad=false kernels (anti-aliased render)."""
    if _REF_NOFMA is None:
        return
    tfv, ttex = torch.from_numpy(fv).to(DEV), torch.from_numpy(tex).to(DEV)
    colors, rp2f, raggr, _ = rc.ref_forward(_REF_NOFMA, tfv, ttex, 2 * isz, raster.FUNC_RGB[rgb], **modes)
    assert np.array_equal(got["images"], TF.avg_pool2d(colors, 2, 2).cpu().numpy()), "images vs reference kernels"
    assert np.array_equal(got["aggrs"], raggr.cpu().numpy()), "aggregation planes vs reference kernels"
    assert np.allclose(got["p2f"], rp2f.cpu().numpy(), rtol=1e-4, atol=1e-6)


LADDER = [65536, 65537, 131071, 327680]


@pytest.mark.parametrize("F", LADDER)
def test_large_face_ladder_umr_configuration(F):
    """UMR's kernels just past the 16-bit face fields and up to a full icosphere(7): both tilings with every pair-buffer
    state, the visibility planes and the visible-face bytes, face F-1 on screen."""
    isz = 32
    fv, tex = _mesh(F)
    g = np.random.default_rng(F).normal(size=(1, 4, isz, isz)).astype(np.float32)
    for rgb in ("softmax", "hard"):
        ref = oracle(fv, tex, isz, True, g, aggr_func_rgb=rgb, **UMR)
        for tile in (16, 32):
            for buf, cand in PAIR_BUFFERS.items():
                got = gpu(fv, tex, isz, True, g, tile=tile, cand=cand, aggr_func_rgb=rgb, **UMR)
                check(got, ref, rgb, "F=%d tile=%d pair buffer=%s" % (F, tile, buf))
                _last_face_is_live(got, ref, rgb)
                if tile == 16 and buf == "full":
                    _vs_reference_planes(fv, tex, isz, got, rgb)
        if rgb == "hard":
            tfv = torch.from_numpy(fv).to(DEV)
            vis = raster.visibility(tfv, isz, anti_aliasing=True, **UMR).cpu().numpy()
            assert np.array_equal(vis, ref["aggrs"])
            faces = raster.visibility(tfv, isz, anti_aliasing=True, want_faces=True, **UMR).cpu().numpy()
            want = np.zeros((1, F), np.uint8)
            want[0, ref["aggrs"][0, 1].astype(np.int64)] = 1   # -1 (background) marks face F-1, like the reference
            assert np.array_equal(faces, want) and faces[0, F - 1] == 1


GENERIC = [("hard", "sum", "surface", "softmax"), ("barycentric", "hard", "vertex", "hard"),
           ("euclidean", "sum", "vertex", "softmax")]


@pytest.mark.parametrize("F", [65537, 327680])
@pytest.mark.parametrize("dist,alpha,textype,rgb", GENERIC)
def test_large_face_ladder_generic(F, dist, alpha, textype, rgb):
    """The generic kernels list and consume the faces in 65536-face windows, pixel state carried across them."""
    isz = 32
    fv, tex = _mesh(F, seed=1)
    if textype == "vertex":
        tex = np.random.default_rng(2).uniform(0, 1, size=(1, F, 3, 3)).astype(np.float32)
    g = np.random.default_rng(F).normal(size=(1, 4, isz, isz)).astype(np.float32)
    kw = dict(SOFT, **_mode_kw(dist, alpha, textype, rgb))
    ref = oracle(fv, tex, isz, True, g, **kw)
    got = gpu(fv, tex, isz, True, g, **kw)
    check(got, ref, rgb, "F=%d" % F)
    _last_face_is_live(got, ref, rgb)
    modes = dict(SOFT, dist=raster.FUNC_DIST[dist], alpha=raster.FUNC_ALPHA[alpha], texture=raster.FUNC_SAMPLE[textype])
    _vs_reference_planes(fv, tex, isz, got, rgb, **modes)


@pytest.mark.parametrize("mode", ["umr", "generic"])
def test_131071_faces_inside_one_tile(mode):
    """Every face of a 131071-face mesh inside one tile (|x|, |y| < 0.25 of a 48-pixel raster): tile lists longer
    than one 65536-face window, in both tilings."""
    fv, tex = _mesh(131071)
    c = fv[:, :, 0::3].mean(), fv[:, :, 1::3].mean()
    fv[:, :, 0::3] = (fv[:, :, 0::3] - c[0]) * 0.3
    fv[:, :, 1::3] = (fv[:, :, 1::3] - c[1]) * 0.3
    assert np.abs(fv[:, :, 0::3]).max() < 0.25 and np.abs(fv[:, :, 1::3]).max() < 0.25
    isz = 24
    g = np.random.default_rng(1).normal(size=(1, 4, isz, isz)).astype(np.float32)
    kw = dict(UMR) if mode == "umr" else dict(SOFT, **_mode_kw("barycentric", "sum", "surface", "softmax"))
    ref = oracle(fv, tex, isz, True, g, **kw)
    for tile in ((16, 32) if mode == "umr" else (0,)):
        got = gpu(fv, tex, isz, True, g, tile=tile, **kw)
        check(got, ref, "softmax", "tile=%d" % tile)
    assert np.abs(ref["grad_faces"]).max() > 0 and (ref["images"][:, 3] > 0).sum() > 8


def _pool_cursor(ws, B, F, S):
    """Entries the coarse bins asked of the wide pool (the layout of raster.cu ws_layout)."""
    a = lambda x: (x + 255) // 256 * 256  # noqa: E731
    n = B * F
    ncb = (S + 63) // 64
    off = a(n * 128) + a(n * 16) + a(n * 16) + a(B * 16)
    cur = off + B * ncb * ncb * 8
    return int(ws[cur:cur + 8].cpu().numpy().view(np.uint64)[0])


def test_coarse_pool_overflow_walks_every_face():
    """Bins that do not fit the wide coarse-list pool (8 entries per face) walk all faces: same planes, bit for bit.
    8192 of the 65536 faces are large slivers behind the far plane whose cull boxes meet all 64 bins of a 512-pixel
    raster, so the bins ask for more than the pool holds."""
    if _REF_NOFMA is None:
        pytest.skip("oracle/_ref/soft_rasterize_ref_nofma.so not built")
    fv, tex = _mesh(65536)
    big = np.array([-0.95, -0.95, 150.0, 0.95, -0.9, 150.0, 0.9, 0.95, 150.0], np.float32)
    fv[0, :8192] = big + np.random.default_rng(3).uniform(-0.01, 0.01, size=(8192, 9)).astype(np.float32)
    isz, S = 256, 512
    lib = _lib.load()
    B, F = 1, fv.shape[1]
    p = raster.make_params(B, F, tex.shape[2], isz, True, (0, 0, 0), 1, 100, True, 1e-3, UMR["sigma_val"], "euclidean",
                           UMR["dist_eps"], UMR["gamma_val"], "softmax", "prod", "surface")
    tfv, ttex = torch.from_numpy(fv).to(DEV), torch.from_numpy(tex).to(DEV)
    images = torch.empty(B, 4, isz, isz, device=DEV)
    colors = torch.empty(B, 4, S, S, device=DEV)
    aggrs = torch.empty(B, 2, S, S, device=DEV)
    p2f = torch.empty(B, F, 2, device=DEV)
    ws = torch.empty(lib.umr_raster_workspace_bytes(B, F, isz, 1), device=DEV, dtype=torch.uint8)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    r = lib.umr_raster_forward(ptr(tfv), ptr(ttex), ptr(images), ptr(colors), ptr(aggrs), ptr(p2f), ctypes.byref(p), ptr(ws),
                               ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check(r, "umr_raster_forward")
    torch.cuda.synchronize()
    assert _pool_cursor(ws, B, F, S) > 8 * B * F
    rcol, rp2f, raggr, _ = rc.ref_forward(_REF_NOFMA, tfv, ttex, S, raster.FUNC_RGB["softmax"])
    assert torch.equal(colors, rcol) and torch.equal(aggrs, raggr)
    assert torch.equal(images, TF.avg_pool2d(rcol, 2, 2))
    assert np.allclose(p2f.cpu().numpy(), rp2f.cpu().numpy(), rtol=1e-4, atol=1e-6)


def test_soft_renderer_camera_hypotheses_on_icosphere7():
    """`nnutils.smr.SoftRenderer` forward + backward with 4 camera hypotheses per mesh of a 327680-face icosphere(7):
    the wide path through the fused vertex kernels and shared textures, against the same renders with the hypotheses
    expanded into a plain batch."""
    from umr_b200.nnutils import smr
    v, f = synth.icosphere(7)
    rng = np.random.default_rng(5)
    B, H, isz = 2, 4, 64
    verts = torch.from_numpy(synth.bird_like(v, rng, B)).to(DEV)
    faces = torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1).to(DEV)
    cams = torch.from_numpy(np.stack([synth.cameras(rng, H) for _ in range(B)])).view(-1, 7).to(DEV)
    tex0 = torch.rand(B, f.shape[0], 4, 3, device=DEV)
    g = torch.randn(B * H, 4, isz, isz, device=DEV)
    outs = []
    for expand in (False, True):
        vv = verts.clone().requires_grad_(True)
        tt = tex0.clone().requires_grad_(True)
        r = smr.SoftRenderer(isz, "softmax")
        if expand:
            img, _, _ = r(vv.repeat_interleave(H, 0), faces.repeat_interleave(H, 0), cams, tt.repeat_interleave(H, 0))
        else:
            img, _, _ = r(vv, faces, cams, tt)
        img.backward(g)
        outs.append((img.detach(), vv.grad, tt.grad))
    assert torch.equal(outs[0][0], outs[1][0])
    assert (outs[0][0][:, 3] > 0).sum() > 100
    for a, b in zip(outs[0][1:], outs[1][1:]):
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6 * float(b.abs().max()) + 1e-7)
        assert float(b.abs().max()) > 0
