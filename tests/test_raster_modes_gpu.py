"""GPU parity across the rasteriser's whole accepted input range, vs CPU oracle B (held bit-exact to the reference's
own code in every mode by test_raster_modes_cpu.py), with the rules of test_raster_edge_gpu.both: 1e-4 relative,
gradients with an atol scaled to the tensor's magnitude, hard-RGB depth / face-id planes bit-exact.

* texture ladder: texture_res 1 .. 257, i.e. texel indices past the 14 / 16 bits a pair record once held, through both
  forward tilings and a full / partial / absent pair buffer;
* all 34 generic mode combinations (every mode but euclidean / prod / surface), at whole tiles with anti-aliasing and
  at an odd size without, and against the reference's own CUDA kernels built with -fmad=false where available;
* shared textures and texture-only gradients in the generic kernels;
* face counts from one cull-box piece (2048) up to the ABI's limit (65535), with the highest face indices on screen."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

import softras
from umr_b200 import _lib, raster, synth
from util import rel_report, scene

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import ref_gpu_compare as rc  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
UMR = dict(sigma_val=1e-5, dist_eps=1e-10, gamma_val=1e-4)
SOFT = dict(sigma_val=1e-4, dist_eps=1e-4, gamma_val=1e-3)   # wider soft edges for the generic modes
PAIR_BUFFERS = {"full": 32.0, "partial": 0.7, "none": 0.0}   # raster.PAIR_CAND_PER_PIXEL


def oracle(fv, tex, isz, aa, g, **kw):
    img, fwd, cfg = softras.render(fv, tex, isz, anti_aliasing=aa, impl="B", **kw)
    gf, gt = softras.render_backward(fwd, cfg, g, anti_aliasing=aa, impl="B")
    return dict(images=img, aggrs=fwd["aggrs_info"], p2f=fwd["p2f_info"], grad_faces=gf, grad_tex=gt)


def gpu(fv, tex, isz, aa, g, tile=0, cand=32.0, geom_grad=True, tex_grad=True, **kw):
    """One forward + backward through the autograd binding; `stats` = the pair buffer's [blocks wanted, tiles unsaved]."""
    old = raster.PAIR_CAND_PER_PIXEL, raster.FORWARD_TILE, raster.PAIR_ADAPTIVE
    raster.PAIR_CAND_PER_PIXEL, raster.FORWARD_TILE, raster.PAIR_ADAPTIVE = cand, tile, False
    try:
        tfv = torch.from_numpy(fv).to(DEV).requires_grad_(geom_grad)
        ttex = torch.from_numpy(tex).to(DEV).requires_grad_(tex_grad)
        img, p2f, aggr = raster.soft_rasterize(tfv, ttex, isz, anti_aliasing=aa, **kw)
        saved = img.grad_fn.saved_tensors
        stats = saved[4][:8].view(torch.int32).cpu().tolist() if len(saved) == 5 else None
        img.backward(torch.from_numpy(g).to(DEV))
        torch.cuda.synchronize()
    finally:
        raster.PAIR_CAND_PER_PIXEL, raster.FORWARD_TILE, raster.PAIR_ADAPTIVE = old
    return dict(images=img.detach().cpu().numpy(), aggrs=aggr.cpu().numpy(), p2f=p2f.cpu().numpy(),
                grad_faces=tfv.grad.cpu().numpy() if geom_grad else None,
                grad_tex=ttex.grad.cpu().numpy() if tex_grad else None, stats=stats)


def check(got, ref, rgb, what=""):
    ok, msgs = True, []
    for name in ("images", "aggrs", "p2f", "grad_faces", "grad_tex"):
        if got.get(name) is None:
            continue
        b = ref[name]
        at = 1e-6 * float(np.abs(b).max() + 1e-30) + 1e-7 if name.startswith("grad") else 1e-6
        o, m = rel_report(name, got[name], b, 1e-4, at)
        ok &= o
        msgs.append(m)
    if rgb == "hard":
        ex = np.array_equal(got["aggrs"], ref["aggrs"])
        msgs.append("hard planes bit-exact: %s" % ex)
        ok &= ex
    assert ok, what + "\n" + "\n".join(msgs)


# ---------------------------------------------------------------------------------------------------------------------
# texture ladder
# ---------------------------------------------------------------------------------------------------------------------
def _large_faces(tex_res):
    """80 large faces (icosphere(1)) over most of an 80 px image (S = 160); the same mesh at every texture size."""
    rng = np.random.default_rng(129)
    v, f = synth.icosphere(1)
    fv = synth.raster_space_faces(synth.bird_like(v, rng, 2), f, synth.cameras(rng, 2))
    tex = np.random.default_rng(tex_res).uniform(0, 1, size=(2, f.shape[0], tex_res * tex_res, 3)).astype(np.float32)
    return fv, tex


def _texel_gradient_reaches(gt, index):
    return bool(np.abs(gt[:, :, index:]).max() > 0) if gt.shape[2] > index else False


LADDER = [(r, rgb, True) for r in (1, 7, 64, 128, 129, 200, 256, 257) for rgb in ("softmax", "hard")] + \
         [(129, "softmax", False), (257, "softmax", False)]   # single-sided past the old 14- and 16-bit fields


@pytest.mark.parametrize("tex_res,rgb,fill_back", LADDER)
def test_texture_ladder(tex_res, rgb, fill_back):
    """The pair record keeps the sampled texel's index for the streamed backward.  Large faces sample texels along the
    whole [0, T2) range (texel_index's mirrored half sends the c1 ~ 0 strip to indices >= (R-1)R), so past 2^14 / 2^16
    a field too narrow for the index sends texel gradients to the wrong texel and can flip the record's front bit."""
    isz = 80
    fv, tex = _large_faces(tex_res)
    g = np.random.default_rng(3).normal(size=(2, 4, isz, isz)).astype(np.float32)
    kw = dict(UMR, aggr_func_rgb=rgb, fill_back=fill_back)
    ref = oracle(fv, tex, isz, True, g, **kw)
    # the ladder is not vacuous: the oracle's gradient reaches the texels a narrow field would lose
    if tex_res >= 129:
        assert _texel_gradient_reaches(ref["grad_tex"], 1 << 14)
    if tex_res >= 257:
        assert _texel_gradient_reaches(ref["grad_tex"], 1 << 16)
    for tile in (16, 32):
        for buf, cand in PAIR_BUFFERS.items():
            got = gpu(fv, tex, isz, True, g, tile=tile, cand=cand, **kw)
            if buf == "none":
                assert got["stats"] is None
            else:
                assert got["stats"][0] > 0 and (got["stats"][1] == 0) == (buf == "full"), (buf, got["stats"])
            check(got, ref, rgb, "texture_res=%d tile=%d pair buffer=%s" % (tex_res, tile, buf))


def test_texture_past_the_32x32_record_field_recomputes():
    """T2 = 1449^2 > 2^21 does not fit the 32x32-tile record's texel field: that forward saves nothing and the backward
    recomputes every tile (16x16 tiles still save: 23 bits).  Two faces covering most of the image."""
    R, isz = 1449, 48
    fv = np.array([[[-0.9, -0.8, 5.0, 0.85, -0.9, 5.5, -0.8, 0.9, 6.0],
                    [0.85, -0.9, 5.5, 0.9, 0.85, 6.5, -0.8, 0.9, 6.0]]], dtype=np.float32)
    tex = np.random.default_rng(4).uniform(0, 1, size=(1, 2, R * R, 3)).astype(np.float32)
    g = np.random.default_rng(5).normal(size=(1, 4, isz, isz)).astype(np.float32)
    ref = oracle(fv, tex, isz, True, g, **UMR)
    assert _texel_gradient_reaches(ref["grad_tex"], 1 << 21)
    for tile in (16, 32):
        check(gpu(fv, tex, isz, True, g, tile=tile, cand=32.0, **UMR), ref, "softmax", "tile=%d" % tile)


# ---------------------------------------------------------------------------------------------------------------------
# generic modes
# ---------------------------------------------------------------------------------------------------------------------
GENERIC = [(d, a, t, r) for d in ("hard", "barycentric", "euclidean") for a in ("hard", "sum", "prod")
           for t in ("surface", "vertex") for r in ("softmax", "hard") if (d, a, t) != ("euclidean", "prod", "surface")]
assert len(GENERIC) == 34
_REF_NOFMA = rc.load("soft_rasterize_ref_nofma")


def _generic_inputs(textype, tex_res, B=2, seed=9):
    fv, tex = scene(B, 2, tex_res, seed=seed)   # 320 faces
    if textype == "vertex":
        tex = np.random.default_rng(seed + 1).uniform(0, 1, size=(B, fv.shape[1], 3, 3)).astype(np.float32)
    return fv, tex


def _mode_kw(dist, alpha, textype, rgb):
    return dict(dist_func=dist, aggr_func_alpha=alpha, texture_type=textype, aggr_func_rgb=rgb)


def _vs_reference_kernels(fv, tex, isz, aa, g, got, dist, alpha, textype, rgb, fill_back):
    """The reference's CUDA kernels built with -fmad=false: same IEEE operation sequence and device expf, so every pixel
    plane must be bit-identical; p2f and vertex gradients differ by float-atomics order only."""
    S = isz * (2 if aa else 1)
    tfv, ttex = torch.from_numpy(fv).to(DEV), torch.from_numpy(tex).to(DEV)
    modes = dict(SOFT, dist=raster.FUNC_DIST[dist], alpha=raster.FUNC_ALPHA[alpha], texture=raster.FUNC_SAMPLE[textype],
                 double_side=fill_back)
    rgb_id = raster.FUNC_RGB[rgb]
    colors, rp2f, raggr, finfo = rc.ref_forward(_REF_NOFMA, tfv, ttex, S, rgb_id, **modes)
    rimg = TF.avg_pool2d(colors, 2, 2) if aa else colors
    assert np.array_equal(got["images"], rimg.cpu().numpy()), "images not bit-exact with the reference kernels"
    assert np.array_equal(got["aggrs"], raggr.cpu().numpy()), "aggregation planes not bit-exact with the reference kernels"
    assert np.allclose(got["p2f"], rp2f.cpu().numpy(), rtol=1e-4, atol=1e-6)
    tg = torch.from_numpy(g).to(DEV)
    ghi = (tg / 4).repeat_interleave(2, dim=2).repeat_interleave(2, dim=3) if aa else tg
    rgf, _ = rc.ref_backward(_REF_NOFMA, tfv, ttex, colors, finfo, raggr, ghi, S, rgb_id, **modes)
    rgf = rgf.cpu().numpy()
    assert np.allclose(got["grad_faces"], rgf, rtol=1e-3, atol=1e-5 * float(np.abs(rgf).max()))


@pytest.mark.parametrize("dist,alpha,textype,rgb", GENERIC)
def test_generic_mode(dist, alpha, textype, rgb):
    """Each generic combination at (anti-aliased, whole 16x16 tiles: the shared-staged 128-bit store epilogue) and at
    (no anti-aliasing, odd size: partial tiles, the per-pixel stores).  fill_back alternates over the list and surface
    textures take T2 = 1, 4, 9 in turn."""
    for isz, aa, fill_back, fv, tex, g, kw in _generic_cases(dist, alpha, textype, rgb):
        ref = oracle(fv, tex, isz, aa, g, **kw)
        got = gpu(fv, tex, isz, aa, g, **kw)
        check(got, ref, rgb, "%s isz=%d aa=%s fill_back=%s T2=%d" % ((dist, alpha, textype, rgb), isz, aa, fill_back,
                                                                     tex.shape[2]))


@pytest.mark.skipif(_REF_NOFMA is None, reason="oracle/_ref/soft_rasterize_ref_nofma.so not built")
@pytest.mark.parametrize("dist,alpha,textype,rgb", GENERIC)
def test_generic_mode_bit_exact_with_reference_kernels(dist, alpha, textype, rgb):
    for isz, aa, fill_back, fv, tex, g, kw in _generic_cases(dist, alpha, textype, rgb):
        got = gpu(fv, tex, isz, aa, g, **kw)
        _vs_reference_kernels(fv, tex, isz, aa, g, got, dist, alpha, textype, rgb, fill_back)


def _generic_cases(dist, alpha, textype, rgb):
    i = GENERIC.index((dist, alpha, textype, rgb))
    fill_back = i % 2 == 0
    fv, tex = _generic_inputs(textype, 1 + i % 3, seed=9 + i)
    kw = dict(SOFT, fill_back=fill_back, **_mode_kw(dist, alpha, textype, rgb))
    for isz, aa in ((32, True), (37, False)):
        g = np.random.default_rng(i).normal(size=(2, 4, isz, isz)).astype(np.float32)
        yield isz, aa, fill_back, fv, tex, g, kw


def test_generic_forward_without_anti_aliasing_into_separate_soft_colors():
    """Through the C ABI without anti-aliasing, `images` and `soft_colors` may be different buffers: both receive the
    raster-resolution planes (the binding passes one buffer, so only a direct call reaches the second store)."""
    lib = _lib.load()
    fv, tex = _generic_inputs("surface", 2)
    B, F, S = fv.shape[0], fv.shape[1], 37
    kw = dict(SOFT, dist_func="barycentric", aggr_func_alpha="sum", texture_type="surface", aggr_func_rgb="softmax")
    p = raster.make_params(B, F, tex.shape[2], S, False, (0.1, 0.2, 0.3), 1, 100, True, 1e-3, kw["sigma_val"], "barycentric",
                           kw["dist_eps"], kw["gamma_val"], "softmax", "sum", "surface")
    ref = oracle(fv, tex, S, False, np.zeros((B, 4, S, S), np.float32), background_color=(0.1, 0.2, 0.3), **kw)
    tfv, ttex = torch.from_numpy(fv).to(DEV), torch.from_numpy(tex).to(DEV)
    images = torch.full((B, 4, S, S), -7.0, device=DEV)
    colors = torch.full((B, 4, S, S), -7.0, device=DEV)
    aggrs = torch.empty(B, 2, S, S, device=DEV)
    p2f = torch.empty(B, F, 2, device=DEV)
    ws = torch.empty(lib.umr_raster_workspace_bytes(B, F, S, 0), device=DEV, dtype=torch.uint8)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc_ = lib.umr_raster_forward(ptr(tfv), ptr(ttex), ptr(images), ptr(colors), ptr(aggrs), ptr(p2f), ctypes.byref(p), ptr(ws),
                                 ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check(rc_, "umr_raster_forward")
    torch.cuda.synchronize()
    assert torch.equal(images, colors)
    check(dict(images=images.cpu().numpy(), aggrs=aggrs.cpu().numpy(), p2f=p2f.cpu().numpy()), ref, "softmax")


@pytest.mark.parametrize("dist,alpha,textype,rgb", [("barycentric", "sum", "vertex", "softmax"),
                                                    ("hard", "hard", "surface", "hard"),
                                                    ("euclidean", "sum", "surface", "softmax")])
@pytest.mark.parametrize("groups", [1, 2])   # textures [G=1 (batch-shared) | 2, F, T2, 3] for B = 4 renders
def test_generic_shared_textures_equal_expanded_copies(dist, alpha, textype, rgb, groups):
    B, isz = 4, 32
    fv, tex = _generic_inputs(textype, 2, B=B, seed=31)
    tex = np.ascontiguousarray(tex[:groups])
    g = np.random.default_rng(8).normal(size=(B, 4, isz, isz)).astype(np.float32)
    kw = dict(SOFT, **_mode_kw(dist, alpha, textype, rgb))
    outs = []
    for shared in (True, False):
        tfv = torch.from_numpy(fv).to(DEV).requires_grad_(True)
        t = torch.from_numpy(tex).to(DEV).requires_grad_(True)
        tin = t if shared else t.repeat_interleave(B // groups, dim=0)
        img, p2f, aggr = raster.soft_rasterize(tfv, tin, isz, anti_aliasing=True, **kw)
        img.backward(torch.from_numpy(g).to(DEV))
        outs.append((img.detach().cpu().numpy(), aggr.cpu().numpy(), tfv.grad.cpu().numpy(), t.grad.cpu().numpy()))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
    for k, name in ((2, "grad_faces"), (3, "grad_tex (group sum)")):
        b = outs[1][k]
        ok, msg = rel_report(name, outs[0][k], b, 1e-4, 1e-6 * float(np.abs(b).max()) + 1e-7)
        assert ok, msg
    assert outs[0][3].shape == tex.shape and np.abs(outs[0][3]).max() > 0


@pytest.mark.parametrize("dist,alpha,textype,rgb", [("barycentric", "prod", "vertex", "softmax"),
                                                    ("hard", "sum", "surface", "hard")])
def test_generic_texture_only_gradient(dist, alpha, textype, rgb):
    fv, tex = _generic_inputs(textype, 3)
    g = np.random.default_rng(2).normal(size=(2, 4, 32, 32)).astype(np.float32)
    kw = dict(SOFT, **_mode_kw(dist, alpha, textype, rgb))
    ref = oracle(fv, tex, 32, True, g, **kw)
    got = gpu(fv, tex, 32, True, g, geom_grad=False, **kw)
    check(got, ref, rgb)
    assert np.abs(got["grad_tex"]).max() > 0


# ---------------------------------------------------------------------------------------------------------------------
# face ladder
# ---------------------------------------------------------------------------------------------------------------------
def _ladder_mesh(F, B=1, seed=0):
    """The F faces of a deformed icosphere(6) nearest the image centre, ordered so that the highest indices are the
    near-side faces closest to the pixel centre (1/64, 1/64) of a 64-pixel raster: face F-1 covers that pixel, in front."""
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(6)
    fv = synth.raster_space_faces(synth.bird_like(v, rng, B), f, synth.cameras(rng, B))
    c = fv[0].reshape(-1, 3, 3).mean(axis=1)
    near = c[:, 2] < np.median(c[:, 2])
    order = np.lexsort((-np.hypot(c[:, 0] - 1 / 64, c[:, 1] - 1 / 64), near))   # far side first, then nearer the pixel
    fv = np.ascontiguousarray(fv[:, order[-F:]])
    tex = rng.uniform(0, 1, size=(B, F, 4, 3)).astype(np.float32)
    return fv, tex


def _last_face_is_live(got, ref, rgb):
    """Face F-1 (the top of the u16 face fields at F = 65535) gets its p2f and its gradients (a face alone at its pixels
    under hard distance has colour == texel, hence no vertex gradient: then its texel gradient)."""
    if rgb != "softmax":
        return
    F = got["grad_faces"].shape[1]
    for out in (ref, got):
        assert np.abs(out["p2f"][:, F - 1]).max() > 0
        assert max(np.abs(out["grad_faces"][:, F - 1]).max(), np.abs(out["grad_tex"][:, F - 1]).max()) > 0


@pytest.mark.parametrize("F", [2048, 2049, 4097, 20480, 65535])
def test_face_ladder_umr_configuration(F):
    """UMR's kernels at F = one cull-box piece, one more, two pieces + 1, and up to the u16 face fields' top: both
    tilings with every pair-buffer state, the visibility planes and the visible-face bytes."""
    isz = 32
    fv, tex = _ladder_mesh(F)
    g = np.random.default_rng(F).normal(size=(1, 4, isz, isz)).astype(np.float32)
    for rgb in ("softmax", "hard"):
        ref = oracle(fv, tex, isz, True, g, aggr_func_rgb=rgb, **UMR)
        for tile in (16, 32):
            for buf, cand in PAIR_BUFFERS.items():
                got = gpu(fv, tex, isz, True, g, tile=tile, cand=cand, aggr_func_rgb=rgb, **UMR)
                check(got, ref, rgb, "F=%d tile=%d pair buffer=%s" % (F, tile, buf))
                _last_face_is_live(got, ref, rgb)
        if rgb == "hard":
            tfv = torch.from_numpy(fv).to(DEV)
            vis = raster.visibility(tfv, isz, anti_aliasing=True, **UMR).cpu().numpy()
            assert np.array_equal(vis, ref["aggrs"])
            faces = raster.visibility(tfv, isz, anti_aliasing=True, want_faces=True, **UMR).cpu().numpy()
            want = np.zeros((1, F), np.uint8)
            want[0, ref["aggrs"][0, 1].astype(np.int64)] = 1   # -1 (background) marks face F-1, like the reference
            assert np.array_equal(faces, want) and faces[0, F - 1] == 1


@pytest.mark.parametrize("F", [2048, 2049, 4097, 20480, 65535])
@pytest.mark.parametrize("dist,alpha,textype,rgb", [("hard", "sum", "surface", "softmax"),
                                                    ("barycentric", "hard", "vertex", "hard"),
                                                    ("euclidean", "sum", "vertex", "softmax")])
def test_face_ladder_generic(F, dist, alpha, textype, rgb):
    """The generic kernels keep the whole tile list in shared memory (128 KB at 65535 faces) and stage the cull boxes
    in 2048-face pieces."""
    isz = 32
    fv, tex = _ladder_mesh(F, seed=1)
    if textype == "vertex":
        tex = np.random.default_rng(2).uniform(0, 1, size=(1, F, 3, 3)).astype(np.float32)
    g = np.random.default_rng(F).normal(size=(1, 4, isz, isz)).astype(np.float32)
    kw = dict(SOFT, **_mode_kw(dist, alpha, textype, rgb))
    ref = oracle(fv, tex, isz, True, g, **kw)
    got = gpu(fv, tex, isz, True, g, **kw)
    check(got, ref, rgb, "F=%d" % F)
    _last_face_is_live(got, ref, rgb)


@pytest.mark.parametrize("mode", ["umr", "generic"])
def test_65535_faces_inside_one_tile(mode):
    """Every face of the largest mesh inside one tile (|x|, |y| < 0.25 of a 48-pixel raster: raster pixels 16-31 of
    the 16x16 tiling, 0-31 of the 32x32 one): tile lists 65535 long."""
    fv, tex = _ladder_mesh(65535)
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
