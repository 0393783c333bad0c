"""The float64 rasteriser (umr_raster_forward_f64 / umr_raster_backward_f64, float64 `soft_rasterize`) on the GPU.

* parity with CPU oracle B's double instantiation (held bit-exact to the reference's own code on the host by
  test_raster_f64_cpu.py) over every mode combination, the bird scene, shared textures and the ends of the input range;
* bit-exact pixel planes against the reference's own CUDA kernels run in double, where they are built;
* bitwise reproducibility, torch.autograd.gradcheck, the dtype contract, and the fp32-vs-fp64 spread the path exists to show.

Tolerances.  Hard-mode depth / face-index planes and hard-mode RGB pass through no exp: bit-exact.  Everything else is held to
RTOL = 1e-11 (CUDA's and glibc's double exp differ by an ulp, which the sigmoid's 1 / sigma slope carries into D) with the
absolute floors ATOL_* below: 1e-13 on values of order one (planes, p2f) and 1e-11 of the tensor's largest magnitude on
gradients, which are sums of thousands of signed terms per element."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

import softras
from umr_b200 import _lib, raster, synth
from umr_b200 import soft_renderer as sr
from umr_b200.nnutils import geom_utils, smr
from util import rel_report, scene

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import ref_gpu_compare as rc  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
UMR = dict(sigma_val=1e-5, dist_eps=1e-10, gamma_val=1e-4)
SOFT = dict(sigma_val=1e-4, dist_eps=1e-4, gamma_val=1e-3)
RTOL, ATOL_PLANE, ATOL_GRAD_REL = 1e-11, 1e-13, 1e-11
BG = (0.25, 0.5, 0.75)   # exact in float32: UmrRasterParams carries the background as float
_REF_NOFMA = rc.load("soft_rasterize_ref_nofma")


def kernel_grid(S, dtype=np.float64):
    """The p2f grid of the kernels: torch's float32 linspace(-1, 1, S) by its per-element definition (start + step * i in the
    lower half, end - step * (S - 1 - i) in the upper), widened.  torch's vectorised CPU linspace, which
    softras.standard_grid calls, rounds some elements one float ulp away from it, so the oracle is handed this grid."""
    step = np.float32(2.0) / np.float32(S - 1)
    i = np.arange(S)
    lo = (np.float32(-1.0) + step * i.astype(np.float32)).astype(np.float32)
    hi = (np.float32(1.0) - step * (S - 1 - i).astype(np.float32)).astype(np.float32)
    x = np.where(i * 2 < S, lo, hi)
    return np.ascontiguousarray(np.stack(np.broadcast_arrays(x[None, :], x[:, None]), axis=-1).astype(dtype))


@pytest.fixture(autouse=True)
def _oracle_on_the_kernel_grid(monkeypatch):
    monkeypatch.setattr(softras, "standard_grid", kernel_grid)


def test_kernel_grid_is_affine_grid_to_one_float_ulp():
    for S in (2, 37, 64, 202, 512):
        g = kernel_grid(S, np.float32)
        ref = TF.affine_grid(torch.tensor([[[1., 0, 0], [0, 1, 0]]]), (1, 1, S, S), align_corners=True)[0].numpy()
        assert g.shape == ref.shape and np.abs(g - ref).max() <= 2.0 ** -23
        dev = TF.affine_grid(torch.tensor([[[1., 0, 0], [0, 1, 0]]], device=DEV), (1, 1, S, S), align_corners=True)[0].cpu().numpy()
        assert np.abs(g - dev).max() <= 2.0 ** -23


def _eps_for_oracle(gamma):
    """kernel.cu:337 seeds the softmax with expf(eps / gamma), a float expression: the device's expf and glibc's round it
    differently for some arguments (by one float ulp at UMR's eps / gamma = 10.000001, 9e-8 of every background weight),
    which is not a property of the kernels.  The comparisons with the CPU oracle use an eps for which the two agree; the
    comparison with the reference's CUDA kernels runs UMR's."""
    libm = ctypes.CDLL("libm.so.6")
    libm.expf.restype, libm.expf.argtypes = ctypes.c_float, [ctypes.c_float]
    for eps in (1e-3, 2e-3, 5e-4, 1.5e-3, 3e-3, 7e-4, 1e-4):
        q = np.float32(eps) / np.float32(gamma)
        if float(torch.exp(torch.tensor(float(q), dtype=torch.float32, device=DEV))) == libm.expf(float(q)):
            return eps
    raise AssertionError("no eps found")


def umr_oracle_kw():
    return dict(UMR, eps=_eps_for_oracle(UMR["gamma_val"]))


def widen(a, seed):
    """float32 test inputs as genuine doubles: widened, then perturbed below float32 resolution."""
    a = np.asarray(a, np.float64)
    return a + np.random.default_rng(seed).normal(size=a.shape) * 1e-9 * (np.abs(a) + 1e-3)


def oracle(fv, tex, isz, aa, g, **kw):
    S = isz * (2 if aa else 1)
    cfg = softras.RasterCfg(S, **kw)
    fwd = softras.forward(fv, tex, cfg, impl="B", dtype=np.float64)
    out = dict(images=softras.avg_pool2(fwd["soft_colors"]) if aa else fwd["soft_colors"], aggrs=fwd["aggrs_info"],
               p2f=fwd["p2f_info"])
    if g is not None:
        ghi = softras.avg_pool2_backward(np.asarray(g, np.float64)) if aa else np.asarray(g, np.float64)
        out["grad_faces"], out["grad_tex"] = softras.backward(fwd, ghi, cfg, impl="B")
    return out


def gpu(fv, tex, isz, aa, g, geom_grad=True, tex_grad=True, **kw):
    tfv = torch.from_numpy(fv).to(DEV).requires_grad_(geom_grad and g is not None)
    ttex = torch.from_numpy(tex).to(DEV).requires_grad_(tex_grad and g is not None)
    img, p2f, aggr = raster.soft_rasterize(tfv, ttex, isz, anti_aliasing=aa, **kw)
    assert img.dtype == p2f.dtype == aggr.dtype == torch.float64
    if g is not None:
        img.backward(torch.from_numpy(np.asarray(g, np.float64)).to(DEV))
    torch.cuda.synchronize()
    return dict(images=img.detach().cpu().numpy(), aggrs=aggr.cpu().numpy(), p2f=p2f.cpu().numpy(),
                grad_faces=tfv.grad.cpu().numpy().reshape(fv.shape[0], -1, 9) if tfv.grad is not None else None,
                grad_tex=ttex.grad.cpu().numpy() if ttex.grad is not None else None)


def check(got, ref, rgb, what=""):
    ok, msgs = True, []
    for name in ("images", "aggrs", "p2f", "grad_faces", "grad_tex"):
        if got.get(name) is None or ref.get(name) is None:
            continue
        b = ref[name]
        at = ATOL_GRAD_REL * float(np.abs(b).max()) + 1e-300 if name.startswith("grad") else ATOL_PLANE
        o, m = rel_report(name, got[name], b, RTOL, at)
        ok &= o and bool(np.array_equal(np.isnan(got[name]), np.isnan(b)))
        msgs.append(m)
    if rgb == "hard":
        ex = np.array_equal(got["aggrs"], ref["aggrs"]) and np.array_equal(got["images"][:, :3], ref["images"][:, :3])
        msgs.append("hard depth / face-index / RGB planes bit-exact: %s" % ex)
        ok &= ex
    assert ok, what + "\n" + "\n".join(msgs)


# ---------------------------------------------------------------------------------------------------------------------
# parity with oracle B in double
# ---------------------------------------------------------------------------------------------------------------------
MODES = [(d, a, t, r) for d in ("hard", "barycentric", "euclidean") for a in ("hard", "sum", "prod")
         for t in ("surface", "vertex") for r in ("softmax", "hard")]


def _mode_inputs(textype, tex_res, B=2, seed=9):
    fv, tex = scene(B, 2, tex_res, seed=seed)   # 320 faces
    if textype == "vertex":
        tex = np.random.default_rng(seed + 1).uniform(0, 1, size=(B, fv.shape[1], 3, 3))
    return widen(fv, seed), widen(tex, seed + 2)


@pytest.mark.parametrize("dist,alpha,textype,rgb", MODES)
def test_every_mode(dist, alpha, textype, rgb):
    """Anti-aliased whole tiles and an odd size without; fill_back alternates over the list, surface textures take
    T2 = 1, 4, 9 in turn."""
    i = MODES.index((dist, alpha, textype, rgb))
    fill_back = i % 2 == 0
    fv, tex = _mode_inputs(textype, 1 + i % 3, seed=9 + i)
    kw = dict(SOFT, fill_back=fill_back, dist_func=dist, aggr_func_alpha=alpha, texture_type=textype, aggr_func_rgb=rgb,
              background_color=BG)
    for isz, aa in ((32, True), (37, False)):
        g = np.random.default_rng(i).normal(size=(2, 4, isz, isz))
        check(gpu(fv, tex, isz, aa, g, **kw), oracle(fv, tex, isz, aa, g, **kw), rgb, "%s isz=%d aa=%s fill_back=%s"
              % ((dist, alpha, textype, rgb), isz, aa, fill_back))


@pytest.mark.parametrize("rgb", ["softmax", "hard"])
@pytest.mark.parametrize("tex_res", [1, 6])
@pytest.mark.parametrize("isz,aa", [(128, True), (101, False)])
def test_bird_scene(rgb, tex_res, isz, aa):
    """The icosphere bird (1280 faces) in UMR's configuration, T2 = 1 and 36."""
    fv, tex = scene(2, 3, tex_res, seed=3)
    fv, tex = widen(fv, 1), widen(tex, 2)
    g = np.random.default_rng(5).normal(size=(2, 4, isz, isz))
    kw = dict(umr_oracle_kw(), aggr_func_rgb=rgb)
    check(gpu(fv, tex, isz, aa, g, **kw), oracle(fv, tex, isz, aa, g, **kw), rgb)


@pytest.mark.parametrize("groups", [1, 2])
@pytest.mark.parametrize("textype,rgb", [("surface", "softmax"), ("vertex", "softmax"), ("surface", "hard")])
def test_shared_textures(textype, rgb, groups):
    """textures [G, F, T2, 3] for B = 4 renders: planes as with expanded copies, the gradient is the group's sum."""
    B, isz = 4, 32
    fv, tex = _mode_inputs(textype, 2, B=B, seed=31)
    g = np.random.default_rng(8).normal(size=(B, 4, isz, isz))
    kw = dict(SOFT, texture_type=textype, aggr_func_rgb=rgb)
    ref = oracle(fv, np.repeat(tex[:groups], B // groups, axis=0), isz, True, g, **kw)
    ref["grad_tex"] = ref["grad_tex"].reshape(groups, B // groups, *tex.shape[1:]).sum(1)
    got = gpu(fv, np.ascontiguousarray(tex[:groups]), isz, True, g, **kw)
    check(got, ref, rgb)
    only_tex = gpu(fv, np.ascontiguousarray(tex[:groups]), isz, True, g, geom_grad=False, **kw)
    assert only_tex["grad_faces"] is None and np.array_equal(only_tex["grad_tex"], got["grad_tex"])
    only_geom = gpu(fv, np.ascontiguousarray(tex[:groups]), isz, True, g, tex_grad=False, **kw)
    assert only_geom["grad_tex"] is None and np.array_equal(only_geom["grad_faces"], got["grad_faces"])


def test_c_abi_direct_and_validation():
    """Through the C entry points: separate `images` / `soft_colors` without anti-aliasing, p2f_info == NULL, and the
    error codes of the float32 entry points."""
    lib = _lib.load()
    fv, tex = _mode_inputs("surface", 2)
    B, F, S = fv.shape[0], fv.shape[1], 37
    kw = dict(SOFT, dist_func="barycentric", aggr_func_alpha="sum", texture_type="surface", aggr_func_rgb="softmax")
    p = raster.make_params(B, F, tex.shape[2], S, False, BG, 1, 100, True, 1e-3, kw["sigma_val"], "barycentric",
                           kw["dist_eps"], kw["gamma_val"], "softmax", "sum", "surface")
    ref = oracle(fv, tex, S, False, None, background_color=BG, **kw)
    tfv, ttex = torch.from_numpy(fv).to(DEV), torch.from_numpy(tex).to(DEV)
    images = torch.full((B, 4, S, S), -7.0, device=DEV, dtype=torch.float64)
    colors = torch.full_like(images, -7.0)
    aggrs = torch.empty(B, 2, S, S, device=DEV, dtype=torch.float64)
    p2f = torch.empty(B, F, 2, device=DEV, dtype=torch.float64)
    ws = torch.empty(lib.umr_raster_workspace_bytes_f64(B, F, S, 0), device=DEV, dtype=torch.uint8)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr() if t is not None else 0)  # noqa: E731
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.umr_raster_forward_f64(ptr(tfv), ptr(ttex), ptr(images), ptr(colors), ptr(aggrs), ptr(p2f), ctypes.byref(p),
                                          ptr(ws), stream), "umr_raster_forward_f64")
    images2 = torch.empty_like(images)
    _lib.check(lib.umr_raster_forward_f64(ptr(tfv), ptr(ttex), ptr(images2), ptr(None), ptr(aggrs), ptr(None), ctypes.byref(p),
                                          ptr(ws), stream), "umr_raster_forward_f64")
    torch.cuda.synchronize()
    assert torch.equal(images, colors) and torch.equal(images, images2)
    check(dict(images=images.cpu().numpy(), aggrs=aggrs.cpu().numpy(), p2f=p2f.cpu().numpy()), ref, "softmax")
    call = lambda q, w=ws, f=tfv: lib.umr_raster_forward_f64(ptr(f), ptr(ttex), ptr(images), ptr(colors), ptr(aggrs), ptr(p2f),  # noqa: E731
                                                            ctypes.byref(q), ptr(w), stream)
    bad = raster.make_params(B, F, tex.shape[2], S, False, BG, 1, 100, True, 1e-3, 1e-4, "barycentric", 1e-4, 1e-3, "softmax",
                             "sum", "surface")
    bad.color_channels = 4
    assert call(bad) == -2                      # UMR_ERR_BAD_ARG: part maps are float32 only
    bad.color_channels, bad.num_faces = 3, (1 << 24) + 1
    assert call(bad) == -3                      # UMR_ERR_TOO_LARGE
    bad.num_faces, bad.func_id_dist = F, 3
    assert call(bad) == -1                      # UMR_ERR_UNSUPPORTED
    assert call(p, f=None) == -2 and call(p, w=None) == -2
    assert lib.umr_raster_backward_f64(ptr(tfv), ptr(ttex), ptr(colors), ptr(aggrs), ptr(images), ptr(None), ptr(None),
                                       ctypes.byref(p), ptr(ws), stream) == -2
    with pytest.raises(ValueError):
        raster.soft_rasterize(tfv, torch.zeros(B, F, 1, 4, device=DEV, dtype=torch.float64), 32)


# ---------------------------------------------------------------------------------------------------------------------
# the reference's own CUDA kernels, run in double
# ---------------------------------------------------------------------------------------------------------------------
def _ref_f64(fv, tex, S, rgb, g_hi, bg=(0, 0, 0), sigma_val=1e-5, dist_eps=1e-10, gamma_val=1e-4):
    """functional/soft_rasterize.py:41-73 with double buffers and the float32 affine_grid widened (the reference's Python
    wrapper allocates float buffers, so the double instantiation of its kernels is only reachable like this)."""
    B, Fn = fv.shape[:2]
    z = lambda *s: torch.zeros(*s, device=DEV, dtype=torch.float64)  # noqa: E731
    faces_info, aggrs, p2f, p2f_sum = z(B, Fn, 27), z(B, 2, S, S), z(B, Fn, 2), z(B, Fn, 2)
    colors = torch.ones(B, 4, S, S, device=DEV, dtype=torch.float64)
    for k in range(3):
        colors[:, k] = bg[k]
    grid = torch.from_numpy(kernel_grid(S)).to(DEV)   # affine_grid in float32, widened
    args = (1.0, 100.0, 1e-3, sigma_val, 2, float(np.log(1.0 / dist_eps - 1.0)), gamma_val, rgb, 2, 0, True)
    _REF_NOFMA.forward_soft_rasterize(fv, tex, faces_info, aggrs, grid, p2f, p2f_sum, colors, S, *args)
    gf, gt = torch.zeros_like(fv), torch.zeros_like(tex)
    _REF_NOFMA.backward_soft_rasterize(fv, tex, colors, faces_info, aggrs, gf, gt, g_hi.contiguous(), S, *args)
    return colors, p2f / p2f_sum.clamp_min(1e-12), aggrs, gf


@pytest.mark.skipif(_REF_NOFMA is None, reason="oracle/_ref/soft_rasterize_ref_nofma.so not built")
@pytest.mark.parametrize("rgb", ["softmax", "hard"])
@pytest.mark.parametrize("B,isz,tex_res", [(2, 128, 1), (16, 256, 6)])   # 128^2, and the C2 shape
def test_bit_exact_with_reference_kernels_in_double(rgb, B, isz, tex_res):
    """Same IEEE operation sequence and the same device exp: every pixel plane bit-identical (un-pooled: the pool is the
    package's); p2f (and vertex gradients, where the reference's backward launches) to 1e-12: its double atomics reorder sums."""
    fv, tex = scene(B, 3, tex_res, seed=3)
    fv, tex = widen(fv, 1), widen(tex, 2)
    S = 2 * isz
    g = np.random.default_rng(5).normal(size=(B, 4, isz, isz))
    tfv = torch.from_numpy(fv).to(DEV).requires_grad_(True)
    ttex = torch.from_numpy(tex).to(DEV)
    tg = torch.from_numpy(g).to(DEV)
    img, p2f, aggr = raster.soft_rasterize(tfv, ttex, isz, anti_aliasing=True, aggr_func_rgb=rgb, **UMR)
    colors_hi = img.grad_fn.saved_tensors[2]
    img.backward(tg)
    ghi = (tg / 4).repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
    colors, rp2f, raggr, rgf = _ref_f64(tfv.detach(), ttex, S, raster.FUNC_RGB[rgb], ghi)
    assert torch.equal(colors_hi, colors), "soft_colors not bit-exact: %d pixels" % int((colors_hi != colors).sum())
    assert torch.equal(aggr, raggr)
    assert torch.equal(img.detach(), TF.avg_pool2d(colors, 2, 2)), "pooled image differs from avg_pool2d of the planes"
    assert torch.allclose(p2f, rp2f, rtol=1e-12, atol=1e-14)
    # the reference's backward kernel, instantiated for double, asks for more registers than its 512-thread launch has
    # (it prints "too many resources requested for launch" and leaves the gradients zero): compared where it ran
    if float(rgf.abs().max()) > 0:
        assert torch.allclose(tfv.grad, rgf, rtol=1e-12, atol=1e-12 * float(rgf.abs().max()))


# ---------------------------------------------------------------------------------------------------------------------
# reproducibility, gradcheck, dtypes
# ---------------------------------------------------------------------------------------------------------------------
def test_bitwise_reproducible_with_and_without_the_deterministic_flag():
    fv, tex = scene(4, 3, 2, seed=11)
    fv, tex = widen(fv, 1), widen(tex, 2)
    g = np.random.default_rng(2).normal(size=(4, 4, 64, 64))
    runs = []
    for det in (False, True, False, True):
        torch.use_deterministic_algorithms(det)
        try:
            torch.randn(1 << 22, device=DEV).sum()   # other work in between
            runs.append(gpu(fv, np.ascontiguousarray(tex[:2]), 64, True, g, **UMR))
        finally:
            torch.use_deterministic_algorithms(False)
    for r in runs[1:]:
        for k, v in runs[0].items():
            assert v.tobytes() == r[k].tobytes(), k
    assert np.abs(runs[0]["p2f"]).max() > 0 and np.abs(runs[0]["grad_faces"]).max() > 0


def _small(textype, B=1):
    fv, tex = scene(B, 1, 2, seed=5)   # 80 faces
    if textype == "vertex":
        tex = np.random.default_rng(6).uniform(0, 1, size=(B, fv.shape[1], 3, 3))
    return torch.from_numpy(widen(fv, 1)).to(DEV), torch.from_numpy(widen(tex, 2)).to(DEV)


@pytest.mark.parametrize("textype,rgb", [("surface", "softmax"), ("vertex", "softmax"), ("surface", "hard"), ("vertex", "hard")])
def test_gradcheck_textures(textype, rgb):
    """The render is linear in the textures."""
    fv, tex = _small(textype)
    tex.requires_grad_(True)
    fn = lambda t: raster.soft_rasterize(fv, t, 16, anti_aliasing=True, texture_type=textype, aggr_func_rgb=rgb, **SOFT)[0]  # noqa: E731
    assert torch.autograd.gradcheck(fn, (tex,), eps=1e-3, atol=1e-9, rtol=1e-7, nondet_tol=0.0)


def test_gradcheck_depth():
    """d / dz only: the reference's analytic gradient ignores the xy-dependence of w_clip / zp / the culls on purpose."""
    fv, tex = _small("surface")
    z = fv.view(1, -1, 3, 3)[..., 2].clone().requires_grad_(True)

    def fn(zz):
        f = torch.cat((fv.view(1, -1, 3, 3)[..., :2], zz[..., None]), dim=-1)
        return raster.soft_rasterize(f, tex, 16, anti_aliasing=True, **SOFT)[0]
    assert torch.autograd.gradcheck(fn, (z,), eps=1e-6, atol=1e-7, rtol=1e-5, nondet_tol=0.0)


def test_dtype_contract():
    fv32, tex32 = scene(2, 2, 2, seed=4)
    a32 = torch.from_numpy(fv32).to(DEV)
    t32 = torch.from_numpy(tex32).to(DEV)

    def render32():
        a, t = a32.clone().requires_grad_(True), t32.clone().requires_grad_(True)
        out = raster.soft_rasterize(a, t, 32, anti_aliasing=True, **UMR)
        out[0].square().sum().backward()
        return [x.detach().cpu().numpy().tobytes() for x in out] + [a.grad.cpu().numpy().tobytes(), t.grad.cpu().numpy().tobytes()], out

    torch.use_deterministic_algorithms(True)   # the float32 atomics would otherwise differ between any two runs
    try:
        before, out32 = render32()
        a = a32.double().requires_grad_(True)
        t = t32.clone().requires_grad_(True)   # float32 textures beside float64 vertices are converted
        img, p2f, aggr = raster.soft_rasterize(a, t, 32, anti_aliasing=True, **UMR)
        assert all(s.dtype == torch.float64 for s in img.grad_fn.saved_tensors) and len(img.grad_fn.saved_tensors) == 4
        img.float().square().sum().backward()
        assert img.dtype == p2f.dtype == aggr.dtype == a.grad.dtype == torch.float64 and t.grad.dtype == torch.float32
        after, _ = render32()
    finally:
        torch.use_deterministic_algorithms(False)
    assert before == after
    assert all(x.dtype == torch.float32 for x in out32)
    h = raster.soft_rasterize(a32.half(), t32.half(), 32, anti_aliasing=True, **UMR)
    assert all(x.dtype == torch.float32 for x in h)
    assert (img.float() - out32[0]).abs().max() < 0.5   # the same picture


def test_renderers_end_to_end_in_float64():
    """nnutils.smr.SoftRenderer and sr.SoftRenderer with float64 input against the same torch vertex chain on the CPU
    followed by oracle B in double."""
    rng = np.random.default_rng(0)
    v, f = synth.icosphere(2)
    B, isz = 2, 32
    verts = synth.bird_like(v, rng, B).astype(np.float64)
    cams = synth.cameras(rng, B).astype(np.float64)
    tex = rng.uniform(0, 1, size=(B, f.shape[0], 4, 3))
    faces = np.repeat(f.astype(np.int64)[None], B, 0)
    r = smr.SoftRenderer(isz, "softmax")
    tv = torch.from_numpy(verts).to(DEV).requires_grad_(True)
    assert not r._projectable(tv)
    img, p2f, aggr = r(tv, torch.from_numpy(faces).to(DEV), torch.from_numpy(cams).to(DEV), torch.from_numpy(tex).to(DEV))
    assert img.dtype == p2f.dtype == aggr.dtype == torch.float64
    img.sum().backward()
    assert tv.grad.dtype == torch.float64 and torch.isfinite(tv.grad).all() and tv.grad.abs().sum() > 0
    # the same chain on CPU tensors, then the oracle
    pv = geom_utils.orthographic_proj_withz(torch.from_numpy(verts), torch.from_numpy(cams), offset_z=5.)
    pv[:, :, 1] *= -1
    mesh = sr.Mesh(pv, torch.from_numpy(faces).int(), torch.from_numpy(tex))
    mesh = r.renderer.transform(r.renderer.lighting(mesh))
    assert mesh.face_vertices.dtype == mesh.face_textures.dtype == torch.float64
    ref = oracle(mesh.face_vertices.numpy().reshape(B, -1, 9), mesh.face_textures.numpy(), isz, True, None, **UMR)
    # the GPU and CPU torch chains round differently (matmul, normalize), and at the renderer's eps / gamma the device's
    # float expf seeds the softmax one float ulp (9e-8) away from glibc's (see _eps_for_oracle)
    assert np.abs(img.detach().cpu().numpy() - ref["images"]).max() < 1e-6
    p2f_v, aggr_v = r.visibility(tv.detach(), torch.from_numpy(faces).to(DEV), torch.from_numpy(cams).to(DEV))
    assert torch.equal(aggr_v, aggr) and r.visible_faces(tv.detach(), torch.from_numpy(faces).to(DEV), torch.from_numpy(cams).to(DEV)) is None
    r2 = sr.SoftRenderer(image_size=isz, camera_mode="look_at", eye=[0.3, 0.2, -2.5], anti_aliasing=True, **UMR)
    out = r2(torch.from_numpy(verts).to(DEV), torch.from_numpy(faces).int().to(DEV), torch.from_numpy(tex).to(DEV))
    out_white = r2(torch.from_numpy(verts).to(DEV), torch.from_numpy(faces).int().to(DEV))
    assert out[0].dtype == out_white[0].dtype == torch.float64 and out[0][:, 3].max() > 0.5


# ---------------------------------------------------------------------------------------------------------------------
# the ends of the input range
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F", [65535, 65536, 131071])
def test_face_counts_with_the_last_face_on_screen(F):
    """Most faces lie far off screen; faces 0, 1023, 1024, F - 2 and F - 1 overlap in the middle of the image."""
    rng = np.random.default_rng(F)
    fv = np.tile(np.array([40.0, 40.0, 5.0, 40.5, 40.0, 5.0, 40.0, 40.5, 5.0]), (1, F, 1))
    fv += rng.uniform(0, 0.1, size=fv.shape)
    for j, i in enumerate((0, 1023, 1024, F - 2, F - 1)):
        fv[0, i] = [-0.6 + 0.1 * j, -0.5, 3.0 + j, 0.7, -0.4 + 0.05 * j, 4.0 + j, -0.1 * j, 0.8, 5.0 - j * 0.3]
    tex = rng.uniform(0, 1, size=(1, F, 1, 3))
    g = rng.normal(size=(1, 4, 24, 24))
    for rgb in ("softmax", "hard"):
        kw = dict(SOFT, aggr_func_rgb=rgb)
        ref = oracle(fv, tex, 24, True, g, **kw)
        got = gpu(fv, tex, 24, True, g, **kw)
        check(got, ref, rgb, "F=%d %s" % (F, rgb))
        if rgb == "hard":
            assert (got["aggrs"][:, 1] == F - 1).any()
        else:
            assert np.abs(got["grad_faces"][0, F - 1]).max() > 0 and np.abs(got["p2f"][0, F - 1]).max() > 0


def test_face_covering_the_whole_raster():
    fv = np.array([[[-5.0, -4.0, 3.0, 6.0, -5.0, 4.0, 0.5, 7.0, 5.0], [-0.5, -0.4, 2.0, 0.6, -0.5, 2.5, 0.1, 0.7, 2.2]]])
    tex = np.random.default_rng(1).uniform(0, 1, size=(1, 2, 9, 3))
    g = np.random.default_rng(2).normal(size=(1, 4, 40, 40))
    for rgb in ("softmax", "hard"):
        kw = dict(umr_oracle_kw(), aggr_func_rgb=rgb)
        check(gpu(fv, tex, 40, True, g, **kw), oracle(fv, tex, 40, True, g, **kw), rgb, rgb)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_non_finite_vertices_render_as_the_oracle_does(bad):
    fv, tex = scene(1, 1, 2, seed=7)
    fv, tex = widen(fv, 1), widen(tex, 2)
    fv[0, 3, 4] = bad        # one coordinate of one face
    fv[0, 10, 6:9] = bad     # a whole corner of another
    g = np.random.default_rng(2).normal(size=(1, 4, 24, 24))
    for rgb in ("softmax", "hard"):
        kw = dict(SOFT, aggr_func_rgb=rgb)
        ref, got = oracle(fv, tex, 24, False, g, **kw), gpu(fv, tex, 24, False, g, **kw)
        for k in ("images", "aggrs", "p2f", "grad_faces", "grad_tex"):
            assert np.array_equal(np.isnan(got[k]), np.isnan(ref[k])), (k, rgb)
            fin = np.isfinite(ref[k])
            assert np.allclose(got[k][fin], ref[k][fin], rtol=1e-9, atol=1e-9 * (np.abs(ref[k][fin]).max() if fin.any() else 1)), (k, rgb)


@pytest.mark.parametrize("tex_res", [1, 6, 17])
def test_texture_resolutions(tex_res):
    rng = np.random.default_rng(129)
    v, f = synth.icosphere(1)
    fv = widen(synth.raster_space_faces(synth.bird_like(v, rng, 2), f, synth.cameras(rng, 2)), 1)
    tex = rng.uniform(0, 1, size=(2, f.shape[0], tex_res * tex_res, 3))
    g = rng.normal(size=(2, 4, 40, 40))
    for rgb in ("softmax", "hard"):
        kw = dict(umr_oracle_kw(), aggr_func_rgb=rgb)
        ref = oracle(fv, tex, 40, True, g, **kw)
        assert tex_res == 1 or np.abs(ref["grad_tex"][:, :, tex_res * tex_res // 2:]).max() > 0
        check(gpu(fv, tex, 40, True, g, **kw), ref, rgb, "texture_res=%d %s" % (tex_res, rgb))


# ---------------------------------------------------------------------------------------------------------------------
# what it is for
# ---------------------------------------------------------------------------------------------------------------------
def test_spread_between_the_float32_and_float64_renders(capsys):
    """At the C2 shape (B = 16, 1280 faces, 256^2 anti-aliased, T2 = 36, UMR's sigma / gamma) the float32 render is
    chaotic on the silhouette fringe; the float64 render of the same float32 inputs shows by how much.  Loose sanity
    bounds only: the numbers are the report (DESIGN.md §9)."""
    fv, tex = scene(16, 3, 6, seed=0)
    g = torch.from_numpy(np.random.default_rng(1).normal(size=(16, 4, 256, 256)).astype(np.float32)).to(DEV)
    res = {}
    for dt in (torch.float32, torch.float64):
        a = torch.from_numpy(fv).to(DEV).to(dt).requires_grad_(True)
        t = torch.from_numpy(tex).to(DEV).to(dt)
        img, _, _ = raster.soft_rasterize(a, t, 256, anti_aliasing=True, **UMR)
        hi = img.grad_fn.saved_tensors[2]
        img.backward(g.to(dt))
        res[dt] = (hi.double(), a.grad.double())
    d = (res[torch.float32][0] - res[torch.float64][0]).abs()
    frac_alpha = float((d[:, 3] > 1e-4).double().mean())
    frac_rgb = float((d[:, :3].amax(1) > 1e-4).double().mean())
    rel = float((res[torch.float32][1] - res[torch.float64][1]).norm() / res[torch.float64][1].norm())
    with capsys.disabled():
        print("\nfp32 vs fp64 at C2 (raster pixels): alpha beyond 1e-4 on %.3f%%, max %.3g; RGB beyond 1e-4 on %.3f%%; "
              "grad_faces rel-L2 %.3g" % (100 * frac_alpha, float(d[:, 3].max()), 100 * frac_rgb, rel))
    assert frac_alpha < 0.2 and frac_rgb < 0.2 and rel < 1.0
    assert float(d.median()) < 1e-6   # away from the fringe the two agree
