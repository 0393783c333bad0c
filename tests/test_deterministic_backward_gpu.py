"""Deterministic backwards of the fused vertex pipeline, the NMR texture gradient and the sampler's image gradient
(torch.use_deterministic_algorithms(True), include/umr_b200.h).  Each entry point's outputs are bitwise equal across runs,
host threads on side streams and CUDA-graph replay, and stay within the gates the default kernels are held to: the
float64 error bounds of test_vertex_range_gpu, oracle/nmr.py's float64 adjoint, and float64 grid_sample.  End to end,
SoftRenderer keeps the fused vertex kernel under the flag, and the train_s2-shaped step with the NMR texture loss is
bitwise reproducible.  With the flag off the three ops launch what they launched before."""
import os

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # generic SoftRenderer configurations (README)

import ctypes  # noqa: E402
import threading  # noqa: E402

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

import nmr as nmr_oracle  # noqa: E402  oracle/nmr.py
import test_deterministic_losses_gpu as DL  # noqa: E402
import test_nmr_gpu as TN  # noqa: E402
import test_vertex_range_gpu as VR  # noqa: E402
from umr_b200 import _lib, ops, synth  # noqa: E402
from umr_b200.neural_renderer import Renderer  # noqa: E402
from umr_b200.nnutils import loss_utils, smr  # noqa: E402
from umr_b200.raster import _ptr, _stream_ptr  # noqa: E402
from umr_b200.vertex import project_faces  # noqa: E402
from util import rel_report  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture
def det():
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(old)


def _host(ts):
    torch.cuda.synchronize()
    return [t.detach().cpu() for t in ts]


def _same(a, b, what):
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y) or (torch.isnan(x) == torch.isnan(y)).all() and torch.equal(x.nan_to_num(), y.nan_to_num()), \
            "%s: output %d differs bitwise" % (what, k)


def assert_reproducible(fn):
    """fn() -> list of tensors, computed on the current stream from static inputs.  Bitwise equal across 3 runs, 4 host
    threads on side streams and 2 replays of one CUDA-graph capture."""
    ref = _host(fn())
    for _ in range(2):
        _same(ref, _host(fn()), "run")
    results = [None] * 4

    def work(i):
        torch.use_deterministic_algorithms(True)
        st = torch.cuda.Stream(device=DEV)
        with torch.cuda.stream(st):
            out = fn()
        st.synchronize()
        results[i] = [t.detach().cpu() for t in out]

    ts = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for r in results:
        _same(ref, r, "thread")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):   # warm-up outside the capture
            fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fn()
    for _ in range(2):
        graph.replay()
        _same(ref, _host(out), "graph replay")
    return ref


# -------------------------------------------------------------------------------------------------
# vertex pipeline
# -------------------------------------------------------------------------------------------------
# (V, F, Bv, H, face layout, light)
VCASES = [
    (3, 1, 1, 1, "2d", "off"),
    (257, 257, 2, 1, "per_mesh", "default"),
    (257, 257, 2, 8, "1", "colour"),
    (642, 1280, 4, 8, "per_mesh", "colour"),
    (642, 1280, 16, 1, "2d", "default"),
    (2562, 1280, 2, 8, "2d", "off"),
    (300, 600, 3, 8, "per_mesh", "off"),
]


def _vertex_fn(verts, cams, faces, lc, g_fv, g_lt, vs=1.0):
    v = verts.to(DEV).requires_grad_(True)
    c = cams.to(DEV).requires_grad_(True)
    f = faces.to(DEV)
    gf = g_fv.to(DEV)
    gl = g_lt.to(DEV) if g_lt is not None else None

    def fn():
        fv, lt = project_faces(v, c, f, offset_z=5.0, eye_z=VR.EYE_Z, viewing_scale=vs, flip_y=True, light=lc)
        outs, grads = ([fv, lt], [gf, gl]) if lt is not None else ([fv], [gf])
        gv, gc = torch.autograd.grad(outs, (v, c), grads)
        return [fv] + ([lt] if lt is not None else []) + [gv, gc]
    return fn


@pytest.mark.parametrize("V,F,Bv,H,layout,light", VCASES)
def test_vertex_backward_matches_float64(det, V, F, Bv, H, layout, light):
    seed = V * 5 + F + Bv * 3 + H
    verts, cams, faces = VR._case(V, F, Bv, H, layout, seed)
    lc = VR._f32(VR.LIGHTS[light])
    kink = VR._kink_faces(verts, cams, faces, True, lc) if lc is not None else None
    g_fv, g_lt = VR._upstream(Bv * H, F, lc, kink, seed)
    fn = _vertex_fn(verts, cams, faces, lc, g_fv, g_lt)
    out = assert_reproducible(fn)
    fv, lt = out[0], (out[1] if lc is not None else None)
    gv, gc = out[-2], out[-1]
    tag = "det V%d F%d Bv%d H%d %s %s" % (V, F, Bv, H, layout, light)
    VR._compare_projection(tag, verts, cams, faces, 1.0, True, lc, g_fv, g_lt, fv, lt, gv, gc)


def test_vertex_backward_327680_faces(det):
    """F = 327680 over 40962 vertices (random corners, light off), 8 hypotheses of one mesh."""
    V, F, H = 40962, 327680, 8
    g = torch.Generator().manual_seed(77)
    verts = (1.4 * torch.rand(1, V, 3, generator=g, dtype=torch.float64) - 0.7).float()
    cams = VR._random_cams(g, H)
    faces = torch.randint(0, V, (F, 3), generator=g, dtype=torch.int32)
    g_fv = torch.randn(H, F, 3, 3, generator=g)
    fn = _vertex_fn(verts, cams, faces, None, g_fv, None)
    out = _host(fn())
    _same(out, _host(fn()), "run")
    VR._compare_projection("det F327680 H8", verts, cams, faces, 1.0, True, None, g_fv, None, out[0], None, out[1], out[2])


@pytest.mark.parametrize("layout", ["2d", "per_mesh"])
def test_vertex_backward_out_of_range_face_index(det, layout):
    """A face with an index outside [0, V) contributes nothing (zeros in the workspace): the gradients are those of the
    valid mesh with that face's upstream gradient zeroed, within the float64 bounds; the forward makes that corner NaN."""
    V, F, Bv, H = 257, 300, 2, 8
    verts, cams, faces = VR._case(V, F, Bv, H, layout, 5)
    lc = VR._f32(VR.LIGHTS["default"])
    kink = VR._kink_faces(verts, cams, faces, True, lc)
    g_fv, g_lt = VR._upstream(Bv * H, F, lc, kink, 5)
    bad = faces.clone()
    if layout == "2d":
        bad[11, 1], bad[40, 2] = V, -1
        hit = [(slice(None), 11, 1), (slice(None), 40, 2)]
    else:
        bad[1, 11, 1], bad[0, 40, 0] = V + 3, -7   # mesh 1's bad index must not reach mesh 2's rows
        hit = [(slice(H, 2 * H), 11, 1), (slice(0, H), 40, 0)]
    for r, k, _ in hit:
        g_fv[r, k] = 0.0
        g_lt[r, k] = 0.0
    out = _host(_vertex_fn(verts, cams, bad, lc, g_fv, g_lt)())
    for r, k, corner in hit:
        assert torch.isnan(out[0][r, k, corner]).all()
    good = _host(_vertex_fn(verts, cams, faces, lc, g_fv, g_lt)())
    VR._compare_projection("det bad index " + layout, verts, cams, faces, 1.0, True, lc, g_fv, g_lt, good[0], good[1],
                           out[2], out[3])


# -------------------------------------------------------------------------------------------------
# NMR texture gradient
# -------------------------------------------------------------------------------------------------
def _with_sliver(verts, faces):
    """Appends one front-most sliver (smallest angle far below the box test's 1e-2 sine): its box is the whole raster."""
    B, V = verts.shape[:2]
    sv = np.array([[-0.8, -0.1, 2.0], [0.8, 0.1, 2.0], [0.8, 0.11, 2.0]], np.float32)
    verts = np.concatenate([verts, np.repeat(sv[None], B, 0)], 1)
    faces = np.concatenate([faces, np.repeat(np.array([[[V, V + 1, V + 2]]], np.int32), B, 0)], 1)
    return verts, faces


def _nmr_det_backward(verts, faces, fidx, tex_shape, g, p):
    lib = _lib.load()
    v, f = torch.from_numpy(verts).to(DEV), torch.from_numpy(faces).to(DEV)
    fi, gg = torch.from_numpy(fidx).to(DEV), torch.from_numpy(g.astype(np.float32)).to(DEV)
    ws = torch.empty(lib.umr_nmr_workspace_bytes(p.batch_size, p.num_faces, p.fill_back), device=DEV, dtype=torch.uint8)

    def fn():
        gt = torch.full(tex_shape, float("nan"), device=DEV)   # the call zero-fills it
        _lib.check(lib.umr_nmr_backward_textures_deterministic(_ptr(v), _ptr(f), _ptr(fi), _ptr(gg), _ptr(gt), ctypes.byref(p),
                                                               _ptr(ws), _stream_ptr(DEV)),
                   "umr_nmr_backward_textures_deterministic")
        return [gt]
    return fn


@pytest.mark.parametrize("fill_back,G,aa,sliver", [(True, 1, True, False), (False, 1, True, False), (True, 8, False, False),
                                                   (False, 8, True, False), (True, 1, True, True), (True, 8, False, True)])
def test_nmr_texture_gradient_matches_the_oracle_adjoint(det, fill_back, G, aa, sliver):
    B = 8 if G == 8 else 2
    verts, faces = TN.nmr_inputs(B, 2, seed=1, soup=8)
    if sliver:
        verts, faces = _with_sliver(verts, faces)
    F = faces.shape[1]
    rng = np.random.default_rng(5)
    tex = rng.uniform(0, 1, size=(B // G, F, 3, 3, 3, 3)).astype(np.float32)
    light = dict(Ia=0.6, Id=0.5, ca=(1, 0.9, 0.8), cd=(0.5, 1, 1), direction=(0.2, 1, -1))
    got, default_backward = TN.abi_forward(verts, faces, tex, 64, aa=aa, fill_back=fill_back, **light)
    g = rng.uniform(0.5, 1.5, size=got["rgb"].shape)   # one sign: no cancellation in the float32 accumulation
    p = TN.params(B, verts.shape[1], F, 3, 64, aa=aa, fill_back=fill_back, G=G, **light)
    gk = assert_reproducible(_nmr_det_backward(verts, faces, got["face_index"], tex.shape, g, p))[0].numpy()
    zb = (got["face_index"], got["raster_depth"])
    gr = nmr_oracle.grad_textures(g, verts, faces, tex.shape, zb, anti_aliasing=aa, fill_back=fill_back, eye_z=TN.EYE,
                                  shared_textures=G, Ia=light["Ia"], Id=light["Id"], ca=light["ca"], cd=light["cd"],
                                  direction=light["direction"])
    assert np.abs(gr).max() > 0
    err = np.abs(gk - gr)
    assert (err <= 1e-5 * np.maximum(np.abs(gk), np.abs(gr)) + 1e-7).all(), err.max()
    gd = default_backward(g)
    assert np.abs(gk - gd).max() <= 1e-5 * np.abs(gd).max()
    if sliver:
        won = (zb[0] == F - 1) | (zb[0] == 2 * F - 1)
        assert won.any() and np.abs(gr[:, F - 1]).max() > 0   # the sliver wins pixels and gets a gradient
    if fill_back:
        back = np.unique(zb[0][zb[0] >= F]) - F
        assert back.size and np.abs(gr[:, back]).max() > 0


def test_nmr_renderer_reproducible_under_the_flag(det):
    """neural_renderer.Renderer's texture gradient through _NmrFunction, G = 8 camera hypotheses sharing a texture."""
    B, G = 8, 8
    verts, faces = TN.nmr_inputs(B, 3, seed=4)
    r = Renderer(image_size=64, camera_mode="look_at", perspective=False, light_intensity_ambient=0.8,
                 light_intensity_directional=0.4, light_direction=[0, 1, -1])
    r.eye = [0, 0, TN.EYE]
    v, f = torch.from_numpy(verts).to(DEV), torch.from_numpy(faces).to(DEV)
    tex = torch.rand(B // G, faces.shape[1], 4, 4, 4, 3, generator=torch.Generator().manual_seed(3)).to(DEV).requires_grad_(True)
    w = torch.rand(B, 3, 64, 64, generator=torch.Generator().manual_seed(4)).to(DEV)

    def fn():
        img = r.render_rgb(v, f, tex)
        return [img, torch.autograd.grad(img, tex, w)[0]]
    out = assert_reproducible(fn)
    assert out[1].abs().max() > 0


# -------------------------------------------------------------------------------------------------
# sampler image gradient
# -------------------------------------------------------------------------------------------------
def _sample_case(C, kind, B=2, H=37, W=45, N=500, seed=0):
    g = torch.Generator().manual_seed(seed + C)
    img = torch.rand(B, C, H, W, generator=g)
    flow = torch.rand(B, N, 2, generator=g) * 2.4 - 1.2   # out-of-range samples included (zero padding)
    if kind == "one_pixel":
        flow[:] = torch.tensor([0.1234, -0.4321])             # every sample in one cell
    elif kind == "nan":
        flow[0, 7, 0] = float("nan")
        flow[1, 100, 1] = float("nan")
        flow[1, 200] = float("nan")
    w = torch.rand(B, N, C, generator=g)
    return img, flow, w


def _sample_fn(img, flow, w):
    i = img.to(DEV).requires_grad_(True)
    fl = flow.to(DEV).requires_grad_(True)
    wd = w.to(DEV)

    def fn():
        out = ops.bilinear_sample(i, fl)
        gi, gf = torch.autograd.grad(out, (i, fl), wd)
        return [out, gi, gf]
    return fn


@pytest.mark.parametrize("C", [1, 2, 3, 4])
@pytest.mark.parametrize("kind", ["random", "one_pixel"])
def test_sampler_image_gradient_matches_float64(det, C, kind):
    img, flow, w = _sample_case(C, kind)
    out, gi, gf = assert_reproducible(_sample_fn(img, flow, w))
    i64 = img.double().requires_grad_(True)
    f64 = flow.double().requires_grad_(True)
    ref = torch.nn.functional.grid_sample(i64, f64[:, :, None], mode="bilinear", padding_mode="zeros",
                                          align_corners=True)[..., 0].permute(0, 2, 1)
    gir, gfr = torch.autograd.grad(ref, (i64, f64), w.double())
    for name, got, r, rtol, atol in (("sample fwd", out, ref, 1e-4, 1e-6),
                                     ("sample dimage", gi, gir, 1e-4, 1e-5),
                                     ("sample dflow", gf, gfr, 1e-4, 1e-4 * float(gfr.abs().max()) * 1e-2 + 1e-6)):
        ok, msg = rel_report(name, got.numpy(), r.detach().numpy(), rtol, atol)
        assert ok, msg
    if kind == "one_pixel":
        assert (gi != 0).sum() == 4 * 2 * C   # the cell's four pixels, in each image and channel
    torch.use_deterministic_algorithms(False)
    d_out, d_gi, d_gf = _host(_sample_fn(img, flow, w)())
    torch.use_deterministic_algorithms(True)
    assert torch.equal(out, d_out) and torch.equal(gf, d_gf)   # grad_flow is the default kernel's


def test_sampler_nan_flow_reaches_the_default_pixels(det):
    img, flow, w = _sample_case(3, "nan")
    out, gi, gf = assert_reproducible(_sample_fn(img, flow, w))
    torch.use_deterministic_algorithms(False)
    d_out, d_gi, d_gf = _host(_sample_fn(img, flow, w)())
    torch.use_deterministic_algorithms(True)
    assert torch.isnan(gi).any()
    assert torch.equal(torch.isnan(gi), torch.isnan(d_gi))
    fin = ~torch.isnan(d_gi)
    assert (gi[fin] - d_gi[fin]).abs().max() <= 1e-5


# -------------------------------------------------------------------------------------------------
# end to end
# -------------------------------------------------------------------------------------------------
def _renderer_case(B=2, H=8, IS=32, T=10):
    rng = np.random.default_rng(12)
    v, f = synth.icosphere(3)
    vs0 = torch.from_numpy(synth.bird_like(v, rng, B))
    fs = torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1).to(DEV)
    cams0 = torch.from_numpy(np.stack([synth.cameras(rng, H) for _ in range(B)])).view(-1, 7)
    tx0 = torch.from_numpy(rng.uniform(0, 1, size=(B, f.shape[0], T * T, 3)).astype(np.float32))
    w = torch.linspace(0.5, 1.5, B * H * 4 * IS * IS, device=DEV).view(B * H, 4, IS, IS)
    return vs0, fs, cams0, tx0, w, IS


def test_soft_renderer_keeps_the_fused_path_under_the_flag(det):
    """SoftRenderer with 8 hypotheses (ambient light only): under the flag it launches the fused projection (forward 1,
    deterministic backward 5) and never materialises [B*H, ...] copies of the textures; its images equal the flag-off
    images bit for bit, and its gradients are reproducible."""
    vs0, fs, cams0, tx0, w, IS = _renderer_case()
    lib = _lib.load()
    copy_bytes = cams0.shape[0] * tx0[0].numel() * 4   # one [B*H, F, T2, 3] texture copy

    def step():
        r = smr.SoftRenderer(IS, "softmax")
        r.ambient_light_only()
        vs = vs0.clone().to(DEV).requires_grad_(True)
        tx = tx0.clone().to(DEV).requires_grad_(True)
        c = cams0.clone().to(DEV).requires_grad_(True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        n0 = lib.umr_launch_count()
        img, _, _ = r(vs, fs, c, tx)
        (img * w).sum().backward()
        torch.cuda.synchronize()
        return (lib.umr_launch_count() - n0, torch.cuda.max_memory_allocated() - base,
                [img.detach().cpu(), vs.grad.cpu(), c.grad.cpu(), tx.grad.cpu()])

    n_fused, peak_fused, out = step()
    for _ in range(2):
        _same(out, step()[2], "SoftRenderer run")
    try:
        smr.SoftRenderer.fuse_vertex_pipeline = False
        n_generic, peak_generic, _ = step()
        torch.use_deterministic_algorithms(False)
        smr.SoftRenderer.fuse_vertex_pipeline = True
        _, _, default = step()
    finally:
        smr.SoftRenderer.fuse_vertex_pipeline = True
        torch.use_deterministic_algorithms(True)
    assert n_fused - n_generic == 6, (n_fused, n_generic)   # umr_project_faces_forward 1 + _backward_deterministic 5
    assert peak_fused < copy_bytes < peak_generic, (peak_fused, copy_bytes, peak_generic)
    assert torch.equal(out[0], default[0])
    for k in (1, 2, 3):
        ok, msg = rel_report("grad", out[k].numpy(), default[k].numpy(), 2e-4, 2e-5 * float(default[k].abs().max()))
        assert ok, msg


# (B, H, IS, icosphere subdivision, T, seed): the NMR texture loss reads 6x6 textures (loss_utils.py:310)
NMR_STEPS = {"scene_shape_t6": (2, 8, 32, 2, 6, 21), "bench_default": DL.STEPS["bench_default"]}


@pytest.mark.parametrize("name", list(NMR_STEPS))
def test_whole_step_with_nmr_texture_loss(det, monkeypatch, name):
    """The train_s2-shaped step with MultiTextureLoss(renderer="nmr", texture_loss_type="l1"): bitwise reproducible, and
    within the step gate of the flag-off step."""
    cls = loss_utils.MultiTextureLoss
    monkeypatch.setattr(loss_utils, "MultiTextureLoss", lambda *a: cls(*a[:5], "nmr"))
    step, leaves = DL.make_step(*NMR_STEPS[name])
    ref = DL._run(step, leaves)
    for _ in range(2):
        DL._assert_equal(ref, DL._run(step, leaves), "step run")
    torch.use_deterministic_algorithms(False)
    default = DL._run(step, leaves)
    torch.use_deterministic_algorithms(True)
    assert all(bool(torch.isfinite(t).all()) for t in ref)
    for k, (x, r) in enumerate(zip(ref, default)):
        ok, msg = rel_report("step output %d" % k, x.numpy(), r.numpy(), 2e-4, 2e-5 * float(r.abs().max()) + 1e-9)
        print(msg)
        assert ok, msg


# -------------------------------------------------------------------------------------------------
# launch counts
# -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["default", "deterministic"])
def test_launch_counts(mode):
    dflt = mode == "default"
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(not dflt)
    try:
        # (forward, backward) launches; the flag-off counts are the ones before the deterministic backwards existed
        want = {"vertex": (1, 2) if dflt else (1, 5), "nmr": (3, 2), "sampler": (1, 1) if dflt else (1, 3)}
        verts, cams, faces = VR._case(257, 300, 2, 8, "per_mesh", 1)
        v = verts.to(DEV).requires_grad_(True)
        c = cams.to(DEV).requires_grad_(True)
        nv, nf = TN.nmr_inputs(8, 2, seed=1)
        r = Renderer(image_size=32, camera_mode="look_at", perspective=False)
        r.eye = [0, 0, TN.EYE]
        tex = torch.rand(1, nf.shape[1], 2, 2, 2, 3, device=DEV).requires_grad_(True)
        img = torch.rand(2, 3, 16, 16, device=DEV).requires_grad_(True)
        flow = (torch.rand(2, 100, 2, device=DEV) * 2 - 1).requires_grad_(True)
        ops_ = {
            "vertex": lambda: project_faces(v, c, faces.to(DEV))[0].sum(),
            "nmr": lambda: r.render_rgb(torch.from_numpy(nv).to(DEV), torch.from_numpy(nf).to(DEV), tex).sum(),
            "sampler": lambda: ops.bilinear_sample(img, flow).sum(),
        }
        for name, op in ops_.items():
            nfw, loss = DL._launches(op)
            nb, _ = DL._launches(loss.backward)
            assert (nfw, nb) == want[name], (name, mode, nfw, nb)
    finally:
        torch.use_deterministic_algorithms(old)
