"""Deterministic mode of the soft rasteriser (torch.use_deterministic_algorithms(True), include/umr_b200.h): images, p2f,
aggrs, vertex and texture gradients are bitwise equal across runs, tilings, pair-buffer settings, host threads, side
streams and CUDA-graph replay, and agree with oracle B and with the default path under the parity gates of
test_raster_modes_gpu (1e-4 relative, magnitude-scaled gradient atol, hard depth / face-id planes bit-exact)."""
import os

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # the generic SoftRenderer chain's matmul (README)

import threading  # noqa: E402

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

import softras  # noqa: E402
from umr_b200 import _lib, raster, synth  # noqa: E402
from umr_b200.nnutils import loss_utils, smr  # noqa: E402
from util import rel_report, scene  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
UMR = dict(sigma_val=1e-5, dist_eps=1e-10, gamma_val=1e-4)
KEYS = ("images", "p2f", "aggrs", "grad_faces", "grad_tex")


@pytest.fixture
def det():
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(old)


def run(fv, tex, isz, aa, g, rgb="softmax", tile=0, cand=8.0, geom_grad=True, tex_grad=True, stream=None, **modes):
    old = raster.PAIR_CAND_PER_PIXEL, raster.FORWARD_TILE
    raster.PAIR_CAND_PER_PIXEL, raster.FORWARD_TILE = cand, tile
    try:
        with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream()):
            tfv = torch.from_numpy(fv).to(DEV).requires_grad_(geom_grad)
            ttex = torch.from_numpy(tex).to(DEV).requires_grad_(tex_grad)
            img, p2f, aggr = raster.soft_rasterize(tfv, ttex, isz, anti_aliasing=aa, aggr_func_rgb=rgb, **dict(UMR, **modes))
            img.backward(torch.from_numpy(g).to(DEV))
            out = dict(images=img.detach(), p2f=p2f, aggrs=aggr, grad_faces=tfv.grad if geom_grad else None,
                       grad_tex=ttex.grad if tex_grad else None)
        torch.cuda.synchronize()
    finally:
        raster.PAIR_CAND_PER_PIXEL, raster.FORWARD_TILE = old
    return {k: (v.cpu() if v is not None else None) for k, v in out.items()}


def assert_equal(a, b, what=""):
    for k in KEYS:
        if a[k] is None:
            assert b[k] is None
            continue
        assert torch.equal(a[k], b[k]), "%s %s differs bitwise" % (what, k)


def check_close(got, ref, rgb, p2f_atol=1e-6):
    ok, msgs = True, []
    for k in KEYS:
        if got[k] is None or ref.get(k) is None:
            continue
        b = np.asarray(ref[k])
        at = 1e-6 * float(np.abs(b).max() + 1e-30) + 1e-7 if k.startswith("grad") else (p2f_atol if k == "p2f" else 1e-6)
        o, m = rel_report(k, np.asarray(got[k]), b, 1e-4, at)
        ok &= o
        msgs.append(m)
    if rgb == "hard":
        ok &= np.array_equal(np.asarray(got["aggrs"]), np.asarray(ref["aggrs"]))
    assert ok, "\n".join(msgs)


def grad_of(shape, seed):
    return np.random.default_rng(seed).uniform(-1, 1, size=shape).astype(np.float32)


def c2_scene():
    fv, tex = scene(16, 3, 6, seed=7)   # B = 16, F = 1280, T2 = 36
    return fv, tex, 256, True


def odd_scene():
    fv, tex = scene(2, 2, 2, seed=8)
    return fv, tex, 45, False


def big_face_scene():
    """A near-plane triangle covering the whole raster on top of an icosphere."""
    fv, tex = scene(2, 2, 2, seed=9)
    big = np.array([-3, -3, 1.5, 3, -3, 1.5, 0, 3, 1.5], np.float32)
    fv = np.concatenate([fv, np.broadcast_to(big, (2, 1, 9))], axis=1).copy()
    tex = np.concatenate([tex, np.full((2, 1, tex.shape[2], 3), 0.5, np.float32)], axis=1)
    return fv, tex, 48, True


def many_faces_scene():
    """F = 65537: off-screen padding first, so the mesh's faces (and face F-1) are the highest indices."""
    fv, tex = scene(1, 3, 1, seed=10)
    pad = 65537 - fv.shape[1]
    off = np.tile(np.array([5, 5, 2, 5.01, 5, 2, 5, 5.01, 2], np.float32), (1, pad, 1))
    fv = np.concatenate([off, fv], axis=1)
    tex = np.concatenate([np.zeros((1, pad, 1, 3), np.float32), tex], axis=1)
    return fv, tex, 64, True


SCENES = {"c2": c2_scene, "odd": odd_scene, "big_face": big_face_scene, "many_faces": many_faces_scene}


def _img_shape(fv, tex, isz):
    return (fv.shape[0], tex.shape[-1] + 1, isz, isz)


@pytest.mark.parametrize("rgb", ["softmax", "hard"])
@pytest.mark.parametrize("name", list(SCENES))
def test_bitwise_reproducible_across_runs_tilings_and_pair_buffers(det, name, rgb):
    fv, tex, isz, aa = SCENES[name]()
    g = grad_of(_img_shape(fv, tex, isz), 1)
    ref = run(fv, tex, isz, aa, g, rgb)
    for tile, cand in ((0, 8.0), (16, 0.0), (32, 32.0)):
        assert_equal(ref, run(fv, tex, isz, aa, g, rgb, tile=tile, cand=cand), "%s tile=%d cand=%g:" % (name, tile, cand))
    if name == "many_faces":
        assert float(ref["images"].abs().max()) > 0
        if rgb == "softmax":   # hard renders never accumulate p2f
            assert float(ref["p2f"][:, -1280:].abs().max()) > 0 and float(ref["grad_faces"][:, -1280:].abs().max()) > 0


@pytest.mark.parametrize("rgb", ["softmax", "hard"])
@pytest.mark.parametrize("name", ["odd", "big_face", "c2"])
def test_matches_oracle_and_default_path(det, name, rgb):
    fv, tex, isz, aa = SCENES[name]()
    if name == "c2":
        fv, tex = fv[:2], tex[:2]
    g = grad_of(_img_shape(fv, tex, isz), 2)
    got = {k: (v.numpy() if v is not None else None) for k, v in run(fv, tex, isz, aa, g, rgb).items()}
    img, fwd, cfg = softras.render(fv, tex, isz, anti_aliasing=aa, impl="B", aggr_func_rgb=rgb, **UMR)
    gf, gt = softras.render_backward(fwd, cfg, g, anti_aliasing=aa, impl="B")
    # The whole-raster face's p2f y is a sum of 9216 pixel terms that cancel to exactly 0 by symmetry; the fixed-point sum
    # gives that 0, while float sums (the oracle's threads, the default kernels' REDs) leave a few 1e-6 of rounding.
    p2f_atol = 1e-5 if name == "big_face" else 1e-6
    check_close(got, dict(images=img, aggrs=fwd["aggrs_info"], p2f=fwd["p2f_info"], grad_faces=gf, grad_tex=gt), rgb, p2f_atol)
    torch.use_deterministic_algorithms(False)
    default = {k: (v.numpy() if v is not None else None) for k, v in run(fv, tex, isz, aa, g, rgb).items()}
    torch.use_deterministic_algorithms(True)
    check_close(got, default, rgb, p2f_atol)
    assert np.array_equal(got["images"], default["images"]) and np.array_equal(got["aggrs"], default["aggrs"])


def test_part_map_shared_textures_and_texture_only(det):
    fv, tex, isz, aa = odd_scene()
    B = fv.shape[0]
    # 4-channel part map: constant textures, vertex gradients only
    tex4 = np.concatenate([tex, tex[..., :1]], axis=-1)
    g4 = grad_of((B, 5, isz, isz), 3)
    a = run(fv, tex4, isz, aa, g4, tex_grad=False)
    assert_equal(a, run(fv, tex4, isz, aa, g4, tex_grad=False, tile=32, cand=0.0), "part map:")
    torch.use_deterministic_algorithms(False)
    check_close({k: (v.numpy() if v is not None else None) for k, v in a.items()},
                {k: (v.numpy() if v is not None else None) for k, v in run(fv, tex4, isz, aa, g4, tex_grad=False).items()},
                "softmax")
    torch.use_deterministic_algorithms(True)
    # shared textures: G = 2 (two images per texture) and G = B (one texture for the batch)
    fv4, tex4b = scene(4, 2, 2, seed=11)
    g = grad_of((4, 4, isz, isz), 4)
    for shared in (tex4b[:2].copy(), tex4b[:1].copy()):
        r1 = run(fv4, shared, isz, aa, g)
        assert_equal(r1, run(fv4, shared, isz, aa, g, tile=32, cand=0.0), "shared %d:" % shared.shape[0])
        torch.use_deterministic_algorithms(False)
        d = run(fv4, shared, isz, aa, g)
        torch.use_deterministic_algorithms(True)
        check_close({k: (v.numpy() if v is not None else None) for k, v in r1.items()},
                    {k: (v.numpy() if v is not None else None) for k, v in d.items()}, "softmax")
    # texture-only backward: same texel gradients as the full backward
    g = grad_of((B, 4, isz, isz), 5)
    full = run(fv, tex, isz, aa, g)
    tonly = run(fv, tex, isz, aa, g, geom_grad=False)
    assert torch.equal(full["grad_tex"], tonly["grad_tex"])


SOFT = dict(sigma_val=1e-4, dist_eps=1e-4, gamma_val=1e-3)   # wider soft edges for the generic modes (as test_raster_modes_gpu)
GENERIC = [dict(dist_func="hard"), dict(dist_func="barycentric"), dict(aggr_func_alpha="hard"), dict(aggr_func_alpha="sum"),
           dict(texture_type="vertex")]


@pytest.mark.parametrize("rgb", ["softmax", "hard"])
@pytest.mark.parametrize("mode", GENERIC, ids=lambda m: "-".join("%s=%s" % kv for kv in m.items()))
def test_generic_modes(det, mode, rgb):
    """One generic combination per distance, alpha and texture mode: bitwise reproducible across runs and pair-buffer
    settings, equal to oracle B and to the default generic kernels under the parity gates; a texture-only backward gives
    the full backward's texture gradient."""
    fv, tex = scene(2, 2, 2, seed=13)
    if mode.get("texture_type") == "vertex":
        tex = np.ascontiguousarray(np.random.default_rng(14).uniform(0, 1, size=(2, fv.shape[1], 3, 3)).astype(np.float32))
    kw = dict(SOFT, **mode)
    isz, aa = 40, True
    g = grad_of((2, 4, isz, isz), 15)
    ref = run(fv, tex, isz, aa, g, rgb, **kw)
    assert_equal(ref, run(fv, tex, isz, aa, g, rgb, tile=32, cand=0.0, **kw), "generic:")
    img, fwd, cfg = softras.render(fv, tex, isz, anti_aliasing=aa, impl="B", aggr_func_rgb=rgb, **dict(UMR, **kw))
    gf, gt = softras.render_backward(fwd, cfg, g, anti_aliasing=aa, impl="B")
    got = {k: (v.numpy() if v is not None else None) for k, v in ref.items()}
    check_close(got, dict(images=img, aggrs=fwd["aggrs_info"], p2f=fwd["p2f_info"], grad_faces=gf, grad_tex=gt), rgb)
    torch.use_deterministic_algorithms(False)
    default = {k: (v.numpy() if v is not None else None) for k, v in run(fv, tex, isz, aa, g, rgb, **kw).items()}
    torch.use_deterministic_algorithms(True)
    check_close(got, default, rgb)
    tonly = run(fv, tex, isz, aa, g, rgb, geom_grad=False, **kw)
    assert torch.equal(ref["grad_tex"], tonly["grad_tex"])


def test_part_matching_loss_under_the_flag(det):
    """part_matching_loss takes its generic two-render branch under the flag (the fused vertex kernel is off there) and is
    bitwise reproducible; its loss and gradient agree with the packed 4-channel render of the default mode."""
    B, IS, T = 2, 32, 2
    rng = np.random.default_rng(11)
    v, f = synth.icosphere(2)
    F_ = f.shape[0]
    part = rng.integers(0, 5, size=(F_, T * T))
    one_hot = torch.zeros(1, F_, T * T, 5)
    one_hot.scatter_(3, torch.from_numpy(part)[None, :, :, None], 1.0)
    verts0 = torch.from_numpy(synth.bird_like(v, rng, B))
    faces = torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1).to(DEV)
    cams = torch.from_numpy(synth.cameras(rng, B)).to(DEV)
    part_segs = torch.rand(B, 5, IS, IS, generator=torch.Generator().manual_seed(1)).to(DEV)

    def step():
        m = loss_utils.part_matching_loss(None, None, 0, im_size=IS, batch_size=B, tex_size=T, stex_one_hot=one_hot).to(DEV)
        vv = verts0.clone().to(DEV).requires_grad_(True)
        loss, projs = m(vv, faces, cams, part_segs)
        loss.backward()
        torch.cuda.synchronize()
        return loss.detach().cpu(), vv.grad.cpu()

    a, b = step(), step()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    torch.use_deterministic_algorithms(False)
    d = step()
    torch.use_deterministic_algorithms(True)
    assert abs(float(a[0]) - float(d[0])) <= 1e-5 * max(1.0, abs(float(d[0])))
    ok, msg = rel_report("dverts", a[1].numpy(), d[1].numpy(), 1e-3, 1e-5 * float(d[1].abs().max()))
    assert ok, msg


def test_threads_side_streams_and_graph_replay(det):
    fv, tex, isz, aa = c2_scene()
    fv, tex = fv[:4], tex[:4]
    g = grad_of((4, 4, isz, isz), 6)
    ref = run(fv, tex, isz, aa, g)
    results = [None] * 4

    def work(i):
        torch.use_deterministic_algorithms(True)
        results[i] = run(fv, tex, isz, aa, g, stream=torch.cuda.Stream(device=DEV))

    ts = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for r in results:
        assert_equal(ref, r, "thread:")
    # CUDA graph: forward + backward captured once, replayed twice
    tfv = torch.from_numpy(fv).to(DEV).requires_grad_(True)
    ttex = torch.from_numpy(tex).to(DEV).requires_grad_(True)
    tg = torch.from_numpy(g).to(DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):  # warm-up outside the capture
            tfv.grad = ttex.grad = None
            img, p2f, aggr = raster.soft_rasterize(tfv, ttex, isz, anti_aliasing=aa, **UMR)
            img.backward(tg)
    torch.cuda.current_stream().wait_stream(s)
    tfv.grad = ttex.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        img, p2f, aggr = raster.soft_rasterize(tfv, ttex, isz, anti_aliasing=aa, **UMR)
        img.backward(tg)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        got = dict(images=img.detach().cpu(), p2f=p2f.cpu(), aggrs=aggr.cpu(), grad_faces=tfv.grad.cpu(), grad_tex=ttex.grad.cpu())
        assert_equal(ref, got, "graph replay:")


def test_soft_renderer_end_to_end(det):
    """SoftRenderer with 4 camera hypotheses per mesh: bitwise-equal gradients for the mean shape, cameras and texture under
    the flag (generic torch vertex chain), and the fused vertex kernel is still taken with the flag off."""
    B, H, IS, T = 2, 4, 32, 6
    rng = np.random.default_rng(12)
    v, f = synth.icosphere(2)
    vs0 = torch.from_numpy(synth.bird_like(v, rng, B))
    fs = torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1).to(DEV)
    cams0 = torch.from_numpy(np.stack([synth.cameras(rng, H) for _ in range(B)])).view(-1, 7)
    tx0 = torch.from_numpy(rng.uniform(0, 1, size=(B, f.shape[0], T * T, 3)).astype(np.float32))
    w = torch.linspace(0.5, 1.5, B * H * 4 * IS * IS, device=DEV).view(B * H, 4, IS, IS)

    def step():
        r = smr.SoftRenderer(IS, "softmax")
        vs = vs0.clone().to(DEV).requires_grad_(True)
        tx = tx0.clone().to(DEV).requires_grad_(True)
        c = cams0.clone().to(DEV).requires_grad_(True)
        img, _, _ = r(vs, fs, c, tx)
        (img * w).sum().backward()
        torch.cuda.synchronize()
        return img.detach().cpu(), vs.grad.cpu(), c.grad.cpu(), tx.grad.cpu()

    outs = [step() for _ in range(3)]
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert torch.equal(a, b)
    # flag off: the fused vertex kernel runs -- 3 more launches than the same step with the pipeline switched off
    # (umr_project_faces_forward: 1, umr_project_faces_backward: 2)
    lib = _lib.load()
    torch.use_deterministic_algorithms(False)
    counts = []
    try:
        for fused in (True, False):
            smr.SoftRenderer.fuse_vertex_pipeline = fused
            n0 = lib.umr_launch_count()
            out = step()
            counts.append(lib.umr_launch_count() - n0)
            if fused:
                default = out
    finally:
        smr.SoftRenderer.fuse_vertex_pipeline = True
        torch.use_deterministic_algorithms(True)
    assert counts[0] - counts[1] == 3, counts
    for k in (0, 1, 2, 3):   # the textured lighting of the two vertex chains agrees to ~1e-7, not bit for bit
        ok, msg = rel_report("grad", outs[0][k].numpy(), default[k].numpy(), 2e-4, 2e-5 * float(default[k].abs().max()))
        assert ok, msg
