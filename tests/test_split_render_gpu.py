"""The split raster backward on the H100, against the two-render composition it replaces on the same inputs: a render of
the live geometry whose alpha plane takes the mask loss, and a render of the detached geometry whose RGB planes take the
texture loss (experiments/train_s2.py: MultiMaskLoss, then MultiTextureLoss on pred_vs.detach()).

Forward planes are bitwise those of the composition.  Gradients agree at the 1e-4 relative gate in the default mode (float
atomics) and bitwise, run after run, in the deterministic mode.  Covered: softmax and hard colours, full / partial / absent
pair buffers, 16x16 and 32x32 tiles, textures shared by G = 1 or 8 renders, 64^2, 256^2 and an odd size, and 65537 faces
(the 32-bit face-index kernels) with face F-1 on screen."""
import contextlib

import numpy as np
import pytest
import torch

from umr_b200 import raster, synth
from umr_b200.nnutils import loss_utils, smr
from util import rel_report, scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
UMR = dict(sigma_val=1e-5, dist_eps=1e-10, gamma_val=1e-4, eps=1e-3, near=1, far=100, fill_back=True)
PAIRS = {"full": 32.0, "partial": 0.7, "absent": 0.0}


@contextlib.contextmanager
def _modes(det=False, cand=32.0, tile=0):
    old = (raster.PAIR_CAND_PER_PIXEL, raster.FORWARD_TILE, raster.PAIR_ADAPTIVE, torch.are_deterministic_algorithms_enabled())
    raster.PAIR_CAND_PER_PIXEL, raster.FORWARD_TILE, raster.PAIR_ADAPTIVE = cand, tile, False
    torch.use_deterministic_algorithms(det)
    try:
        yield
    finally:
        raster.PAIR_CAND_PER_PIXEL, raster.FORWARD_TILE, raster.PAIR_ADAPTIVE = old[:3]
        torch.use_deterministic_algorithms(old[3])


def _render(fn, fv, tex, size, rgb, g, geom=True, texg=True):
    tfv = fv.clone().requires_grad_(geom)
    ttex = tex.clone().requires_grad_(texg)
    img, p2f, aggr = fn(tfv, ttex, size, aggr_func_rgb=rgb, anti_aliasing=True, **UMR)
    saved = img.grad_fn.saved_tensors
    stats = saved[4][:8].view(torch.int32).cpu().tolist() if len(saved) == 5 else None
    img.backward(g)
    torch.cuda.synchronize()
    return dict(images=img.detach(), p2f=p2f, aggrs=aggr, grad_faces=tfv.grad, grad_tex=ttex.grad, stats=stats)


def _split_and_composed(fv, tex, size, rgb, g):
    split = _render(raster.soft_rasterize_split, fv, tex, size, rgb, g)
    g_alpha = g.clone()
    g_alpha[:, :3] = 0
    g_rgb = g.clone()
    g_rgb[:, 3] = 0
    mask = _render(raster.soft_rasterize, fv, tex, size, rgb, g_alpha, texg=False)   # the mask branch: alpha only
    texr = _render(raster.soft_rasterize, fv, tex, size, rgb, g_rgb, geom=False)     # the texture branch: detached geometry
    assert torch.equal(split["images"][:, 3], mask["images"][:, 3]), "alpha vs the mask render"
    assert torch.equal(split["images"][:, :3], texr["images"][:, :3]), "RGB vs the textured render"
    assert torch.equal(split["aggrs"], texr["aggrs"])
    return split, mask, texr


def _inputs(B, G, subdiv, tex_res, size, seed):
    fv, tex = scene(B, subdiv, tex_res, seed=seed)
    fv = torch.from_numpy(fv).to(DEV)
    tex = torch.from_numpy(tex[:B // G]).to(DEV)
    g = torch.from_numpy(np.random.default_rng(seed + 1).normal(size=(B, 4, size, size)).astype(np.float32)).to(DEV)
    return fv, tex, g


def _close(name, got, ref, rtol=1e-4):
    got, ref = got.detach().cpu().numpy(), ref.detach().cpu().numpy()
    at = 1e-6 * float(np.abs(ref).max() + 1e-30) + 1e-7
    ok, msg = rel_report(name, got, ref, rtol, at)
    print(msg)
    assert ok, msg


SIZES = [(16, 3, 3, 64), (16, 3, 6, 256), (8, 2, 2, 61)]   # (renders, icosphere subdivision, texture side, image size)


@pytest.mark.parametrize("B,subdiv,tex_res,size", SIZES)
@pytest.mark.parametrize("G", [1, 8])
@pytest.mark.parametrize("tile", [16, 32])
@pytest.mark.parametrize("pairs", sorted(PAIRS))
@pytest.mark.parametrize("rgb", ["softmax", "hard"])
def test_split_backward_default_mode(rgb, pairs, tile, G, B, subdiv, tex_res, size):
    fv, tex, g = _inputs(B, G, subdiv, tex_res, size, seed=size + G)
    with _modes(cand=PAIRS[pairs], tile=tile):
        split, mask, texr = _split_and_composed(fv, tex, size, rgb, g)
    if pairs == "full":
        assert split["stats"][1] == 0 and split["stats"][0] > 0, split["stats"]
    elif pairs == "partial":
        assert split["stats"][1] > 0, "the partial buffer must leave tiles unsaved: %s" % (split["stats"],)
    else:
        assert split["stats"] is None
    _close("grad_faces", split["grad_faces"], mask["grad_faces"])
    _close("grad_tex", split["grad_tex"], texr["grad_tex"])


@pytest.mark.parametrize("B,subdiv,tex_res,size", SIZES)
@pytest.mark.parametrize("G", [1, 8])
@pytest.mark.parametrize("rgb", ["softmax", "hard"])
def test_split_backward_deterministic_is_bitwise(rgb, G, B, subdiv, tex_res, size):
    fv, tex, g = _inputs(B, G, subdiv, tex_res, size, seed=size + G)
    with _modes(det=True):
        split, mask, texr = _split_and_composed(fv, tex, size, rgb, g)
        again = _render(raster.soft_rasterize_split, fv, tex, size, rgb, g)
    assert torch.equal(split["grad_faces"], mask["grad_faces"])
    assert torch.equal(split["grad_tex"], texr["grad_tex"])
    assert torch.equal(split["grad_faces"], again["grad_faces"]) and torch.equal(split["grad_tex"], again["grad_tex"])
    assert split["grad_faces"].abs().sum() > 0 and split["grad_tex"].abs().sum() > 0


def _wide_mesh(F=65537, B=2, seed=0):
    """F faces of a deformed icosphere(7), ordered so that face F-1 is a near-side face at the raster's centre."""
    v, f = synth.icosphere(7)
    rng = np.random.default_rng(seed)
    fv = synth.raster_space_faces(synth.bird_like(v, rng, B), f, synth.cameras(rng, B))
    c = fv[0].reshape(-1, 3, 3).mean(axis=1)
    near = c[:, 2] < np.median(c[:, 2])
    order = np.lexsort((-np.hypot(c[:, 0] - 1 / 64, c[:, 1] - 1 / 64), near))
    fv = np.ascontiguousarray(fv[:, order[-F:]])
    tex = rng.uniform(0, 1, size=(B, F, 4, 3)).astype(np.float32)
    return torch.from_numpy(fv).to(DEV), torch.from_numpy(tex).to(DEV)


@pytest.mark.parametrize("mode", ["default-full", "default-partial", "default-absent", "default-tile32", "deterministic"])
def test_split_backward_65537_faces(mode):
    fv, tex = _wide_mesh()
    size = 64
    g = torch.from_numpy(np.random.default_rng(3).normal(size=(fv.shape[0], 4, size, size)).astype(np.float32)).to(DEV)
    det = mode == "deterministic"
    cand = PAIRS.get(mode.split("-")[-1], 32.0)
    with _modes(det=det, cand=cand, tile=32 if mode == "default-tile32" else 0):
        split, mask, texr = _split_and_composed(fv, tex, size, "softmax", g)
    if det:
        assert torch.equal(split["grad_faces"], mask["grad_faces"]) and torch.equal(split["grad_tex"], texr["grad_tex"])
    else:
        _close("grad_faces", split["grad_faces"], mask["grad_faces"])
        _close("grad_tex", split["grad_tex"], texr["grad_tex"])
    # face F-1 covers pixels (its p2f) and takes texel gradient (an interior face: alpha == 1 there, so the alpha path
    # gives its vertices no gradient -- in the composition as here)
    F = fv.shape[1]
    assert split["p2f"][:, F - 1].abs().max() > 0, "face F-1 must be on screen"
    assert split["grad_tex"][:, F - 1].abs().sum() > 0
    assert split["grad_faces"].abs().sum() > 0


# --- MultiMaskTextureLoss against the composed modules ---------------------------------------------------------------
H = 8


def _scene(B, IS, dtype, seed=21):
    """The train-step scene of test_train_step_gpu at raster size IS: B meshes x 8 camera hypotheses."""
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(2)
    T = 3
    d = dict(
        vs=torch.from_numpy(synth.bird_like(v, rng, B)),
        fs=torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1),
        cams=torch.from_numpy(np.stack([synth.cameras(rng, H) for _ in range(B)])),
        probs=torch.softmax(torch.from_numpy(rng.normal(size=(B, H)).astype(np.float32)), 1),
        masks=torch.from_numpy(synth.ellipse_masks(rng, B, IS)),
        imgs=torch.from_numpy(synth.smooth_images(rng, B, IS)),
        flow=torch.from_numpy(synth.texture_flow(rng, B, f.shape[0], T)),
        tx=torch.from_numpy(rng.uniform(0, 1, size=(B, f.shape[0], T * T, 3)).astype(np.float32)),
    )
    d["dts"] = torch.from_numpy(np.stack([synth.dt_barrier(m) for m in d["masks"].numpy()]))[:, None]
    d["proj_cam"] = d["cams"][:, 0].clone()
    return {k: (t.to(DEV).to(dtype) if t.is_floating_point() else t.to(DEV)) for k, t in d.items()}


LEAVES = ("vs", "cams", "probs", "tx", "flow")


def _step(d, IS, fused):
    x = {k: (d[k].clone().requires_grad_(True) if k in LEAVES else d[k]) for k in d}
    if fused:
        m = loss_utils.MultiMaskTextureLoss(x["vs"].shape[0], H, IS, "softmax", texture_loss_type="l1")
        out = m(x["vs"], x["fs"], x["cams"], x["probs"], x["proj_cam"], x["imgs"], x["masks"], x["tx"], x["flow"], x["dts"])
    else:
        mm = loss_utils.MultiMaskLoss(IS, "softmax", H)
        mt = loss_utils.MultiTextureLoss(x["vs"].shape[0], H, IS, "softmax", texture_loss_type="l1")
        mask_loss, mask_all = mm(x["vs"], x["fs"], x["cams"], x["probs"], x["masks"])
        out = (mask_loss, mask_all) + tuple(mt(x["vs"].detach(), x["fs"], x["cams"].detach(), x["probs"].detach(),
                                               x["proj_cam"], x["imgs"], x["masks"], mask_all, x["tx"], x["flow"], x["dts"]))
    mask_loss, mask_all, tex_loss, dt_loss, cyc_loss, tex_pred = out
    total = mask_loss + 0.5 * tex_loss + 0.25 * dt_loss + 0.125 * cyc_loss
    grads = torch.autograd.grad(total, [x[k] for k in LEAVES])
    torch.cuda.synchronize()
    return [t.detach() for t in out], dict(zip(LEAVES, grads))


@pytest.mark.parametrize("IS", [64, 256, 61])
@pytest.mark.parametrize("det", [False, True])
def test_multi_mask_texture_loss_matches_composed_modules(IS, det):
    d = _scene(2, IS, torch.float32)
    with _modes(det=det, cand=raster.PAIR_CAND_PER_PIXEL, tile=0):
        got_out, got_g = _step(d, IS, True)
        ref_out, ref_g = _step(d, IS, False)
        again_out, again_g = _step(d, IS, True) if det else (None, None)
    assert torch.equal(got_out[1], ref_out[1]), "mask_all_hypo"
    assert torch.equal(got_out[5], ref_out[5]), "texture_pred"
    for i, name in ((0, "mask_loss"), (2, "tex_loss"), (3, "tex_dt_loss"), (4, "tex_cycle_loss")):
        if det:
            assert torch.equal(got_out[i], ref_out[i]), name
        else:
            _close(name, got_out[i], ref_out[i])
    for k in LEAVES:
        assert got_g[k].abs().sum() > 0 or k == "flow", k
        if det:
            assert torch.equal(got_g[k], ref_g[k]), k
            assert torch.equal(got_g[k], again_g[k]), k
        else:
            _close("grad " + k, got_g[k], ref_g[k])


def test_multi_mask_texture_loss_float64_composes():
    IS = 32
    d = _scene(2, IS, torch.float64)
    with _modes(det=False):
        got_out, got_g = _step(d, IS, True)
        ref_out, ref_g = _step(d, IS, False)
    assert got_out[1].dtype == torch.float64
    for i in range(6):
        _close("output %d" % i, got_out[i], ref_out[i], rtol=1e-10)
    for k in LEAVES:
        _close("grad " + k, got_g[k], ref_g[k], rtol=1e-10)


def _kernel_counts(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return {k: sum(1 for n in names if k in n) for k in ("k_project_faces", "k_raster_fwd", "k_raster_bwd2")}


def test_launch_count_one_render_instead_of_two():
    IS = 64
    d = _scene(2, IS, torch.float32)
    with _modes():
        fused = _kernel_counts(lambda: _step(d, IS, True))
        composed = _kernel_counts(lambda: _step(d, IS, False))
    # both also project once for MultiTextureLoss's hard visibility render (k_visible_faces, not a raster forward)
    assert composed == {"k_project_faces": 3, "k_raster_fwd": 2, "k_raster_bwd2": 2}, composed
    assert fused == {"k_project_faces": 2, "k_raster_fwd": 1, "k_raster_bwd2": 1}, fused


@pytest.mark.parametrize("det", [False, True])
def test_cuda_graph_replay_equals_eager(det):
    IS = 64
    d = _scene(2, IS, torch.float32)
    r = smr.SoftRenderer(IS, "softmax")
    r.ambient_light_only()
    vs = d["vs"].clone().requires_grad_(True)
    cams = d["cams"].view(-1, 7).clone().requires_grad_(True)
    tx = d["tx"].clone().requires_grad_(True)
    target = torch.rand(vs.shape[0] * H, 4, IS, IS, device=DEV)

    def step():
        images, _, _ = r.render_split(vs, d["fs"], cams, tx)
        loss = ((images - target) ** 2).mean()
        return (loss,) + torch.autograd.grad(loss, (vs, cams, tx))

    with _modes(det=det, cand=raster.PAIR_CAND_PER_PIXEL):
        eager = [t.detach().clone() for t in step()]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                step()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static = step()
        for _ in range(2):
            graph.replay()
            torch.cuda.synchronize()
            for name, a, b in zip(("loss", "vs", "cams", "tx"), static, eager):
                if det:
                    assert torch.equal(a, b), name
                else:
                    _close("replay " + name, a, b)
