"""The silhouette render on the H100, against the full render it replaces on the same inputs.

Alpha is bitwise the full render's alpha plane.  The vertex gradient equals the full render's gradient when only the
alpha plane has an adjoint: at the 1e-4 relative gate in the default mode (float atomics), bitwise and bitwise run after
run in the deterministic mode.  Covered: softmax and hard colours of the full render, anti-aliasing on and off, 64^2,
256^2 and an odd size, 16x16 and 32x32 tiles, full / partial / absent pair buffers, 65535 and 65537 faces, near / far
planes that cut faces, a NaN vertex, MultiMaskLoss with 1 and 8 camera hypotheses, launch counts, memory and CUDA-graph
replay."""
import contextlib

import numpy as np
import pytest
import torch

from umr_b200 import raster, synth
from umr_b200.graph import GraphedStep
from umr_b200.nnutils import loss_utils
from util import rel_report, scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
UMR = dict(sigma_val=1e-5, dist_eps=1e-10, gamma_val=1e-4, eps=1e-3, fill_back=True)
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


def _stats(out):
    saved = out.grad_fn.saved_tensors
    return saved[-1][:8].view(torch.int32).cpu().tolist() if saved[-1].dtype == torch.uint8 else None


def _full(fv, tex, size, rgb, g, aa, near=1, far=100):
    """The full render, backward with the alpha adjoint g [B,is,is] and zero colour adjoints."""
    tfv = fv.clone().requires_grad_(True)
    img, _, _ = raster.soft_rasterize(tfv, tex, size, aggr_func_rgb=rgb, anti_aliasing=aa, near=near, far=far, **UMR)
    stats = _stats(img)
    gi = torch.zeros_like(img)
    gi[:, 3] = g
    img.backward(gi)
    torch.cuda.synchronize()
    return dict(alpha=img.detach()[:, 3], grad=tfv.grad, stats=stats)


def _sil(fv, size, g, aa, near=1, far=100):
    tfv = fv.clone().requires_grad_(True)
    alpha = raster.soft_rasterize_silhouettes(tfv, size, anti_aliasing=aa, near=near, far=far, **UMR)
    stats = _stats(alpha)
    alpha.backward(g)
    torch.cuda.synchronize()
    return dict(alpha=alpha.detach(), grad=tfv.grad, stats=stats)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _inputs(B, subdiv, tex_res, size, seed):
    fv, tex = scene(B, subdiv, tex_res, seed=seed)
    g = np.random.default_rng(seed + 1).normal(size=(B, size, size)).astype(np.float32)
    return torch.from_numpy(fv).to(DEV), torch.from_numpy(tex).to(DEV), torch.from_numpy(g).to(DEV)


def _close(name, got, ref, rtol=1e-4):
    got, ref = got.detach().cpu().numpy(), ref.detach().cpu().numpy()
    at = 1e-6 * float(np.abs(ref).max() + 1e-30) + 1e-7
    ok, msg = rel_report(name, got, ref, rtol, at)
    print(msg)
    assert ok, msg


SIZES = [(16, 3, 3, 64), (16, 3, 6, 256), (8, 2, 2, 61)]   # (renders, icosphere subdivision, texture side, image size)


@pytest.mark.parametrize("B,subdiv,tex_res,size", SIZES)
@pytest.mark.parametrize("tile", [16, 32])
@pytest.mark.parametrize("pairs", sorted(PAIRS))
@pytest.mark.parametrize("rgb", ["softmax", "hard"])
def test_silhouette_default_mode(rgb, pairs, tile, B, subdiv, tex_res, size):
    fv, tex, g = _inputs(B, subdiv, tex_res, size, seed=size + tile)
    with _modes(cand=PAIRS[pairs], tile=tile):
        sil = _sil(fv, size, g, True)
        full = _full(fv, tex, size, rgb, g, True)
    assert torch.equal(_bits(sil["alpha"]), _bits(full["alpha"]))
    if pairs == "full":
        assert sil["stats"][1] == 0 and sil["stats"][0] > 0, sil["stats"]
        assert sil["stats"] == full["stats"], "the same pairs, the same blocks"
    elif pairs == "partial":
        assert sil["stats"][1] > 0, "the partial buffer must leave tiles unsaved: %s" % (sil["stats"],)
    else:
        assert sil["stats"] is None
    assert sil["grad"].abs().sum() > 0
    _close("grad_faces", sil["grad"], full["grad"])


@pytest.mark.parametrize("B,subdiv,tex_res,size", SIZES)
@pytest.mark.parametrize("tile", [16, 32])
def test_silhouette_without_anti_aliasing(tile, B, subdiv, tex_res, size):
    fv, tex, g = _inputs(B, subdiv, tex_res, size, seed=size + 3)
    with _modes(tile=tile):
        sil = _sil(fv, size, g, False)
        full = _full(fv, tex, size, "softmax", g, False)
    with _modes(det=True):
        sil_d = _sil(fv, size, g, False)
        full_d = _full(fv, tex, size, "softmax", g, False)
    assert torch.equal(_bits(sil["alpha"]), _bits(full["alpha"]))
    assert torch.equal(_bits(sil_d["alpha"]), _bits(full["alpha"]))
    _close("grad_faces", sil["grad"], full["grad"])
    assert torch.equal(_bits(sil_d["grad"]), _bits(full_d["grad"]))


@pytest.mark.parametrize("B,subdiv,tex_res,size", SIZES)
@pytest.mark.parametrize("rgb", ["softmax", "hard"])
def test_silhouette_deterministic_is_bitwise(rgb, B, subdiv, tex_res, size):
    fv, tex, g = _inputs(B, subdiv, tex_res, size, seed=size)
    with _modes(det=True):
        sil = _sil(fv, size, g, True)
        full = _full(fv, tex, size, rgb, g, True)
        again = _sil(fv, size, g, True)
    assert torch.equal(_bits(sil["alpha"]), _bits(full["alpha"]))
    assert torch.equal(_bits(sil["grad"]), _bits(full["grad"]))
    assert torch.equal(_bits(sil["grad"]), _bits(again["grad"]))
    assert sil["grad"].abs().sum() > 0


def _wide_mesh(F, B=2, seed=0):
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


@pytest.mark.parametrize("F", [65535, 65537])
@pytest.mark.parametrize("mode", ["default-full", "default-partial", "default-tile32", "deterministic"])
def test_silhouette_large_meshes(F, mode):
    fv, tex = _wide_mesh(F)
    size = 64
    g = torch.from_numpy(np.random.default_rng(3).normal(size=(fv.shape[0], size, size)).astype(np.float32)).to(DEV)
    det = mode == "deterministic"
    with _modes(det=det, cand=PAIRS.get(mode.split("-")[-1], 32.0), tile=32 if mode == "default-tile32" else 0):
        sil = _sil(fv, size, g, True)
        full = _full(fv, tex, size, "softmax", g, True)
    assert torch.equal(_bits(sil["alpha"]), _bits(full["alpha"]))
    if det:
        assert torch.equal(_bits(sil["grad"]), _bits(full["grad"]))
    else:
        _close("grad_faces", sil["grad"], full["grad"])
    assert sil["grad"].abs().sum() > 0


@pytest.mark.parametrize("det", [False, True])
def test_near_and_far_planes_cutting_faces(det):
    fv, tex, g = _inputs(8, 3, 3, 64, seed=5)
    z = fv.view(8, -1, 3, 3)[..., 2]
    near, far = float(torch.quantile(z, 0.3)), float(torch.quantile(z, 0.7))   # both planes cut through the meshes
    with _modes(det=det):
        sil = _sil(fv, 64, g, True, near=near, far=far)
        full = _full(fv, tex, 64, "softmax", g, True, near=near, far=far)
        uncut = _sil(fv, 64, g, True)
    assert torch.equal(_bits(sil["alpha"]), _bits(full["alpha"]))
    assert torch.equal(_bits(sil["alpha"]), _bits(uncut["alpha"])), "pairs outside (near, far) still count in alpha"
    assert not torch.equal(sil["grad"], uncut["grad"]), "... and get no gradient"
    if det:
        assert torch.equal(_bits(sil["grad"]), _bits(full["grad"]))
    else:
        _close("grad_faces", sil["grad"], full["grad"])


@pytest.mark.parametrize("det", [False, True])
def test_nan_vertex(det):
    fv, tex, g = _inputs(4, 3, 3, 64, seed=7)
    fv = fv.clone()
    fv.view(4, -1, 9)[1, 40, 0] = float("nan")
    with _modes(det=det):
        sil = _sil(fv, 64, g, True)
        full = _full(fv, tex, 64, "softmax", g, True)
    assert torch.equal(_bits(sil["alpha"]), _bits(full["alpha"]))
    assert torch.equal(torch.isnan(sil["grad"]), torch.isnan(full["grad"]))
    if det:
        assert torch.equal(_bits(sil["grad"]), _bits(full["grad"]))
    else:
        ok = ~torch.isnan(full["grad"])
        _close("grad_faces (finite)", sil["grad"][ok], full["grad"][ok])


# --- MultiMaskLoss: the silhouette route against the full render (taken while a wrapper sits on SoftRasterizeFunction) --
@contextlib.contextmanager
def _full_route():
    orig = raster.SoftRasterizeFunction.apply
    raster.SoftRasterizeFunction.apply = staticmethod(lambda *a: orig(*a))
    try:
        yield
    finally:
        raster.SoftRasterizeFunction.apply = orig


def _mask_step(d, IS, H, full):
    vs = d["vs"].clone().requires_grad_(True)
    cams = d["cams"].clone().requires_grad_(True)
    probs = d["probs"].clone().requires_grad_(True)
    m = loss_utils.MultiMaskLoss(IS, "softmax", H)
    with (_full_route() if full else contextlib.nullcontext()):
        loss, mask_all = m(vs, d["fs"], cams, probs, d["masks"])
        grads = torch.autograd.grad(loss, (vs, cams, probs))
    torch.cuda.synchronize()
    return loss.detach(), mask_all.detach(), grads


def _mask_scene(B, H, IS, seed=21):
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(2)
    d = dict(vs=torch.from_numpy(synth.bird_like(v, rng, B)),
             fs=torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1),
             cams=torch.from_numpy(np.stack([synth.cameras(rng, H) for _ in range(B)])),
             probs=torch.softmax(torch.from_numpy(rng.normal(size=(B, H)).astype(np.float32)), 1),
             masks=torch.from_numpy(synth.ellipse_masks(rng, B, IS)))
    return {k: t.to(DEV) for k, t in d.items()}


@pytest.mark.parametrize("IS", [64, 61])
@pytest.mark.parametrize("H", [1, 8])
@pytest.mark.parametrize("det", [False, True])
def test_multi_mask_loss_matches_the_full_render(det, H, IS):
    d = _mask_scene(2, H, IS)
    with _modes(det=det, cand=raster.PAIR_CAND_PER_PIXEL):
        got = _mask_step(d, IS, H, False)
        ref = _mask_step(d, IS, H, True)
        again = _mask_step(d, IS, H, False)
    assert torch.equal(_bits(got[1]), _bits(ref[1])), "mask_all_hypo"
    if det:
        assert torch.equal(got[0], ref[0]), "mask_loss"
    else:
        _close("mask_loss", got[0], ref[0])
    for name, a, b, c in zip(("vs", "cams", "probs"), got[2], ref[2], again[2]):
        assert a.abs().sum() > 0, name
        if det:
            assert torch.equal(_bits(a), _bits(b)), name
            assert torch.equal(_bits(a), _bits(c)), name
        else:
            _close("grad " + name, a, b)


def _kernel_counts(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return {k: sum(1 for n in names if k in n) for k in ("k_project_faces", "k_raster_fwd", "k_raster_bwd2", "k_p2f_finalize")}


def test_launch_count_one_forward_one_backward():
    d = _mask_scene(2, 8, 64)
    with _modes():
        sil = _kernel_counts(lambda: _mask_step(d, 64, 8, False))
        full = _kernel_counts(lambda: _mask_step(d, 64, 8, True))
    assert sil["k_project_faces"] == full["k_project_faces"] > 0, (sil, full)
    assert (sil["k_raster_fwd"], sil["k_raster_bwd2"], sil["k_p2f_finalize"]) == (1, 1, 0), sil
    assert (full["k_raster_fwd"], full["k_raster_bwd2"], full["k_p2f_finalize"]) == (1, 1, 1), full


def test_no_colour_or_aggregation_planes_are_allocated():
    B, IS = 16, 128
    S = 2 * IS
    fv, _, g = _inputs(B, 3, 3, IS, seed=9)
    fv = fv.clone().requires_grad_(True)
    colors_hi, aggrs = B * 4 * S * S * 4, B * 2 * S * S * 4
    alpha_hi = B * S * S * 4
    with _modes(cand=0.0):   # no pair buffer: what remains is the planes and the workspace
        raster.soft_rasterize_silhouettes(fv, IS, anti_aliasing=True, **UMR).backward(g)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        alpha = raster.soft_rasterize_silhouettes(fv, IS, anti_aliasing=True, **UMR)
        alpha.backward(g)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
    ws = raster._lib.load().umr_raster_workspace_bytes(B, fv.shape[1], IS, 1)
    # alpha, alpha_hi, two workspaces at most (forward's is freed before the backward's), grad_faces and allocator slack
    assert peak < alpha_hi + 2 * ws + B * IS * IS * 4 + fv.numel() * 4 + (4 << 20), peak
    assert peak < ws + min(colors_hi, aggrs), (peak, ws, colors_hi, aggrs)


@pytest.mark.parametrize("det", [False, True])
def test_graphed_step_replay_equals_eager(det):
    IS, H = 64, 8
    d = _mask_scene(2, H, IS)
    vs = d["vs"].clone().requires_grad_(True)
    cams = d["cams"].clone().requires_grad_(True)
    probs = d["probs"].clone().requires_grad_(True)
    m = loss_utils.MultiMaskLoss(IS, "softmax", H)

    def step():
        loss, _ = m(vs, d["fs"], cams, probs, d["masks"])
        return (loss,) + torch.autograd.grad(loss, (vs, cams, probs))

    with _modes(det=det, cand=raster.PAIR_CAND_PER_PIXEL):
        eager = [t.detach().clone() for t in step()]
        graphed = GraphedStep(step, warmup=2)
        for _ in range(2):
            out = graphed()
            torch.cuda.synchronize()
            for name, a, b in zip(("loss", "vs", "cams", "probs"), out, eager):
                if det:
                    assert torch.equal(a, b), name
                else:
                    _close("replay " + name, a, b)
