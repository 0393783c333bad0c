"""Cost of the deterministic mode (torch.use_deterministic_algorithms(True)): the train_s2-shaped loss step of
tools/train_step_bench.py with the flag off and on, and every loss op that has a deterministic entry point, default vs
deterministic, at the C2 / C3 batch shapes of BASELINE.md.  CUDA events after warm-up, one process; medians.
--texture-renderer picks MultiTextureLoss's renderer (the soft rasteriser or the NMR z-buffer); --no-ops skips the
per-op table.

    python tools/deterministic_step_bench.py [--iters 20] [--steps 10] [--texture-renderer smr|nmr] [--no-ops]
                                             [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # SoftRenderer's generic torch chain, where it falls back to it
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from umr_b200 import ops, synth  # noqa: E402
from umr_b200 import soft_renderer as sr  # noqa: E402
from umr_b200.nnutils import chamfer_python, geom_utils, loss_utils  # noqa: E402

DEV = torch.device("cuda:0")
SIZES = {"C2": (16, 256), "C3": (256, 512)}   # renders, image side


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


def timed(fn, iters, warmup=3):
    """Median forward and backward milliseconds of fn() -> (loss to backprop)."""
    for _ in range(warmup):
        fn().backward()
    f_ms, b_ms = [], []
    for _ in range(iters):
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        loss = fn()
        e1.record()
        loss.backward()
        e2.record()
        torch.cuda.synchronize()
        f_ms.append(e0.elapsed_time(e1))
        b_ms.append(e1.elapsed_time(e2))
    return float(np.median(f_ms)), float(np.median(b_ms))


def op_cases(B, S):
    g = torch.Generator().manual_seed(0)
    rgba = torch.rand(B, 4, S, S, generator=g).to(DEV).requires_grad_(True)
    gt = torch.rand(B, 3, S, S, generator=g).to(DEV)
    m = (torch.rand(B, S, S, generator=g) > 0.5).float().to(DEV)
    F, T = 1280, 6
    flow = (torch.rand(B, F, T, T, 2, generator=g) * 2 - 1).to(DEV).requires_grad_(True)
    prob = (torch.rand(B, F, 2, generator=g) * 2 - 1).to(DEV)
    vis = (torch.rand(B, F, generator=g) > 0.5).to(torch.uint8).to(DEV)
    rng = np.random.default_rng(0)
    v, f = synth.icosphere(3)
    x = torch.from_numpy(synth.bird_like(v, rng, B)).to(DEV).requires_grad_(True)
    faces = torch.from_numpy(f.astype(np.int64))
    lap, flat = sr.LaplacianLoss(torch.from_numpy(v), faces).to(DEV), sr.FlattenLoss(faces).to(DEV)
    a = (torch.rand(B, 642, 2, generator=g) - 0.5).to(DEV).requires_grad_(True)
    b = (torch.rand(B, 1000, 2, generator=g) - 0.5).to(DEV).requires_grad_(True)
    parts = [torch.from_numpy(p) for p in synth.part_vertex_sets(rng, v.shape[0], sizes=(20, 40, 20, 40))]
    corr = loss_utils.CorrLossChamfer(None, S, part_vertices=parts)
    pts = [torch.from_numpy(p).to(DEV) for p in synth.part_points(rng, B)]
    cams = torch.from_numpy(synth.cameras(rng, B)).to(DEV).requires_grad_(True)
    mean_shape = torch.from_numpy(v.astype(np.float32)).to(DEV).requires_grad_(True)
    return {
        "iou (alpha plane)": lambda: loss_utils.neg_iou_loss(rgba[:, 3], m),
        "masked_l1": lambda: loss_utils.texture_loss_masks(rgba[:, :3], gt, m, rgba[:, 3]),
        "loss_head": lambda: ops.mask_texture_loss(rgba, gt, m)[0],
        "texcycle (visible)": lambda: ops.tex_cycle(flow, prob, None, vis),
        "laplacian": lambda: lap(x).mean(),
        "flatten": lambda: flat(x).mean(),
        "chamfer 642x1000": lambda: sum(o.mean() for o in chamfer_python.distChamfer(a, b)[:2]),
        "corr (shared mesh)": lambda: corr(pts[0], pts[1], pts[2], pts[3], mean_shape[None].expand(B, -1, -1), cams,
                                           avg=False).mean(),
    }


def make_step(B=16, H=8, IS=256, subdiv=3, T=6, texture_renderer="smr"):
    """tools/train_step_bench.py's step: -> (step() returning the total loss after its backward)."""
    rng = np.random.default_rng(0)
    v, f = synth.icosphere(subdiv)
    V, F = v.shape[0], f.shape[0]
    fs = torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1).to(DEV)
    imgs = torch.from_numpy(synth.smooth_images(rng, B, IS)).to(DEV)
    masks = torch.from_numpy(synth.ellipse_masks(rng, B, IS)).to(DEV)
    dts = torch.from_numpy(np.stack([synth.dt_barrier(m) for m in masks.cpu().numpy()]))[:, None].to(DEV)
    part_segs = torch.from_numpy(rng.uniform(0, 1, size=(B, 5, IS, IS)).astype(np.float32)).to(DEV)
    part = rng.integers(0, 5, size=(F, T * T))
    one_hot = torch.zeros(1, F, T * T, 5)
    one_hot.scatter_(3, torch.from_numpy(part)[None, :, :, None], 1.0)
    part_vertices = [torch.from_numpy(p) for p in synth.part_vertex_sets(rng, V, sizes=(20, 40, 20, 40))]
    head, belly, neck, back = [torch.from_numpy(p).to(DEV) for p in synth.part_points(rng, B)]
    rep = lambda t: t.unsqueeze(1).repeat(1, H, 1, 1).view(-1, t.size(1), t.size(2))
    mask_fn = loss_utils.MultiMaskLoss(IS, "softmax", H).to(DEV)
    tex_fn = loss_utils.MultiTextureLoss(B, H, IS, "softmax", "l1", texture_renderer).to(DEV)
    part_fn = loss_utils.part_matching_loss(None, None, 0, im_size=IS, batch_size=B, tex_size=T, stex_one_hot=one_hot).to(DEV)
    corr_fn = loss_utils.CorrLossChamfer(None, IS, part_vertices=part_vertices)
    fcpu = torch.from_numpy(f.astype(np.int64))
    lap_fn = sr.LaplacianLoss(torch.from_numpy(v), fcpu).to(DEV)
    flat_fn = sr.FlattenLoss(fcpu).to(DEV)
    mean_shape = torch.from_numpy(v.astype(np.float32)).to(DEV).requires_grad_(True)
    delta = (0.05 * torch.from_numpy(synth.bird_like(v, rng, B) - v[None])).float().to(DEV).requires_grad_(True)
    cams = torch.from_numpy(np.stack([synth.cameras(rng, H) for _ in range(B)])).to(DEV).requires_grad_(True)
    logits = torch.zeros(B, H, device=DEV, requires_grad=True)
    flow = torch.from_numpy(synth.texture_flow(rng, B, F, T)).to(DEV).requires_grad_(True)
    leaves = [mean_shape, delta, cams, logits, flow]

    def step():
        for t in leaves:
            t.grad = None
        pred_vs = mean_shape[None] + delta
        probs = torch.softmax(logits, 1)
        proj_cam = cams[:, 0].detach()
        mask_loss, mask_all = mask_fn(pred_vs, fs, cams, probs, masks)
        tri = lap_fn(pred_vs).mean()
        flat = flat_fn(pred_vs).mean()
        tex = geom_utils.sample_textures(flow, imgs).contiguous().view(B, F, T * T, 3)
        tl, tdt, tcyc, _ = tex_fn(pred_vs.detach(), fs, cams.detach(), probs.detach(), proj_cam, imgs, masks, mask_all,
                                  tex, flow, dts)
        pl, _ = part_fn(pred_vs, fs, proj_cam, part_segs)
        ms_rep = mean_shape[None].expand(B, -1, -1).unsqueeze(1).repeat(1, H, 1, 1).view(-1, V, 3)
        corr = corr_fn(rep(head), rep(belly), rep(back), rep(neck), ms_rep, cams.view(-1, 7), avg=False)
        corr = (corr.view(B, H) * probs).sum(1).mean()
        total = mask_loss.mean() + 0.1 * tri + 0.005 * flat + 3.0 * tl.mean() + 3.0 * tdt.mean() + tcyc.mean() \
            + 0.1 * pl.mean() + corr
        total.backward()
        return [total] + [t.grad for t in leaves]
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--texture-renderer", choices=("smr", "nmr"), default="smr")
    ap.add_argument("--no-ops", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("deterministic_step_bench needs a CUDA device")
    res = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "ops": {}}
    print("device: %s, power limit %s" % (res["device"], res["power_limit"]))

    step = make_step(texture_renderer=args.texture_renderer)
    row = {}
    for mode in ("default", "deterministic"):
        torch.use_deterministic_algorithms(mode == "deterministic")
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        ms, first, equal = [], None, True
        for _ in range(args.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = step()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
            out = [t.detach().clone() for t in out]
            if first is None:
                first = out
            else:
                equal &= all(torch.equal(x, y) for x, y in zip(first, out))
        row[mode] = {"step_ms": float(np.median(ms)), "bitwise_equal": bool(equal)}
    torch.use_deterministic_algorithms(False)
    row["ratio"] = row["deterministic"]["step_ms"] / row["default"]["step_ms"]
    row["texture_renderer"] = args.texture_renderer
    res["step"] = row
    print("train_s2-shaped step (16 x 8 hypotheses, 256^2, 1280 faces, T=6):", json.dumps(row))
    del step
    torch.cuda.empty_cache()

    for shape, (B, S) in ({} if args.no_ops else SIZES).items():
        cases = op_cases(B, S)
        for name, fn in cases.items():
            r = {}
            for mode in ("default", "deterministic"):
                torch.use_deterministic_algorithms(mode == "deterministic")
                f, b = timed(fn, args.iters)
                r[mode] = {"fwd_ms": f, "bwd_ms": b}
            torch.use_deterministic_algorithms(False)
            d, t = r["default"], r["deterministic"]
            r["ratio_total"] = (t["fwd_ms"] + t["bwd_ms"]) / (d["fwd_ms"] + d["bwd_ms"])
            res["ops"]["%s %s" % (shape, name)] = r
            print("%s B=%d %d^2  %-20s default %.3f + %.3f ms, deterministic %.3f + %.3f ms (x%.2f)"
                  % (shape, B, S, name, d["fwd_ms"], d["bwd_ms"], t["fwd_ms"], t["bwd_ms"], r["ratio_total"]))
        del cases
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
