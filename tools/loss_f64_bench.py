"""Timing and precision of the float64 loss kernels (DESIGN.md §10), CUDA events, one JSON line per measurement.

* Per op, forward + backward in float64 and, alternating call by call in the same process, in float32 on the same
  (widened) inputs, at the C2 (B = 16 images x 8 camera hypotheses, 256^2, 1280 faces, T = 6) and C3 (B = 32, 512^2)
  shapes of bench.py: the sampler (sample_textures), IoU, masked L1, the fused loss head, TexCycle, Laplacian, flatten and
  CorrLossChamfer.
* The whole train_s2-shaped loss step (tests/test_loss_f64_gpu.py `make_step`: renders, the four loss modules, the mesh
  regularisers) in float64 vs float32.
* The fp32-vs-fp64 spread of that step: rel-L2 and max |difference| / max |float64| of every loss value and every leaf
  gradient, from the same float32 inputs widened to float64.

The card's name, power limit and maximum SM clock are read in the same run and printed with every line.

    python tools/loss_f64_bench.py [--shapes C2,C3] [--iters 30] [--warmup 5] [--step-shapes C2]   (an empty list skips)
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import numpy as np
import torch

from umr_b200 import ops, synth
from umr_b200 import soft_renderer as sr
from umr_b200.nnutils import geom_utils, loss_utils

SHAPES = {"C2": dict(B=16, H=8, IS=256, subdiv=3, T=6), "C3": dict(B=32, H=8, IS=512, subdiv=3, T=6)}
DEV = "cuda:0"


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit and clocks unknown"


def op_cases(c):
    """name -> (fn(dtype) -> closure running forward + backward once)."""
    B, H, IS, T = c["B"], c["H"], c["IS"], c["T"]
    rng = np.random.default_rng(0)
    v, f = synth.icosphere(c["subdiv"])
    F = f.shape[0]
    cpu = dict(imgs=synth.smooth_images(rng, B, IS), flow=synth.texture_flow(rng, B, F, T),
               rgba=rng.uniform(0, 1, size=(B * H, 4, IS, IS)).astype(np.float32),
               masks=(rng.uniform(0, 1, size=(B * H, IS, IS)) > 0.5).astype(np.float32),
               prob=rng.uniform(-1, 1, size=(B, F, 2)).astype(np.float32),
               verts=synth.bird_like(v, rng, B), cams=synth.cameras(rng, B * H))
    vis = torch.from_numpy(rng.integers(0, 2, size=(B, F)).astype(np.uint8)).to(DEV)
    faces = torch.from_numpy(f.astype(np.int64))
    lap, flat = sr.LaplacianLoss(torch.from_numpy(v), faces).to(DEV), sr.FlattenLoss(faces).to(DEV)
    parts = [torch.from_numpy(p) for p in synth.part_vertex_sets(rng, v.shape[0], sizes=(20, 40, 20, 40))]
    corr = loss_utils.CorrLossChamfer(None, IS, part_vertices=parts)
    pts_np = synth.part_points(rng, B * H)

    def make(name, dtype):
        t = {k: torch.from_numpy(np.asarray(a)).to(DEV, dtype) for k, a in cpu.items()}
        pts = [torch.from_numpy(p).to(DEV, dtype) for p in pts_np]
        leaf = lambda x: x.requires_grad_(True)   # noqa: E731
        if name == "sampler":
            flow, imgs = leaf(t["flow"]), leaf(t["imgs"])
            return lambda: geom_utils.sample_textures(flow, imgs).sum().backward()
        if name == "iou":
            x = leaf(t["rgba"])
            return lambda: loss_utils.neg_iou_loss(x[:, 3], t["masks"]).backward()
        if name == "masked_l1":
            x = leaf(t["rgba"])
            return lambda: loss_utils.texture_loss_masks(x[:, :3], x[:, :3].detach(), t["masks"], x[:, 3]).backward()
        if name == "loss_head":
            x = leaf(t["rgba"])
            return lambda: ops.mask_texture_loss(x, x[:, :3].detach(), t["masks"])[0].backward()
        if name == "texcycle":
            flow = leaf(t["flow"])
            return lambda: loss_utils.TexCycle()(flow, t["prob"], None, visible=vis)[0].backward()
        if name == "laplacian":
            x = leaf(t["verts"])
            return lambda: lap(x).sum().backward()
        if name == "flatten":
            x = leaf(t["verts"])
            return lambda: flat(x).sum().backward()
        if name == "corr":
            x, cams = leaf(t["verts"][:1].clone()), leaf(t["cams"])
            return lambda: corr(pts[0], pts[1], pts[2], pts[3], x.expand(B * H, -1, -1), cams)[0].backward()
        raise KeyError(name)
    return ["sampler", "iou", "masked_l1", "loss_head", "texcycle", "laplacian", "flatten", "corr"], make


def time_alternating(fns, iters, warmup):
    """Median ms per call of each closure, calls interleaved so that both see the same machine state."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(warmup):
        for fn in fns:
            fn()
    torch.cuda.synchronize()
    ms = [[] for _ in fns]
    for _ in range(iters):
        for k, fn in enumerate(fns):
            ev[0].record()
            fn()
            ev[1].record()
            ev[1].synchronize()
            ms[k].append(ev[0].elapsed_time(ev[1]))
    return [float(np.median(m)) for m in ms], [float(np.min(m)) for m in ms], [float(np.max(m)) for m in ms]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="C2,C3")
    ap.add_argument("--step-shapes", default="C2")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("loss_f64_bench needs a GPU: there is nothing to time without one")
    gpu = card()
    for shape in filter(None, args.shapes.split(",")):
        names, make = op_cases(SHAPES[shape])
        for name in names:
            f64, f32 = make(name, torch.float64), make(name, torch.float32)
            med, lo, hi = time_alternating([f64, f32], args.iters, args.warmup)
            print(json.dumps({"kind": "op_fwd_bwd", "shape": shape, "op": name, "f64_median_ms": round(med[0], 4),
                              "f32_median_ms": round(med[1], 4), "ratio": round(med[0] / med[1], 2),
                              "f64_min_max_ms": [round(lo[0], 4), round(hi[0], 4)],
                              "f32_min_max_ms": [round(lo[1], 4), round(hi[1], 4)], "calls": args.iters, "gpu": gpu}),
                  flush=True)
        torch.cuda.empty_cache()
    from test_loss_f64_gpu import make_step
    names = ["total", "mask", "laplacian", "flatten", "tex_l1", "tex_dt", "tex_cycle", "part", "corr",
             "d/dmean_shape", "d/ddelta", "d/dcams", "d/dcam_logits", "d/dtex_flow"]
    for shape in filter(None, args.step_shapes.split(",")):
        c = SHAPES[shape]
        s64, l64 = make_step(c["B"], c["H"], c["IS"], c["subdiv"], c["T"], 0, torch.float64)
        s32, l32 = make_step(c["B"], c["H"], c["IS"], c["subdiv"], c["T"], 0, torch.float32)
        med, lo, hi = time_alternating([lambda: s64(*l64), lambda: s32(*l32)], max(args.iters // 3, 5), 2)
        print(json.dumps({"kind": "train_step", "shape": shape, "f64_median_ms": round(med[0], 3),
                          "f32_median_ms": round(med[1], 3), "ratio": round(med[0] / med[1], 2), "gpu": gpu}), flush=True)
        o64, o32 = s64(*l64), s32(*l32)
        torch.cuda.synchronize()
        for name, a, b in zip(names, o64, o32):
            a, b = a.detach().double().cpu(), b.detach().double().cpu()
            d = (a - b).abs()
            print(json.dumps({"kind": "fp32_vs_fp64", "shape": shape, "output": name,
                              "rel_l2": float(d.norm() / (a.norm() + 1e-300)),
                              "max_abs_over_max_f64": float(d.max() / (a.abs().max() + 1e-300)), "gpu": gpu}), flush=True)
        del s64, l64, s32, l32
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
