"""Timing of the one-render mask + texture step (MultiMaskTextureLoss, DESIGN.md §11) against the two modules it replaces
(MultiMaskLoss, then MultiTextureLoss on the detached geometry, as experiments/train_s2.py calls them), forward +
backward to every leaf, CUDA events, one JSON line per (shape, mode).

* Shapes of bench.py: C2 (16 images x 8 camera hypotheses, 256^2, 1280 faces, T^2 = 36) and C3 (32 x 8, 512^2).
* Modes: default (float atomics) and deterministic (torch.use_deterministic_algorithms(True)).
* Both variants alternate call by call in the same process; the median of each of two runs is printed, with min / max.
* The card's name, power limit and maximum SM clock are read in the same run and printed with every line.

    python tools/split_render_bench.py [--shapes C2,C3] [--modes default,deterministic] [--iters 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from umr_b200 import synth
from umr_b200.nnutils import loss_utils

SHAPES = {"C2": dict(B=16, H=8, IS=256, subdiv=3, T=6), "C3": dict(B=32, H=8, IS=512, subdiv=3, T=6)}
DEV = "cuda:0"
LEAVES = ("vs", "cams", "probs", "tx", "flow")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit and clocks unknown"


def inputs(c, seed=0):
    B, H, IS, T = c["B"], c["H"], c["IS"], c["T"]
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(c["subdiv"])
    F = f.shape[0]
    d = dict(vs=synth.bird_like(v, rng, B), cams=np.stack([synth.cameras(rng, H) for _ in range(B)]),
             probs=rng.dirichlet(np.ones(H), size=B).astype(np.float32), masks=synth.ellipse_masks(rng, B, IS),
             imgs=synth.smooth_images(rng, B, IS), flow=synth.texture_flow(rng, B, F, T),
             tx=rng.uniform(0, 1, size=(B, F, T * T, 3)).astype(np.float32))
    d["dts"] = np.stack([synth.dt_barrier(m) for m in d["masks"]])[:, None]
    t = {k: torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for k, a in d.items()}
    t["fs"] = torch.from_numpy(f.astype(np.int64)).to(DEV)[None].repeat(B, 1, 1)
    t["proj_cam"] = t["cams"][:, 0].clone()
    for k in LEAVES:
        t[k].requires_grad_(True)
    return t


def step_fn(c, t, fused):
    """A closure: one forward + backward of the mask and texture losses to every leaf."""
    B, H, IS = c["B"], c["H"], c["IS"]
    leaves = [t[k] for k in LEAVES]
    if fused:
        m = loss_utils.MultiMaskTextureLoss(B, H, IS, "softmax", texture_loss_type="l1")

        def run():
            out = m(t["vs"], t["fs"], t["cams"], t["probs"], t["proj_cam"], t["imgs"], t["masks"], t["tx"], t["flow"], t["dts"])
            total = out[0] + out[2] + out[3] + out[4]
            return torch.autograd.grad(total, leaves)
        return run
    mm = loss_utils.MultiMaskLoss(IS, "softmax", H)
    mt = loss_utils.MultiTextureLoss(B, H, IS, "softmax", texture_loss_type="l1")

    def run():
        mask_loss, mask_all = mm(t["vs"], t["fs"], t["cams"], t["probs"], t["masks"])
        tex_loss, dt_loss, cyc_loss, _ = mt(t["vs"].detach(), t["fs"], t["cams"].detach(), t["probs"].detach(), t["proj_cam"],
                                            t["imgs"], t["masks"], mask_all, t["tx"], t["flow"], t["dts"])
        return torch.autograd.grad(mask_loss + tex_loss + dt_loss + cyc_loss, leaves)
    return run


def time_alternating(fns, iters, warmup):
    """Median / min / max ms per call of each closure, calls interleaved so that both see the same machine state."""
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
    return [(float(np.median(m)), float(np.min(m)), float(np.max(m))) for m in ms]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="C2,C3")
    ap.add_argument("--modes", default="default,deterministic")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("split_render_bench needs a GPU: there is nothing to time without one")
    gpu = card()
    for shape in filter(None, args.shapes.split(",")):
        c = SHAPES[shape]
        t = inputs(c)
        for mode in filter(None, args.modes.split(",")):
            torch.use_deterministic_algorithms(mode == "deterministic")
            try:
                composed, fused = step_fn(c, t, False), step_fn(c, t, True)
                runs = [time_alternating([composed, fused], args.iters, args.warmup) for _ in range(2)]
            finally:
                torch.use_deterministic_algorithms(False)
            med_c = [r[0][0] for r in runs]
            med_f = [r[1][0] for r in runs]
            print(json.dumps({"kind": "mask_texture_step_fwd_bwd", "shape": shape, "mode": mode,
                              "composed_median_ms": [round(x, 3) for x in med_c],
                              "split_median_ms": [round(x, 3) for x in med_f],
                              "composed_min_max_ms": [round(min(r[0][1] for r in runs), 3), round(max(r[0][2] for r in runs), 3)],
                              "split_min_max_ms": [round(min(r[1][1] for r in runs), 3), round(max(r[1][2] for r in runs), 3)],
                              "saved_ms": [round(a - b, 3) for a, b in zip(med_c, med_f)],
                              "speedup": [round(a / b, 3) for a, b in zip(med_c, med_f)],
                              "calls_per_run": args.iters, "gpu": gpu}), flush=True)
            torch.cuda.empty_cache()
        del t
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
