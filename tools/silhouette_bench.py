"""Timing of MultiMaskLoss through the silhouette render (DESIGN.md §12) against the same module through the full render
(taken while a pass-through wrapper sits on SoftRasterizeFunction.apply), forward + backward to every leaf, CUDA events,
one JSON line per (shape, mode).

* Shapes of bench.py: C2 (16 images x 8 camera hypotheses, 256^2, 1280 faces) and C3 (32 x 8, 512^2).
* Modes: default (float atomics) and deterministic (torch.use_deterministic_algorithms(True)).
* Both routes alternate call by call in the same process; the median of each of two runs is printed, with min / max.
* The card's name, power limit and maximum SM clock are read in the same run and printed with every line.

    python tools/silhouette_bench.py [--shapes C2,C3] [--modes default,deterministic] [--iters 20] [--warmup 5]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch

from split_render_bench import card, inputs, time_alternating
from umr_b200 import raster
from umr_b200.nnutils import loss_utils

SHAPES = {"C2": dict(B=16, H=8, IS=256, subdiv=3, T=6), "C3": dict(B=32, H=8, IS=512, subdiv=3, T=6)}
LEAVES = ("vs", "cams", "probs")


def step_fn(c, t, silhouette):
    """A closure: MultiMaskLoss forward + backward to vertices, cameras and camera probabilities."""
    m = loss_utils.MultiMaskLoss(c["IS"], "softmax", c["H"])
    leaves = [t[k] for k in LEAVES]
    orig = raster.SoftRasterizeFunction.apply

    def run():
        if not silhouette:   # a wrapper on apply: MultiMaskLoss takes the full render, through it
            raster.SoftRasterizeFunction.apply = staticmethod(lambda *a: orig(*a))
        try:
            loss, _ = m(t["vs"], t["fs"], t["cams"], t["probs"], t["masks"])
        finally:
            raster.SoftRasterizeFunction.apply = orig
        return torch.autograd.grad(loss, leaves)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="C2,C3")
    ap.add_argument("--modes", default="default,deterministic")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("silhouette_bench needs a GPU: there is nothing to time without one")
    gpu = card()
    for shape in filter(None, args.shapes.split(",")):
        c = SHAPES[shape]
        t = inputs(c)
        for mode in filter(None, args.modes.split(",")):
            torch.use_deterministic_algorithms(mode == "deterministic")
            try:
                full, sil = step_fn(c, t, False), step_fn(c, t, True)
                runs = [time_alternating([full, sil], args.iters, args.warmup) for _ in range(2)]
            finally:
                torch.use_deterministic_algorithms(False)
            med_f = [r[0][0] for r in runs]
            med_s = [r[1][0] for r in runs]
            print(json.dumps({"kind": "multi_mask_loss_fwd_bwd", "shape": shape, "mode": mode,
                              "full_render_median_ms": [round(x, 3) for x in med_f],
                              "silhouette_median_ms": [round(x, 3) for x in med_s],
                              "full_render_min_max_ms": [round(min(r[0][1] for r in runs), 3), round(max(r[0][2] for r in runs), 3)],
                              "silhouette_min_max_ms": [round(min(r[1][1] for r in runs), 3), round(max(r[1][2] for r in runs), 3)],
                              "saved_ms": [round(a - b, 3) for a, b in zip(med_f, med_s)],
                              "speedup": [round(a / b, 3) for a, b in zip(med_f, med_s)],
                              "calls_per_run": args.iters, "gpu": gpu}), flush=True)
            torch.cuda.empty_cache()
        del t
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
