"""Timing of part_matching_loss forward + backward to vertices and cameras with its head on the part-head kernels
(DESIGN.md §13) against the same module with the head as the torch composition (`loss_utils.part_head_torch`), CUDA
events, one JSON line per (shape, mode).  Both routes share the one 4-channel part render; the difference is the head.

* Shapes: B = 16 at 256^2 (train_s2's) and B = 32 at 512^2, an icosphere of 1280 faces, 6 x 6 texels per face.
* Modes: default and deterministic (torch.use_deterministic_algorithms(True)).
* Both routes alternate call by call in the same process; the median of each of two runs is printed, with min / max.
* The card's name, power limit and maximum SM clock are read in the same run and printed with every line.

    python tools/part_head_bench.py [--shapes S256,S512] [--modes default,deterministic] [--iters 20] [--warmup 5]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch

from split_render_bench import card, time_alternating
from umr_b200 import synth
from umr_b200.nnutils import loss_utils

DEV = "cuda:0"
SHAPES = {"S256": dict(B=16, IS=256, subdiv=3, T=6), "S512": dict(B=32, IS=512, subdiv=3, T=6)}


def inputs(c, seed=0):
    B, IS, T = c["B"], c["IS"], c["T"]
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(c["subdiv"])
    part = rng.integers(0, 5, size=(f.shape[0], T * T))
    one_hot = torch.zeros(1, f.shape[0], T * T, 5)
    one_hot.scatter_(3, torch.from_numpy(part)[None, :, :, None], 1.0)
    t = dict(one_hot=one_hot,
             vs=torch.from_numpy(synth.bird_like(v, rng, B)).to(DEV).requires_grad_(True),
             fs=torch.from_numpy(f.astype(np.int64)).to(DEV)[None].repeat(B, 1, 1),
             cams=torch.from_numpy(synth.cameras(rng, B)).to(DEV).requires_grad_(True),
             segs=torch.softmax(torch.from_numpy(rng.normal(size=(B, 5, IS, IS)).astype(np.float32)), 1).to(DEV))
    return t


def step_fn(c, t, kernels):
    """A closure: part_matching_loss forward + backward to vertices and cameras."""
    m = loss_utils.part_matching_loss(None, None, 0, im_size=c["IS"], batch_size=c["B"], tex_size=c["T"],
                                      stex_one_hot=t["one_hot"]).to(DEV)
    on_device = loss_utils.part_head_on_device

    def run():
        if not kernels:
            loss_utils.part_head_on_device = lambda *a: False
        try:
            loss, _ = m(t["vs"], t["fs"], t["cams"], t["segs"])
        finally:
            loss_utils.part_head_on_device = on_device
        return torch.autograd.grad(loss, (t["vs"], t["cams"]))
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="S256,S512")
    ap.add_argument("--modes", default="default,deterministic")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("part_head_bench needs a GPU: there is nothing to time without one")
    gpu = card()
    for shape in filter(None, args.shapes.split(",")):
        c = SHAPES[shape]
        t = inputs(c)
        for mode in filter(None, args.modes.split(",")):
            torch.use_deterministic_algorithms(mode == "deterministic")
            try:
                torch_head, kernel_head = step_fn(c, t, False), step_fn(c, t, True)
                runs = [time_alternating([torch_head, kernel_head], args.iters, args.warmup) for _ in range(2)]
            finally:
                torch.use_deterministic_algorithms(False)
            med_t = [r[0][0] for r in runs]
            med_k = [r[1][0] for r in runs]
            print(json.dumps({"kind": "part_matching_loss_fwd_bwd", "shape": shape, "B": c["B"], "size": c["IS"],
                              "mode": mode,
                              "torch_head_median_ms": [round(x, 3) for x in med_t],
                              "kernel_head_median_ms": [round(x, 3) for x in med_k],
                              "torch_head_min_max_ms": [round(min(r[0][1] for r in runs), 3), round(max(r[0][2] for r in runs), 3)],
                              "kernel_head_min_max_ms": [round(min(r[1][1] for r in runs), 3), round(max(r[1][2] for r in runs), 3)],
                              "saved_ms": [round(a - b, 3) for a, b in zip(med_t, med_k)],
                              "speedup": [round(a / b, 3) for a, b in zip(med_t, med_k)],
                              "calls_per_run": args.iters, "gpu": gpu}), flush=True)
            torch.cuda.empty_cache()
        del t
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
