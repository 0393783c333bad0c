"""Time neural_renderer's functional pipeline (DESIGN.md §15).

1. `lighting` forward + backward (faces, textures, [B,3] colours and direction all requiring grad) against the same
   formula composed from torch ops, at batch 16 with 1280 faces and T = 6, and with 5120 faces and T = 8.
2. The light-parameter gradient's cost at 65537 faces: forward + backward with and without colours and direction
   requiring grad (B = 16, T = 2).
3. One whole functional step at batch 16, 256^2 with anti-aliasing, 1280 faces, T = 6: get_points_from_angles,
   look_at, perspective, lighting, vertices_to_faces, rasterize_rgbad, then the backward of rgb + alpha into the
   vertices, the eye and the textures.
CUDA events around each call, medians over the timed calls after warm-up.  Prints one JSON line with the card's name,
power limit and max SM clock, read in the same run.

    python tools/nmr_pipeline_bench.py [--iters 50] [--warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as tF

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from umr_b200 import synth  # noqa: E402
from umr_b200 import neural_renderer as nr  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable: %s" % q.stderr.strip()


def torch_lighting(faces, textures, Ia, Id, ca, cd, d):
    """The light formula composed from torch ops, out of place."""
    B, F = faces.shape[:2]
    fv = faces.reshape(B * F, 3, 3)
    n = tF.normalize(torch.cross(fv[:, 0] - fv[:, 1], fv[:, 2] - fv[:, 1], dim=-1), eps=1e-5).reshape(B, F, 3)
    cos = tF.relu((n * d[:, None, :]).sum(2))
    light = Ia * ca[:, None, :] + Id * (cd[:, None, :] * cos[:, :, None])
    return textures * light[:, :, None, None, None, :]


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * iters)]
    for i in range(iters):
        ev[2 * i].record()
        fn()
        ev[2 * i + 1].record()
    torch.cuda.synchronize()
    return round(float(np.median([ev[2 * i].elapsed_time(ev[2 * i + 1]) for i in range(iters)])), 4)


def lighting_case(B, F, T, iters, warmup, dev):
    rng = np.random.default_rng(0)
    faces = torch.from_numpy(rng.uniform(-1, 1, (B, F, 3, 3)).astype(np.float32)).to(dev).requires_grad_(True)
    tex = torch.rand(B, F, T, T, T, 3, device=dev, requires_grad=True)
    ca, cd = (torch.rand(B, 3, device=dev, requires_grad=True) for _ in range(2))
    d = (torch.rand(B, 3, device=dev) + 0.2).requires_grad_(True)
    g = torch.rand(B, F, T, T, T, 3, device=dev) - 0.5
    params = (faces, tex, ca, cd, d)

    def run(fn):
        def step():
            out = fn(faces, tex, 0.5, 0.5, ca, cd, d)
            torch.autograd.grad(out, params, g)
        return step
    with torch.no_grad():
        err = float((nr.lighting(*params[:2], 0.5, 0.5, *params[2:]) -
                     torch_lighting(*params[:2], 0.5, 0.5, *params[2:])).abs().max())
    res = {}
    for _ in range(2):       # alternate the two, twice
        res.setdefault("kernel_ms", []).append(timed(run(nr.lighting), iters, warmup))
        res.setdefault("torch_ms", []).append(timed(run(torch_lighting), iters, warmup))
    return {"B": B, "F": F, "T": T, "fwd_bwd_kernel_ms": res["kernel_ms"], "fwd_bwd_torch_ms": res["torch_ms"],
            "max_abs_diff_fwd": err}


def reduce_case(B, F, T, iters, warmup, dev):
    """The cost of the light-parameter gradient (k_nmr_light_reduce: F dependent adds per sum, plus the [3] arguments'
    batch sums): `lighting` forward + backward with and without colours and direction requiring grad."""
    rng = np.random.default_rng(1)
    faces = torch.from_numpy(rng.uniform(-1, 1, (B, F, 3, 3)).astype(np.float32)).to(dev).requires_grad_(True)
    tex = torch.rand(B, F, T, T, T, 3, device=dev, requires_grad=True)
    g = torch.rand(B, F, T, T, T, 3, device=dev) - 0.5
    light = [torch.rand(B, 3, device=dev) + 0.2 for _ in range(3)]

    def run(with_light):
        args = [t.clone().requires_grad_(with_light) for t in light]
        wrt = (faces, tex, *args) if with_light else (faces, tex)

        def step():
            torch.autograd.grad(nr.lighting(faces, tex, 0.5, 0.5, *args), wrt, g)
        return step
    res = {"with_light_grad_ms": [], "without_ms": []}
    for _ in range(2):
        res["with_light_grad_ms"].append(timed(run(True), iters, warmup))
        res["without_ms"].append(timed(run(False), iters, warmup))
    return {"B": B, "F": F, "T": T, **res}


def step_case(iters, warmup, dev):
    B, IS, T = 16, 256, 6
    v, f = synth.icosphere(3)
    f = torch.from_numpy(f.astype(np.int32))[None].repeat(B, 1, 1).to(dev)
    verts = torch.from_numpy(v.astype(np.float32))[None].repeat(B, 1, 1).to(dev).requires_grad_(True)
    tex = torch.rand(B, f.shape[1], T, T, T, 3, device=dev, requires_grad=True)
    el = torch.full((B,), 20.0, device=dev)
    az = torch.linspace(0, 345, B, device=dev)
    dist = torch.full((B,), 3.0, device=dev, requires_grad=True)
    g = [torch.rand(B, 3, IS, IS, device=dev) - 0.5, torch.rand(B, IS, IS, device=dev) - 0.5]

    def step():
        eye = nr.get_points_from_angles(dist, el, az)
        lit = nr.lighting(nr.vertices_to_faces(verts, f), tex, 0.5, 0.5, direction=(0.3, 1.0, -0.5))
        cam = nr.perspective(nr.look_at(verts, eye), 30.0)
        out = nr.rasterize_rgbad(nr.vertices_to_faces(cam, f), lit, IS, True, return_depth=False)
        torch.autograd.grad([out["rgb"], out["alpha"]], [verts, tex, dist], g)
    return {"B": B, "is": IS, "F": int(f.shape[1]), "T": T, "step_ms": [timed(step, iters, warmup) for _ in range(2)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("nmr_pipeline_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    print(json.dumps({"lighting": [lighting_case(16, 1280, 6, a.iters, a.warmup, dev),
                                   lighting_case(16, 5120, 8, a.iters, a.warmup, dev)],
                      "light_parameter_gradient": reduce_case(16, 65537, 2, a.iters, a.warmup, dev),
                      "functional_step": step_case(a.iters, a.warmup, dev),
                      "iters": a.iters, "card": card(), "torch": torch.__version__}))


if __name__ == "__main__":
    main()
