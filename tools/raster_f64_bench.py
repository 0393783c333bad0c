"""Timing of the float64 rasteriser (DESIGN.md §9), CUDA events, one JSON line per shape.

At the C2 (B = 16, 1280 faces, 256^2 anti-aliased, T2 = 36) and C3 (B = 32, 512^2) shapes of bench.py, softmax, UMR's
sigma / gamma: forward and backward of `soft_rasterize` in float64 and, alternating call by call in the same process, in
float32 on the same (widened) inputs; and the reference's CUDA kernels run in double from oracle/_ref (-fmad=false build)
where they were built (fewer calls: they take seconds at C3).  The card's name, power limit and maximum SM clock are read
in the same run and printed with every line.

    python tools/raster_f64_bench.py [--shapes C2,C3] [--iters 50] [--warmup 10] [--ref-iters 3]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch
import torch.nn.functional as F

import ref_gpu_compare as rc
from umr_b200 import raster, synth

SHAPES = {"C2": dict(batch=16, image_size=256, subdiv=3, tex_res=6), "C3": dict(batch=32, image_size=512, subdiv=3, tex_res=6)}
UMR = dict(sigma_val=1e-5, dist_eps=1e-10, gamma_val=1e-4)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit and clocks unknown"


def stats(ms):
    a = np.asarray(ms)
    return {"median_ms": round(float(np.median(a)), 4), "min_ms": round(float(a.min()), 4), "max_ms": round(float(a.max()), 4),
            "calls": int(a.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="C2,C3")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--ref-iters", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("raster_f64_bench needs a GPU: there is nothing to time without one")
    dev = "cuda:0"
    ref = rc.load("soft_rasterize_ref_nofma")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    for name in args.shapes.split(","):
        c = SHAPES[name]
        rng = np.random.default_rng(0)
        v, f = synth.icosphere(c["subdiv"])
        B, isz = c["batch"], c["image_size"]
        fv32 = torch.from_numpy(synth.raster_space_faces(synth.bird_like(v, rng, B), f, synth.cameras(rng, B))).to(dev)
        tex32 = torch.from_numpy(rng.uniform(0, 1, size=(B, f.shape[0], c["tex_res"] ** 2, 3)).astype(np.float32)).to(dev)
        g32 = torch.randn(B, 4, isz, isz, device=dev)
        inputs = {torch.float32: (fv32, tex32, g32), torch.float64: (fv32.double(), tex32.double(), g32.double())}

        def ours(dt):
            fv, tex, g = inputs[dt]
            a, t = fv.clone().requires_grad_(True), tex.clone().requires_grad_(True)
            ev[0].record()
            img, _, _ = raster.soft_rasterize(a, t, isz, anti_aliasing=True, **UMR)
            ev[1].record()
            img.backward(g)
            ev[2].record()
            torch.cuda.synchronize()
            return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])

        def reference():
            fv, tex, g = inputs[torch.float64]
            S = 2 * isz
            z = lambda *s: torch.zeros(*s, device=dev, dtype=torch.float64)  # noqa: E731
            ev[0].record()
            info, aggrs, p2f, p2f_sum = z(B, fv.shape[1], 27), z(B, 2, S, S), z(B, fv.shape[1], 2), z(B, fv.shape[1], 2)
            colors = torch.ones(B, 4, S, S, device=dev, dtype=torch.float64)
            colors[:, :3] = 0.0
            theta = torch.tensor([[1, 0, 0], [0, 1, 0]], dtype=torch.float)
            grid = F.affine_grid(theta.unsqueeze(0), (1, 1, S, S), align_corners=True).view(S, S, 2).double().to(dev).contiguous()
            modes = (1.0, 100.0, 1e-3, UMR["sigma_val"], 2, float(np.log(1.0 / UMR["dist_eps"] - 1.0)), UMR["gamma_val"], 1, 2, 0, True)
            ref.forward_soft_rasterize(fv, tex, info, aggrs, grid, p2f, p2f_sum, colors, S, *modes)
            F.avg_pool2d(colors, 2, 2)
            ev[1].record()
            ghi = (g / 4).repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
            gf, gt = torch.zeros_like(fv), torch.zeros_like(tex)
            ref.backward_soft_rasterize(fv, tex, colors, info, aggrs, gf, gt, ghi.contiguous(), S, *modes)
            ev[2].record()
            torch.cuda.synchronize()
            # a backward that left no gradient did not launch (the double instantiation can exceed the launch's registers)
            return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]) if float(gf.abs().max()) > 0 else float("nan")

        for _ in range(args.warmup):
            ours(torch.float64)
            ours(torch.float32)
        t = {torch.float32: [], torch.float64: []}
        for _ in range(args.iters):   # alternating, so both see the same clocks and neighbours
            for dt in (torch.float64, torch.float32):
                t[dt].append(ours(dt))
        out = {"shape": name, "batch": B, "image_size": isz, "faces": int(f.shape[0]), "texture_size": c["tex_res"] ** 2,
               "card": card()}
        for dt, key in ((torch.float64, "float64"), (torch.float32, "float32")):
            a = np.asarray(t[dt])
            out[key] = {"forward": stats(a[:, 0]), "backward": stats(a[:, 1])}
        out["float64_over_float32"] = {k: round(out["float64"][k]["median_ms"] / out["float32"][k]["median_ms"], 2)
                                       for k in ("forward", "backward")}
        if ref is not None and args.ref_iters > 0:
            reference()
            a = np.asarray([reference() for _ in range(args.ref_iters)])
            out["reference_double_kernels"] = {"forward": stats(a[:, 0])}
            out["reference_over_float64"] = {"forward": round(out["reference_double_kernels"]["forward"]["median_ms"] /
                                                              out["float64"]["forward"]["median_ms"], 1)}
            if np.isnan(a[:, 1]).any():
                out["reference_double_kernels"]["backward"] = "not measured (the kernel does not launch in double)"
            else:
                out["reference_double_kernels"]["backward"] = stats(a[:, 1])
                out["reference_over_float64"]["backward"] = round(out["reference_double_kernels"]["backward"]["median_ms"] /
                                                                  out["float64"]["backward"]["median_ms"], 1)
        else:
            out["reference_double_kernels"] = "not measured (oracle/_ref/soft_rasterize_ref_nofma.so not built)"
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
