"""Time the geometry gradient of the functional NMR rasteriser (umr_nmr_backward_faces, DESIGN.md §14) at the shape of
UMR's training visuals: batch 16, 256^2 with anti-aliasing, 1280 faces, T = 6.  `rasterize_rgbad` forward, then the
backward of rgb + alpha + depth (geometry and texture gradients), each timed with CUDA events per call; medians over
the timed calls after warm-up.  Prints one JSON line with the card's name, power limit and max SM clock.

    python tools/nmr_grad_bench.py [--iters 50] [--warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from umr_b200 import synth  # noqa: E402
from umr_b200 import neural_renderer as nr  # noqa: E402
from umr_b200.nnutils import geom_utils  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable: %s" % q.stderr.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--image-size", type=int, default=256)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("nmr_grad_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    B, IS, T = a.batch, a.image_size, 6
    rng = np.random.default_rng(0)
    v, f = synth.icosphere(3)
    verts = torch.from_numpy(synth.bird_like(v, rng, B)).to(dev)
    cams = torch.from_numpy(synth.cameras(rng, B)).to(dev)
    faces = torch.from_numpy(f)[None].repeat(B, 1, 1).to(dev)
    vs = geom_utils.orthographic_proj_withz(verts, cams, offset_z=5.)
    vs[:, :, 1] *= -1
    vs[:, :, 2] += 2.732          # the look_at translation of UMR's eye (0, 0, -2.732)
    fv0 = nr.vertices_to_faces(vs, faces).detach()
    tex = torch.rand(B, f.shape[0], T, T, 3, device=dev).unsqueeze(4).repeat(1, 1, 1, 1, T, 1).requires_grad_(True)
    g = [torch.rand(B, 3, IS, IS, device=dev) - 0.5, torch.rand(B, IS, IS, device=dev) - 0.5,
         torch.rand(B, IS, IS, device=dev) - 0.5]

    def step(times=None):
        fv = fv0.clone().requires_grad_(True)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        out = nr.rasterize_rgbad(fv, tex, IS, True)
        ev[1].record()
        torch.autograd.backward([out["rgb"], out["alpha"], out["depth"]], g)
        ev[2].record()
        torch.cuda.synchronize()
        if times is not None:
            times[0].append(ev[0].elapsed_time(ev[1]))
            times[1].append(ev[1].elapsed_time(ev[2]))

    for _ in range(a.warmup):
        step()
    times = ([], [])
    for _ in range(a.iters):
        step(times)
    print(json.dumps({"workload": "nmr rasterize_rgbad B=%d is=%d F=%d T=%d aa, rgb+alpha+depth adjoints"
                                  % (B, IS, f.shape[0], T),
                      "forward_ms_median": round(float(np.median(times[0])), 4),
                      "backward_ms_median": round(float(np.median(times[1])), 4),
                      "backward_ms_min_max": [round(min(times[1]), 4), round(max(times[1]), 4)],
                      "iters": a.iters, "card": card(), "torch": torch.__version__}))


if __name__ == "__main__":
    main()
