"""Time the NMR renderer (csrc/nmr.cu) at the shape of UMR's training visuals (train_s2.py:322-324: batch 16, 256^2,
1280 faces, T = 6 texture cube): `Renderer.render_rgb` forward and its texture backward, with CUDA events after
warm-up.  Prints one JSON line with the card's name and power limit read in the same run.

    python tools/nmr_bench.py [--iters 50] [--warmup 10]
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
from umr_b200.neural_renderer import Renderer  # noqa: E402
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
        sys.exit("nmr_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    B, IS, T = a.batch, a.image_size, 6
    rng = np.random.default_rng(0)
    v, f = synth.icosphere(3)
    verts = torch.from_numpy(synth.bird_like(v, rng, B)).to(dev)
    cams = torch.from_numpy(synth.cameras(rng, B)).to(dev)
    faces = torch.from_numpy(f)[None].repeat(B, 1, 1).to(dev)
    vs = geom_utils.orthographic_proj_withz(verts, cams, offset_z=5.)
    vs[:, :, 1] *= -1
    tex = torch.rand(B, f.shape[0], T, T, 3, device=dev).unsqueeze(4).repeat(1, 1, 1, 1, T, 1).requires_grad_(True)
    r = Renderer(image_size=IS, anti_aliasing=True, camera_mode="look_at", perspective=False)
    r.eye = [0, 0, -2.732]
    r.light_intensity_ambient, r.light_intensity_directional, r.light_direction = 0.8, 0.4, [0, 1, -1]
    grad = torch.rand(B, 3, IS, IS, device=dev)

    def fwd():
        return r.render_rgb(vs, faces, tex)

    for _ in range(a.warmup):
        fwd().backward(grad)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    t_f = t_b = 0.0
    for _ in range(a.iters):
        ev[0].record()
        img = fwd()
        ev[1].record()
        img.backward(grad)
        ev[2].record()
        torch.cuda.synchronize()
        t_f += ev[0].elapsed_time(ev[1])
        t_b += ev[1].elapsed_time(ev[2])
    print(json.dumps({"workload": "nmr render_rgb B=%d is=%d F=%d T=%d fill_back" % (B, IS, f.shape[0], T),
                      "forward_ms": round(t_f / a.iters, 4), "texture_backward_ms": round(t_b / a.iters, 4),
                      "iters": a.iters, "card": card(), "torch": torch.__version__}))


if __name__ == "__main__":
    main()
