"""Forward and backward time of the soft rasteriser on large meshes (UMR configuration, softmax, anti-aliased), CUDA
events around the autograd calls, median of --iters after --warmup:

  * F = 65535 and F = 65536 on the same mesh and image: the last 16-bit-index workload and the first 32-bit one (the
    65536th face is a copy of face 0 moved behind the far plane, so both render the same picture);
  * a 327680-face icosphere(7) at 256^2 and 1024^2 output, against the reference's CUDA kernels (oracle/_ref, FMA build)
    on the same inputs when they were built.

Prints one JSON line per workload with the card's name and power limit."""
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

from umr_b200 import raster, synth
import ref_gpu_compare as rc  # noqa: E402

DEV = "cuda:0"
UMR = dict(sigma_val=1e-5, dist_eps=1e-10, gamma_val=1e-4)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().split("\n")[0]
    except Exception:
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def ours(fv, tex, isz, g, iters, warmup):
    tfv = torch.from_numpy(fv).to(DEV).requires_grad_(True)
    ttex = torch.from_numpy(tex).to(DEV).requires_grad_(True)
    state = {}

    def fwd():
        state["img"] = raster.soft_rasterize(tfv, ttex, isz, anti_aliasing=True, **UMR)[0]

    def bwd():
        torch.autograd.grad(state["img"], (tfv, ttex), g, retain_graph=True)

    t_f = timed(fwd, iters, warmup)
    fwd()
    t_b = timed(bwd, iters, warmup)
    return t_f, t_b


def reference(mod, fv, tex, isz, g, iters, warmup):
    S = 2 * isz
    tfv, ttex = torch.from_numpy(fv).to(DEV), torch.from_numpy(tex).to(DEV)
    ghi = (g / 4).repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
    out = {}

    def fwd():
        out["f"] = rc.ref_forward(mod, tfv, ttex, S, 1)

    def bwd():
        colors, _, aggrs, finfo = out["f"]
        rc.ref_backward(mod, tfv, ttex, colors, finfo, aggrs, ghi, S, 1)

    t_f = timed(fwd, iters, warmup)
    fwd()
    t_b = timed(bwd, iters, warmup)
    return t_f, t_b


def mesh(subdiv, B, seed=0):
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(subdiv)
    fv = synth.raster_space_faces(synth.bird_like(v, rng, B), f, synth.cameras(rng, B))
    tex = rng.uniform(0, 1, size=(B, f.shape[0], 4, 3)).astype(np.float32)
    return fv, tex


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4)
    args = ap.parse_args()
    gpu = card()
    B = args.batch
    # the selection pair: 65535 faces of icosphere(7), and the same plus one face behind the far plane
    fv7, tex7 = mesh(7, B)
    base_fv, base_tex = fv7[:, :65535], tex7[:, :65535]
    extra = base_fv[:, :1].copy()
    extra[..., 2::3] = 500.0
    pair = {65535: (np.ascontiguousarray(base_fv), np.ascontiguousarray(base_tex)),
            65536: (np.ascontiguousarray(np.concatenate([base_fv, extra], 1)),
                    np.ascontiguousarray(np.concatenate([base_tex, base_tex[:, :1]], 1)))}
    isz = 256
    g = torch.randn(B, 4, isz, isz, device=DEV)
    for F, (fv, tex) in pair.items():
        t_f, t_b = ours(fv, tex, isz, g, args.iters, args.warmup)
        print(json.dumps(dict(workload="selection pair", faces=F, batch=B, image_size=isz, fwd_ms=t_f, bwd_ms=t_b,
                              path="16-bit" if F <= 65535 else "32-bit", gpu=gpu)), flush=True)
    # one image: the reference walks all faces for every pixel (1.4e12 face visits per forward at 1024^2 output)
    mod = rc.load("soft_rasterize_ref")
    fv7, tex7 = np.ascontiguousarray(fv7[:1]), np.ascontiguousarray(tex7[:1])
    for isz in (256, 1024):
        g = torch.randn(1, 4, isz, isz, device=DEV)
        t_f, t_b = ours(fv7, tex7, isz, g, args.iters, args.warmup)
        row = dict(workload="icosphere(7)", faces=fv7.shape[1], batch=1, image_size=isz, fwd_ms=t_f, bwd_ms=t_b, gpu=gpu)
        if mod is not None:
            r_f, r_b = reference(mod, fv7, tex7, isz, g, 3, 1)
            row.update(ref_fwd_ms=r_f, ref_bwd_ms=r_b)
        else:
            row.update(ref="oracle/_ref/soft_rasterize_ref.so not built")
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
