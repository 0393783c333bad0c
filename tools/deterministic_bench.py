"""Cost of the rasteriser's deterministic mode: forward and backward call times (CUDA events, after warm-up), default vs
deterministic, at the C2 / C3 / C5 raster shapes of BASELINE.md, and a bitwise check of repeated deterministic calls.

    python tools/deterministic_bench.py [--shapes C2,C3,C5] [--iters 10] [--out FILE.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from umr_b200 import raster, synth  # noqa: E402

SHAPES = {"C2": (16, 3, 256), "C3": (32, 3, 512), "C5": (8, 4, 1024)}   # B, icosphere subdivision, output size (2x AA)
# C5_bigface: C5 plus one near-plane triangle covering the whole raster in every image (the deterministic backward walks it
# on one warp per image)
UMR = dict(sigma_val=1e-5, dist_eps=1e-10, gamma_val=1e-4, anti_aliasing=True)


def inputs(B, subdiv, seed=0, big_face=False):
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(subdiv)
    verts = synth.bird_like(v, rng, B)
    cams = synth.cameras(rng, B)
    fv = synth.raster_space_faces(verts, f, cams)
    tex = rng.uniform(0, 1, size=(B, f.shape[0], 36, 3)).astype(np.float32)
    if big_face:
        big = np.array([-3, -3, 6.0, 3, -3, 6.0, 0, 3, 6.0], np.float32)
        fv = np.concatenate([fv, np.broadcast_to(big, (B, 1, 9))], axis=1)
        tex = np.concatenate([tex, np.full((B, 1, 36, 3), 0.5, np.float32)], axis=1)
    return torch.from_numpy(np.ascontiguousarray(fv, np.float32)).cuda(), torch.from_numpy(tex).cuda()


def one(fv, tex, isz, g):
    a = fv.clone().requires_grad_(True)
    t = tex.clone().requires_grad_(True)
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    e0.record()
    img, p2f, aggr = raster.soft_rasterize(a, t, isz, **UMR)
    e1.record()
    img.backward(g)
    e2.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), e1.elapsed_time(e2), (img.detach(), p2f, aggr, a.grad, t.grad)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="C2,C3,C5")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("deterministic_bench needs a CUDA device")
    res = {"device": torch.cuda.get_device_name(0), "shapes": {}}
    for name in args.shapes.split(","):
        B, subdiv, isz = SHAPES[name.replace("_bigface", "")]
        fv, tex = inputs(B, subdiv, big_face=name.endswith("_bigface"))
        g = torch.linspace(-1, 1, B * 4 * isz * isz, device="cuda").view(B, 4, isz, isz)
        row = {}
        for mode in ("default", "deterministic"):
            torch.use_deterministic_algorithms(mode == "deterministic")
            for _ in range(3):
                one(fv, tex, isz, g)
            f_ms, b_ms, first = [], [], None
            equal = True
            for _ in range(args.iters):
                f, b, out = one(fv, tex, isz, g)
                f_ms.append(f)
                b_ms.append(b)
                if first is None:
                    first = out
                else:
                    equal &= all(torch.equal(x, y) for x, y in zip(first, out))
            row[mode] = {"fwd_ms": float(np.median(f_ms)), "bwd_ms": float(np.median(b_ms)), "bitwise_equal": bool(equal)}
        torch.use_deterministic_algorithms(False)
        d, r = row["default"], row["deterministic"]
        row["ratio_fwd"] = r["fwd_ms"] / d["fwd_ms"]
        row["ratio_bwd"] = r["bwd_ms"] / d["bwd_ms"]
        row["ratio_total"] = (r["fwd_ms"] + r["bwd_ms"]) / (d["fwd_ms"] + d["bwd_ms"])
        res["shapes"][name] = row
        print(name, json.dumps(row))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
