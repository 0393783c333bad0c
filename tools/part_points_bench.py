"""Time the batched SCOPS part centres and part points (umr_b200.utils.image.part_points) against the reference's per-image
CPU composition (utils/image.py:168-206, called as data/base.py:155-166 calls it): B = 32 images of 256 x 256 x 5 SCOPS
probabilities, counts (10, 10, 30, 30) for channels 1-4, in one run.

The per-image arm is the loader's work for one batch: per image, `prob2center` and `sample_prob` for each of the four
channels (numpy masked centroid, torch float32 centroid sums, torch.multinomial without replacement, topk), run serially in
this process with torch's default CPU threads; timed with the host clock, median of --reps batches.  The batched arm is
one `part_points` call on the device (uniform draw, two kernels and the status read), timed with CUDA events around
--calls back-to-back calls, median of --reps windows, after a warm-up call.  The card's name and power limit are printed
with the numbers.

    python tools/part_points_bench.py [--batch 32] [--reps 7] [--calls 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from umr_b200.utils import image  # noqa: E402

CHANNELS, COUNTS = (1, 2, 3, 4), (10, 10, 30, 30)


def maps(rng, B, S, C=5):
    """SCOPS-like probabilities [B,S,S,C] float32 (softmax of smooth random logits) and soft ellipse masks [B,S,S] float64."""
    yy, xx = np.mgrid[0:S, 0:S] / S
    logits = np.zeros((B, S, S, C))
    for b in range(B):
        for c in range(C):
            for _ in range(3):
                (cx, cy), w = rng.uniform(0.2, 0.8, 2), rng.uniform(0.05, 0.2)
                logits[b, :, :, c] += 3 * np.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / (2 * w * w))
    e = np.exp(logits - logits.max(-1, keepdims=True))
    prob = (e / e.sum(-1, keepdims=True)).astype(np.float32)
    r = ((xx[None] - 0.5) / 0.35) ** 2 + ((yy[None] - 0.5) / 0.3) ** 2
    mask = np.clip((1.1 - np.repeat(r, B, 0)) * 4, 0, 1)
    return prob, mask


def per_image(prob, mask):
    """The reference's per-image calls: numpy centroid, then float32 torch sampling, per channel."""
    S = prob.shape[0]
    x_map = torch.from_numpy((np.tile(np.arange(S), (S, 1)) / S * 2 - 1.0).astype(np.float32))
    y_map = torch.from_numpy((np.tile(np.arange(S), (S, 1)).T / S * 2 - 1.0).astype(np.float32))
    out = []
    for ch, n in zip(CHANNELS, COUNTS):
        q = prob[:, :, ch] * mask
        pdf = torch.from_numpy(q / float(q.sum())).float()
        center = torch.stack([(pdf * x_map).sum(), (pdf * y_map).sum()])
        p, m = torch.from_numpy(prob).float(), torch.from_numpy(mask).float()
        qs = p[:, :, ch] * m
        pdf = qs / float(qs.sum())
        samples = torch.multinomial(pdf.view(-1), num_samples=int(1.5 * n))
        coords = torch.stack([samples % S, samples // S], dim=1).float() / 256.0 * 2 - 1
        dist = torch.sum((coords - center) * (coords - center), dim=1)
        _, top = torch.topk(dist, k=n, largest=False)
        out.append((center, coords[top]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "part_points_bench needs a GPU"
    rng = np.random.default_rng(0)
    prob, mask = maps(rng, args.batch, args.size)
    res = dict(batch=args.batch, size=args.size, counts=COUNTS, torch_threads=torch.get_num_threads())

    per_image(prob[0], mask[0])
    cpu = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        for b in range(args.batch):
            per_image(prob[b], mask[b])
        cpu.append(time.perf_counter() - t0)
    res["per_image_cpu_ms_per_batch"] = 1e3 * float(np.median(cpu))

    dev = torch.device("cuda:0")
    p = torch.from_numpy(prob).to(dev)
    m = torch.from_numpy(mask).to(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    image.part_points(p, m, COUNTS, CHANNELS, generator=g)
    torch.cuda.synchronize()
    gpu = []
    for _ in range(args.reps):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(args.calls):
            image.part_points(p, m, COUNTS, CHANNELS, generator=g)
        stop.record()
        torch.cuda.synchronize()
        gpu.append(start.elapsed_time(stop) / args.calls)
    res["batched_gpu_ms_per_batch"] = float(np.median(gpu))
    res["batched_gpu_ms_spread"] = [float(min(gpu)), float(max(gpu))]
    res["speedup"] = res["per_image_cpu_ms_per_batch"] / res["batched_gpu_ms_per_batch"]
    try:
        res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                    capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        res["gpu"] = torch.cuda.get_device_name(dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
