"""Time the batch crop (umr_b200.utils.image.crop_batch) against the host path it replaces, in one run: B = 32 CUB-shaped
images (500 x 375 RGB sources, ~310 px square boxes, some past the border), S = 256, 5 SCOPS part channels.

Three arms:
- gpu: one `crop_batch` call with the part maps (table copy, two kernels), CUDA events around --calls back-to-back calls
  after a warm-up, median of --reps windows;
- h2d: the pinned host-to-device copy of the packed batch (pack and table), CUDA events, median of --reps;
- host: the reference's per-image host work for one batch -- `crop` in float64 with background padding, `cv2.resize` of
  image and mask, the coin-flip mirror, the float64 collate and float32 cast, and `set_input`'s per-image Normalize loop
  -- on one thread of this machine's CPU, host clock, median of --reps batches.  Without cv2 it prints "not measured".
The loader's new host half (box, window slice, points, collate) is timed as `loader_host_ms_per_batch`.  The card's name
and power limit are read in the same run and printed with the numbers.

    python tools/crop_bench.py [--batch 32] [--size 256] [--reps 7] [--calls 50]
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
from umr_b200.utils import crop_loader as cl  # noqa: E402
from umr_b200.utils import image  # noqa: E402

KP_PERM = np.array([1, 2, 3, 4, 5, 6, 11, 12, 13, 10, 7, 8, 9, 14, 15]) - 1
MEAN, STD = torch.tensor([0.485, 0.456, 0.406])[:, None, None], torch.tensor([0.229, 0.224, 0.225])[:, None, None]


def sources(rng, B):
    """CUB-shaped inputs: RGB 375 x 500 uint8 images, 0/1 ellipse masks, tight boxes of 250-300 px (1-indexed)."""
    items = []
    yy, xx = np.mgrid[:375, :500]
    for b in range(B):
        img = rng.integers(0, 256, (375, 500, 3), dtype=np.uint8)
        cx, cy = rng.uniform(150, 350), rng.uniform(120, 255)
        w, h = rng.uniform(250, 300), rng.uniform(200, 280)
        mask = (((xx - cx) / (w / 2)) ** 2 + ((yy - cy) / (h / 2)) ** 2 < 1).astype(np.uint8)
        items.append((img, mask, np.array([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2])))
    return items


def host_path(items, S, cv2):
    """The reference's pixel work for one batch on the host (utils/image.py crop / resize_img, data/base.py mirror,
    default_collate, set_input's float cast and Normalize loop)."""
    imgs, masks = [], []
    for img, mask, box in items:
        box = cl.square_bbox(cl.peturb_bbox(box - 1, 0.05, 0.05))
        b = [int(round(c)) for c in box]
        L = b[2] - b[0] + 1
        xs, xe, ys, ye = max(0, b[0]), min(500, b[2] + 1), max(0, b[1]), min(375, b[3] + 1)
        out = []
        for src, bg in ((img / 255.0, 1.0), (mask[:, :, None], 0.0)):
            frame = np.ones((L, L, src.shape[2])) * bg
            frame[ys - b[1]:ye - b[1], xs - b[0]:xe - b[0], :] = src[ys:ye, xs:xe, :]
            out.append(cv2.resize(frame, (S, S)))
        im, mk = out
        if np.random.rand(1) > 0.5:
            im, mk = im[:, ::-1, :].copy(), mk[:, ::-1].copy()
        imgs.append(np.transpose(im, (2, 0, 1)))
        masks.append(mk)
    img_t = torch.from_numpy(np.stack(imgs)).type(torch.FloatTensor)
    input_t = img_t.clone()
    for b in range(input_t.size(0)):
        input_t[b] = (input_t[b] - MEAN) / STD
    return input_t, torch.from_numpy(np.stack(masks)).type(torch.FloatTensor)


def loader_host(items, S):
    """The new loader half for one batch: box, window slice, flip, points, collate."""
    sfm = [np.float64(100.0), np.array([10.0, 5.0]), np.array([1.0, 0.0, 0.0, 0.0])]
    kp = np.ones((15, 3))
    batch = []
    for img, mask, box in items:
        win, kpn, _, _ = cl.crop_item(img, mask, box, kp, [np.copy(s) for s in sfm], S, 0.05, 0.05, True, KP_PERM)
        batch.append({"crop": win, "kp": kpn})
    return cl.collate(batch)


def events_ms(fn, calls, reps):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(calls):
            fn()
        stop.record()
        torch.cuda.synchronize()
        out.append(start.elapsed_time(stop) / calls)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "crop_bench needs a GPU"
    B, S = args.batch, args.size
    rng = np.random.default_rng(0)
    np.random.seed(0)
    items = sources(rng, B)
    res = dict(batch=B, size=S, part_channels=5)

    t = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        batch = loader_host(items, S)
        t.append(time.perf_counter() - t0)
    res["loader_host_ms_per_batch"] = 1e3 * float(np.median(t))
    res["pack_bytes"] = int(batch["crop_pack"].numel())
    res["mean_frame_side"] = float(batch["crop_table"][:, 6].float().mean())

    try:
        import cv2
    except ImportError:
        cv2 = None
    if cv2 is None:
        res["host_path_ms_per_batch"] = "not measured"
    else:
        cv2.setNumThreads(1)
        torch_threads = torch.get_num_threads()
        torch.set_num_threads(1)
        host_path(items[:2], S, cv2)
        t = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            host_path(items, S, cv2)
            t.append(time.perf_counter() - t0)
        torch.set_num_threads(torch_threads)
        res["host_path_ms_per_batch"] = 1e3 * float(np.median(t))
        res["host_path_threads"] = 1

    dev = torch.device("cuda:0")
    pack_h, table_h = batch["crop_pack"].pin_memory(), batch["crop_table"].pin_memory()
    pack_d = torch.empty_like(pack_h, device=dev)
    table_d = torch.empty_like(table_h, device=dev)

    def h2d():
        pack_d.copy_(pack_h, non_blocking=True)
        table_d.copy_(table_h, non_blocking=True)
    h = events_ms(h2d, args.calls, args.reps)
    res["h2d_pinned_ms_per_batch"] = float(np.median(h))

    part = torch.rand(B, S, S, 5, device=dev)
    g = events_ms(lambda: image.crop_batch(pack_d, table_h, S, part), args.calls, args.reps)
    res["gpu_ms_per_batch"] = float(np.median(g))
    res["gpu_ms_spread"] = [float(min(g)), float(max(g))]
    try:
        res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                    capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        res["gpu"] = torch.cuda.get_device_name(dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
