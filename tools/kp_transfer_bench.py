"""Time batched keypoint transfer (umr_b200.nnutils.kp_transfer) against the per-pair torch composition of
experiments/test_kp.py:125-193 on the same GPU: 1000 pairs x 15 keypoints, F = 1280 faces, T = 6, 256 x 256 images.

The per-pair path is the reference's: K heat maps drawn on the host per pair (kp_utils.draw_labelmap), copied to the
device, two grid_sample calls (here with align_corners=True, the convention the batched kernels use) and a copy back
(flow); nonzero and two chamfer searches per pair (cam).  Both are timed from first launch to a device synchronise with
CUDA events, median of --reps windows (200 back-to-back calls per window for the batched kernels, one pass over
all pairs for the per-pair path), after a warm-up call; the card's name and power limit are printed with the numbers.

    python tools/kp_transfer_bench.py [--pairs 1000] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as Fn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from umr_b200.nnutils import kp_transfer  # noqa: E402


def draw_labelmap(img, pt, sigma):
    """kp_utils.py:42-69 restated (numpy, on the host)."""
    ul = [int(pt[0] - 3 * sigma), int(pt[1] - 3 * sigma)]
    br = [int(pt[0] + 3 * sigma + 1), int(pt[1] + 3 * sigma + 1)]
    if ul[0] >= img.shape[1] or ul[1] >= img.shape[0] or br[0] < 0 or br[1] < 0:
        return img
    size = 6 * sigma + 1
    x = np.arange(0, size, 1, float)
    y = x[:, np.newaxis]
    g = np.exp(- ((x - size // 2) ** 2 + (y - size // 2) ** 2) / (2 * sigma ** 2))
    g_x = max(0, -ul[0]), min(br[0], img.shape[1]) - ul[0]
    g_y = max(0, -ul[1]), min(br[1], img.shape[0]) - ul[1]
    img_x = max(0, ul[0]), min(br[0], img.shape[1])
    img_y = max(0, ul[1]), min(br[1], img.shape[0])
    img[img_y[0]:img_y[1], img_x[0]:img_x[1]] = g[g_y[0]:g_y[1], g_x[0]:g_x[1]]
    return img


def per_pair_flow(kps, fs, ft, S, sigma, sgrid):
    out = []
    for p in range(kps.shape[0]):
        nf = ft.shape[1]
        p2face = Fn.grid_sample(sgrid, ft[p].view(1, nf, -1, 2), align_corners=True)
        p2face = torch.mean(p2face, dim=-1).permute(0, 2, 1).cpu().squeeze(0)
        K = kps.shape[1]
        hp = np.zeros((1, K, S, S), np.float32)
        pts = (kps[p] + 1) / 2.0 * 256
        for k in range(K):
            draw_labelmap(hp[0, k], (pts[k, 0], pts[k, 1]), sigma)
        k2face = Fn.grid_sample(torch.from_numpy(hp).cuda(), fs[p].view(1, nf, -1, 2), align_corners=True)
        idx = torch.mean(k2face, dim=-1).cpu().max(dim=-1)[1]
        out.append(p2face[idx[0]])
    return torch.stack(out)


def dist_chamfer(a, b):
    """nnutils/chamfer_python.py:43-64 restated: nearest indices both ways."""
    xx, yy, zz = torch.bmm(a, a.transpose(2, 1)), torch.bmm(b, b.transpose(2, 1)), torch.bmm(a, b.transpose(2, 1))
    ia = torch.arange(a.shape[1], device=a.device)
    ib = torch.arange(b.shape[1], device=b.device)
    rx = xx[:, ia, ia].unsqueeze(1).expand_as(zz.transpose(2, 1))
    ry = yy[:, ib, ib].unsqueeze(1).expand_as(zz)
    P = rx.transpose(2, 1) + ry - 2 * zz
    return P.min(2)[1], P.min(1)[1]


def per_pair_cam(kps, ps, pt, mask, sgrid):
    out = []
    for p in range(kps.shape[0]):
        fg_idx = torch.nonzero(mask[p].view(-1)).squeeze()
        fg = sgrid[fg_idx, :]
        _, proj2fg = dist_chamfer(fg.unsqueeze(0), pt[p:p + 1])
        kp2proj, _ = dist_chamfer(kps[p:p + 1], ps[p:p + 1])
        out.append(fg[proj2fg[0][kp2proj[0]]].cpu())
    return torch.stack(out)


def timed(fn, reps, calls=1):
    """(median ms per call over `reps` windows of `calls` back-to-back calls, the last result)"""
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(calls):
            r = fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b) / calls)
    return float(np.median(ms)), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    P, K, F, T, S, V, sigma = args.pairs, 15, 1280, 6, 256, 642, 3
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    centre = rng.uniform(-1, 1, (P, F, 1, 2))
    fs = torch.from_numpy((centre + rng.uniform(-0.04, 0.04, (P, F, T * T, 2))).astype(np.float32)).to(dev)
    ft = torch.from_numpy((rng.uniform(-1, 1, (P, F, 1, 2)) + rng.uniform(-0.04, 0.04, (P, F, T * T, 2))).astype(np.float32)).to(dev)
    kps = rng.uniform(-0.9, 0.9, (P, K, 2)).astype(np.float32)
    kd = torch.from_numpy(kps).to(dev)
    ps = torch.from_numpy(rng.uniform(-0.9, 0.9, (P, V, 2)).astype(np.float32)).to(dev)
    pt = torch.from_numpy(rng.uniform(-0.9, 0.9, (P, V, 2)).astype(np.float32)).to(dev)
    yy, xx = np.mgrid[0:S, 0:S] / (S - 1) * 2 - 1
    mask = torch.from_numpy(np.stack([((xx - c[0]) ** 2 + (yy - c[1]) ** 2 < 0.3).astype(np.float32)
                                      for c in rng.uniform(-0.3, 0.3, (P, 2))])).to(dev)
    lin = torch.linspace(-1, 1, S)
    sgrid_img = torch.stack([lin[None, :].expand(S, S), lin[:, None].expand(S, S)])[None].to(dev)    # [1,2,S,S]
    sgrid_flat = sgrid_img[0].permute(1, 2, 0).reshape(-1, 2)

    grid = kp_transfer._grid(S, dev)

    def cam_batched():
        from umr_b200 import _lib
        from umr_b200.raster import _ptr, _stream_ptr
        out = torch.empty(P, K, 2, device=dev)
        _lib.check(_lib.load().umr_kp_transfer_cam(_ptr(kd), _ptr(ps), _ptr(pt), _ptr(mask), _ptr(grid), _ptr(out), P, K, V,
                                                   S, _stream_ptr(dev)), "cam")
        return out

    res = {}
    # the batched calls take milliseconds: each timed window holds 200 of them (about half a second or more)
    res["flow_batched_ms"], fb = timed(lambda: kp_transfer.transfer_flow(kd, fs, ft, sigma, S), args.reps, 200)
    res["flow_per_pair_ms"], fp = timed(lambda: per_pair_flow(kps, fs, ft, S, sigma, sgrid_img), args.reps)
    res["cam_batched_ms"], cb = timed(cam_batched, args.reps, 200)
    res["cam_per_pair_ms"], cp = timed(lambda: per_pair_cam(kd, ps, pt, mask, sgrid_flat), args.reps)
    res["flow_speedup"] = res["flow_per_pair_ms"] / res["flow_batched_ms"]
    res["cam_speedup"] = res["cam_per_pair_ms"] / res["cam_batched_ms"]
    # agreement with the per-pair path: torch's grid_sample, mean and bmm round differently, so outputs agree to float32
    # rounding where both pick the same face / vertex / pixel, and differ only at near-ties
    for mode, a, b in (("flow", fb.cpu(), fp), ("cam", cb.cpu(), cp)):
        res[mode + "_agree_1e-5"] = float(((a - b).abs() <= 1e-5).all(-1).float().mean())
    res.update(pairs=P, keypoints=K, faces=F, T=T, image=S, vertices=V, sigma=sigma)
    try:
        res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                    capture_output=True, text=True).stdout.strip()
    except OSError:
        res["gpu"] = torch.cuda.get_device_name(dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
