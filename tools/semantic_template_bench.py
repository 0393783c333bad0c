"""Time the SCOPS semantic template (umr_b200.utils.semantic_template) against the reference's GPU torch composition
(experiments/avg_uv.py:203-293), restated here, on the same seeded inputs: B = 32 images of 256 x 256 x 5 SCOPS
probabilities per batch, a 128 x 256 UV image, and the icosphere(3) template (V = 642, F = 1280, num_sym_faces = 624,
T = 6).

Averaging, per batch: the reference arm is `grid_sample` (align_corners=True), the MSE to the exemplar, `topk` and the
sum of the k = 5 nearest maps; the kernel arm is one `UVPartAverage.add`.  Each is timed with CUDA events around --batches
back-to-back batches, median of --reps windows, after a warm-up.  Labelling: the reference arm is `grid_sample` at the
uv_sampler, the per-face `most_freq` and the per-vertex loop (`nonzero`, `most_freq` and `if label > 0` per vertex); the
kernel arm is one `semantic_template` call.  Both synchronise with the host, so each is timed with the host clock around
a call that ends in a device synchronise, median of --reps.  The two arms' outputs are compared (labels exactly, averages
within float32 tolerance) and the card's name and power limit are printed with the numbers.

    python tools/semantic_template_bench.py [--batches 20] [--reps 7]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import semantic_template_oracle as sto  # noqa: E402
from umr_b200 import synth  # noqa: E402
from umr_b200.utils import semantic_template as st  # noqa: E402

B, C, S, H, W, K, T, NUM_SYM = 32, 5, 256, 128, 256, 5, 6, 624


def most_freq(arr):
    """avg_uv.py:119-131."""
    n, d = arr.size()
    k = torch.max(torch.unique(arr)) + 1
    one_hot = torch.zeros(n * d, k, device=arr.device)
    one_hot.scatter_(1, arr.view(-1, 1), 1)
    return torch.argmax(torch.sum(one_hot.view(n, d, k), dim=1), dim=1)


def ref_add(acc, segs, uv, best_uv):
    """avg_uv.py:213-225 for one batch; returns the new accumulator."""
    parts = torch.nn.functional.grid_sample(segs, uv.permute(0, 2, 3, 1), align_corners=True)
    dist = torch.sum(torch.nn.MSELoss(reduction="none")(parts, best_uv.expand_as(parts)), dim=(1, 2, 3))
    _, idx = torch.topk(dist, k=K, largest=False)
    s = torch.sum(parts[idx], dim=0)
    return s if acc is None else acc + s


def ref_label(avg_prob, uv_sampler, faces):
    """avg_uv.py:255-293 from avg_prob [H,W,C]: (label image, vertex labels, part lists)."""
    uv_label = avg_prob.permute(2, 0, 1).unsqueeze(0)
    tex = torch.nn.functional.grid_sample(uv_label, uv_sampler, align_corners=True)
    tex = tex.view(tex.size(0), -1, tex.size(2), T, T).permute(0, 2, 3, 4, 1)
    tex = torch.cat([tex, tex[:, -NUM_SYM:]], 1)
    tex = torch.argmax(tex.view(tex.size(0), tex.size(1), -1, C), dim=-1)
    face_labels = most_freq(tex.squeeze()).float()
    parts, vert = [[] for _ in range(C - 1)], []
    for v in range(int(faces.max()) + 1):
        hit = (faces[:, 0] == v) * 1 + (faces[:, 1] == v) * 1 + (faces[:, 2] == v) * 1
        idx = torch.nonzero(hit).squeeze()
        label = most_freq(face_labels[idx].long().view(1, idx.size(0)))
        if label > 0:
            parts[label - 1].append(v)
        vert.append(int(label))
    return torch.argmax(avg_prob, dim=2).to(torch.uint8), vert, parts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "semantic_template_bench needs a GPU"
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    batches = [(torch.from_numpy(sto.part_segs(rng, B, C, S)).to(dev), torch.from_numpy(sto.uvimage_pred(rng, B, H, W)).to(dev))
               for _ in range(args.batches)]
    best_uv = torch.nn.functional.grid_sample(batches[0][0][:1], batches[0][1][:1].permute(0, 2, 3, 1),
                                              align_corners=True)[0]
    verts, f = synth.icosphere(3)
    faces = torch.from_numpy(f.astype(np.int64)).to(dev)
    uv_sampler = torch.from_numpy(sto.uv_sampler(verts, f[:f.shape[0] - NUM_SYM], T)).to(dev)[None]
    res = dict(batch=B, channels=C, size=S, uv=[H, W], k=K, batches=args.batches, faces=int(f.shape[0]),
               vertices=int(verts.shape[0]), tex_size=T)

    def ref_average():
        acc = None
        for segs, uv in batches:
            acc = ref_add(acc, segs, uv, best_uv[None])
        return (acc / (K * len(batches))).permute(1, 2, 0).contiguous()

    def kernel_average():
        avg = st.UVPartAverage(best_uv, K)
        for segs, uv in batches:
            avg.add(segs, uv)
        return avg.mean()

    def events(fn):
        fn()
        torch.cuda.synchronize()
        out = []
        for _ in range(args.reps):
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            fn()
            stop.record()
            torch.cuda.synchronize()
            out.append(start.elapsed_time(stop) / args.batches)
        return out

    def host(fn):
        fn()
        torch.cuda.synchronize()
        out = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            out.append(1e3 * (time.perf_counter() - t0))
        return out

    for name, fn in (("reference_average_ms_per_batch", ref_average), ("kernel_average_ms_per_batch", kernel_average)):
        t = events(fn)
        res[name], res[name + "_spread"] = float(np.median(t)), [float(min(t)), float(max(t))]
    ref_avg, ker_avg = ref_average(), kernel_average()
    res["average_max_abs_diff"] = float((ref_avg - ker_avg).abs().max())

    for name, fn in (("reference_labels_ms", lambda: ref_label(ker_avg, uv_sampler, faces)),
                     ("kernel_labels_ms", lambda: st.semantic_template(ker_avg, uv_sampler, faces, NUM_SYM))):
        t = host(fn)
        res[name], res[name + "_spread"] = float(np.median(t)), [float(min(t)), float(max(t))]
    img, vert, parts = ref_label(ker_avg, uv_sampler, faces)
    tpl = st.semantic_template(ker_avg, uv_sampler, faces, NUM_SYM)
    res["labels_equal"] = bool(torch.equal(img, tpl.label_image) and vert == tpl.vertex_labels.tolist()
                               and all(p == q.tolist() for p, q in zip(parts, tpl.part_vertices)))
    res["label_image_equal_on_reference_average"] = bool(torch.equal(torch.argmax(ref_avg, dim=2).to(torch.uint8),
                                                                     tpl.label_image))
    res["part_sizes"] = [len(p) for p in parts]
    try:
        res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                    capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        res["gpu"] = torch.cuda.get_device_name(dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
