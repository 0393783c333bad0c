"""Time `voxelization` on the GPU: ours (`umr_voxelize`, csrc/voxel.cu) and, where oracle/_ref holds it, the reference's
own extension driven by its own host loop (functional/voxelization.py:9-58, restated below with device allocations; its
fill syncs the host after every sweep through `visible.sum()`).

Shapes: B in {1, 16, 64} x icosphere subdivision 3 / 4 (1280 / 5120 faces) deformed by synth.bird_like x vs in
{32, 64, 128}: the sizes a 3D-IoU evaluation of predicted meshes voxelises at.  Per shape and implementation: CUDA-event
time per call (mean over --iters calls after --warmup) and host wall time per call (ending in a device synchronise),
plus the reference's sweep count.  Ours and the reference alternate per shape in the same process.  Prints one JSON
line per shape; --out writes them all to a file.

    python tools/voxel_bench.py [--iters 20] [--warmup 3] [--no-ref] [--out /tmp/voxel_bench.json]
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from umr_b200 import ops, synth  # noqa: E402


def load_ref(name="voxelization_ref"):
    """The reference extension built by oracle/build_ref_voxel.py, or None."""
    path = os.path.join(ROOT, "oracle", "_ref", name + ".so")
    if not os.path.exists(path):
        return None
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def ref_voxelization(mod, faces, size, normalize=False, stats=None):
    """functional/voxelization.py:9-58 on the reference extension `mod`; stats["sweeps"] counts voxelize_sub4 calls."""
    faces = faces.clone()
    if not normalize:
        faces *= size
    bs, dev = faces.size(0), faces.device

    def sub1(dim):
        f = faces
        if dim == 0:
            f = faces[:, :, :, [2, 1, 0]].contiguous()
        elif dim == 1:
            f = faces[:, :, :, [0, 2, 1]].contiguous()
        vox = torch.zeros(bs, size, size, size, dtype=torch.int32, device=dev)
        return mod.voxelize_sub1(f, vox)[0].transpose(dim + 1, -1)

    v0, v1, v2 = sub1(0), sub1(1), sub1(2)
    v3 = mod.voxelize_sub2(faces, torch.zeros(bs, size, size, size, dtype=torch.int32, device=dev))[0]
    # .contiguous(): current torch keeps the transposed layout of v0 through the sum (torch 1.1 returned a contiguous
    # tensor), and the extension requires contiguous voxels
    voxels = ((v0 + v1 + v2 + v3) > 0).int().contiguous()
    visible = torch.zeros_like(voxels, dtype=torch.int32)
    voxels, visible = mod.voxelize_sub3(faces, voxels, visible)
    sum_visible = visible.sum()
    sweeps = 0
    while True:
        voxels, visible = mod.voxelize_sub4(faces, voxels, visible)
        sweeps += 1
        if visible.sum() == sum_visible:
            break
        sum_visible = visible.sum()
    if stats is not None:
        stats["sweeps"] = sweeps
    return 1 - visible


def meshes(B, subdiv, seed=0):
    v, f = synth.icosphere(subdiv)
    verts = synth.bird_like(v, np.random.default_rng(seed), B) * 0.45 + 0.5  # inside the unit cube
    return torch.from_numpy(np.ascontiguousarray(verts[:, f])).float()


def time_calls(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / iters
    return e0.elapsed_time(e1) / iters, wall * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-ref", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("voxel_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    ref = None if a.no_ref else load_ref()
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        gpu = torch.cuda.get_device_name(dev)
    rows = []
    print(json.dumps({"gpu": gpu, "reference_extension": ref is not None}), flush=True)
    for B in (1, 16, 64):
        for subdiv in (3, 4):
            faces = meshes(B, subdiv).to(dev)
            for vs in (32, 64, 128):
                ours = lambda: ops.voxelize(faces, vs)  # noqa: E731
                row = {"B": B, "faces": int(faces.shape[1]), "vs": vs}
                row["ours_event_ms"], row["ours_wall_ms"] = time_calls(ours, a.iters, a.warmup)
                got = ours()
                row["ours_status"] = ops.voxelize_status(dev)
                if ref is not None:
                    st = {}
                    want = ref_voxelization(ref, faces, vs, stats=st)
                    row["ref_sweeps"] = st["sweeps"]
                    row["equal_to_ref_fma_build"] = bool(torch.equal(got, want))
                    row["ref_event_ms"], row["ref_wall_ms"] = time_calls(lambda: ref_voxelization(ref, faces, vs), a.iters,
                                                                         a.warmup)
                    # second leg of ours, alternating with the reference in the same session
                    row["ours_event_ms_2"], row["ours_wall_ms_2"] = time_calls(ours, a.iters, a.warmup)
                    row["speedup_wall"] = row["ref_wall_ms"] / min(row["ours_wall_ms"], row["ours_wall_ms_2"])
                rows.append(row)
                print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"gpu": gpu, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
