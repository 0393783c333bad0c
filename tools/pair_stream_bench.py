"""Raster forward / backward times and the pair-record traffic between them, at C2 (or any shape given).

    python tools/pair_stream_bench.py [--iters 200] [--warmup 20] [--B 16] [--is 256] [--subdiv 3] [--R 6]
    UMR_B200_LIB=/path/to/other/libumr_b200.so python tools/pair_stream_bench.py   # time another build

Prints ONE JSON line:
  fwd_kernel_ms / bwd_kernel_ms   median CUDA-event time of the main raster kernel(s) of the call, recorded by the C ABI
                                  around the launch (UmrRasterParams.ev_kernel_*, as bench.py's roofline does)
  fwd_call_ms / bwd_call_ms       median CUDA-event time of the whole autograd call (k_prep, memsets, fallback included)
  pairs                           surviving (pixel, face) pairs of one step: the survivor counts of the block headers
  record_mb_written / _read       pairs x record bytes: what the forward stores and the backward streams back per step
  header_words                    the pair buffer's first word: block headers the render wanted (segment heads included)
  blocks, block_mb                32-slot record blocks among them and their footprint (32 slots + a 4-byte header)
The record size follows the library's ABI version (203: 32-byte records, earlier: 48), so the parent build of a change
to the record can be measured by the same script.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from umr_b200 import _lib, raster, synth

UMR = dict(sigma_val=1e-5, dist_eps=1e-10, gamma_val=1e-4, eps=1e-3, near=1, far=100, fill_back=True,
           aggr_func_rgb="softmax", anti_aliasing=True)


def align256(x):
    return (x + 255) & ~255


def record_stats(pairs, B, S):
    """(header words wanted, tiles unsaved, record blocks, surviving pairs) of the pair buffer after a forward (layout:
    raster_stream.cuh).  Blocks and pairs are None when a tile was left unsaved: its headers were never written."""
    wanted, unsaved = (int(x) for x in pairs[:8].view(torch.int32).cpu().tolist())
    if unsaved:
        return wanted, unsaved, None, None
    nt = B * ((S + 15) // 16) ** 2
    hdr_off = 256 + 2 * align256(nt * 4)
    hdr = pairs[hdr_off:hdr_off + 4 * wanted].view(torch.int32).cpu().numpy().view(np.uint32)
    # segments are reserved back to back: [#blocks, next, #blocks block headers (face | count << 16)]
    blocks, survivors, pos = 0, 0, 0
    while pos + 2 <= hdr.size:
        nb = int(hdr[pos])
        blocks += nb
        survivors += int((hdr[pos + 2:pos + 2 + nb] >> 16).sum())
        pos += nb + 2
    return wanted, unsaved, blocks, survivors


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=16)
    ap.add_argument("--is", dest="isz", type=int, default=256)
    ap.add_argument("--subdiv", type=int, default=3)
    ap.add_argument("--R", type=int, default=6)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("pair_stream_bench.py times the GPU kernels: no CUDA device")
    lib = _lib.load()
    version = int(lib.umr_version())
    rec_bytes = 32 if version >= 203 else 48
    blk_bytes = 32 * rec_bytes + 4
    rng = np.random.default_rng(0)
    v, f = synth.icosphere(a.subdiv)
    verts = synth.bird_like(v, rng, a.B)
    cams = synth.cameras(rng, a.B)
    fv = torch.from_numpy(synth.raster_space_faces(verts, f, cams)).cuda().requires_grad_(True)
    F, T2 = f.shape[0], a.R * a.R
    tex = torch.rand(1, F, T2, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(0)).requires_grad_(True)
    g = torch.randn(a.B, 4, a.isz, a.isz, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    S = 2 * a.isz

    def step():
        img, _, _ = raster.soft_rasterize(fv, tex, a.isz, **UMR)
        return img

    for _ in range(a.warmup):   # also lets the adaptive pair-buffer sizing settle, as in a training run
        step().backward(g)
    torch.cuda.synchronize()
    sink = []
    raster.set_profile_sink(sink)
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(a.iters)]
    for e in ev:
        e[0].record()
        img = step()
        e[1].record()
        img.backward(g)
        e[2].record()
    torch.cuda.synchronize()
    raster.set_profile_sink(None)
    kern = raster.collect_profile(sink)
    img = step()
    pairs = img.grad_fn.saved_tensors[4]
    wanted, unsaved, blocks, survivors = record_stats(pairs, a.B, S)
    mb = lambda n, size: None if n is None else n * size / 1e6
    img.backward(g)
    torch.cuda.synchronize()
    med = lambda xs: float(np.median(xs))
    out = {
        "lib": _lib.LIB_PATH, "abi_version": version, "gpu": torch.cuda.get_device_name(),
        "shape": "B=%d is=%d (raster %d^2) F=%d T2=%d softmax" % (a.B, a.isz, S, F, T2), "iters": a.iters,
        "fwd_kernel_ms": med(kern["fwd"]), "bwd_kernel_ms": med(kern["bwd"]),
        "fwd_call_ms": med([e[0].elapsed_time(e[1]) for e in ev]), "bwd_call_ms": med([e[1].elapsed_time(e[2]) for e in ev]),
        "bwd_kernel_ms_min_max": [min(kern["bwd"]), max(kern["bwd"])],
        "pair_buffer_mb": pairs.numel() / 1e6, "tiles_unsaved": unsaved,
        "pairs": survivors, "record_bytes": rec_bytes,
        "record_mb_written": mb(survivors, rec_bytes), "record_mb_read": mb(survivors, rec_bytes),
        "header_words": wanted, "blocks": blocks, "block_mb": mb(blocks, blk_bytes),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
