"""Three-way check on the H100 (SURVEY.md §8c "Gate 2" and the "kernel to beat"):
  ours  vs  the reference's own soft_rasterize CUDA extension rebuilt for sm_90a
            (oracle/_ref/soft_rasterize_ref.so, default nvcc flags = FMA contraction on)
        vs  the same sources built with -fmad=false (soft_rasterize_ref_nofma.so)
and a timing of the reference kernels against ours on the same inputs (CUDA events).
The reference modules are built by oracle/build_ref_gpu.py (from __graft_entry__.build()) where the reference
checkout exists; the reference sources are not needed at run time.  Test infrastructure, not product.
"""
import importlib.util
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.nn.functional as F

from umr_b200 import raster, synth


def load(name):
    path = os.path.join(ROOT, "oracle", "_ref", name + ".so")
    if not os.path.exists(path):
        return None
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _mode_args(sigma_val, dist, dist_eps, gamma_val, rgb, alpha, texture, double_side):
    # (image_size precedes) near, far, eps, sigma, func_id_dist, dist_eps (log form, soft_rasterize.py:35), gamma,
    # func_id_rgb, func_id_alpha, texture_sample_type, double_side
    return (1.0, 100.0, 1e-3, sigma_val, dist, float(np.log(1.0 / dist_eps - 1.0)), gamma_val, rgb, alpha, texture,
            bool(double_side))


def ref_forward(mod, fv, tex, S, rgb, sigma_val=1e-5, dist=2, dist_eps=1e-10, gamma_val=1e-4, alpha=2, texture=0,
                double_side=True):
    """functional/soft_rasterize.py:41-73 restated with device-side allocations.  Mode ids as in raster.FUNC_*; the
    defaults are UMR's configuration."""
    B, Fn = fv.shape[:2]
    dev = fv.device
    faces_info = torch.zeros(B, Fn, 27, device=dev)
    aggrs = torch.zeros(B, 2, S, S, device=dev)
    p2f = torch.zeros(B, Fn, 2, device=dev)
    p2f_sum = torch.zeros(B, Fn, 2, device=dev)
    colors = torch.ones(B, 4, S, S, device=dev)
    colors[:, :3] = 0.0
    theta = torch.tensor([[1, 0, 0], [0, 1, 0]], dtype=torch.float)
    grid = F.affine_grid(theta.unsqueeze(0), (1, 1, S, S), align_corners=True).view(S, S, 2).to(dev).contiguous()
    mod.forward_soft_rasterize(fv, tex, faces_info, aggrs, grid, p2f, p2f_sum, colors, S,
                               *_mode_args(sigma_val, dist, dist_eps, gamma_val, rgb, alpha, texture, double_side))
    return colors, p2f / p2f_sum.clamp_min(1e-12), aggrs, faces_info


def ref_backward(mod, fv, tex, colors, faces_info, aggrs, g, S, rgb, sigma_val=1e-5, dist=2, dist_eps=1e-10,
                 gamma_val=1e-4, alpha=2, texture=0, double_side=True):
    gf = torch.zeros_like(fv)
    gt = torch.zeros_like(tex)
    mod.backward_soft_rasterize(fv, tex, colors, faces_info, aggrs, gf, gt, g.contiguous(), S,
                                *_mode_args(sigma_val, dist, dist_eps, gamma_val, rgb, alpha, texture, double_side))
    return gf, gt


def stats(a, b):
    a, b = a.double(), b.double()
    d = (a - b).abs()
    bad = d > (1e-6 + 1e-4 * torch.maximum(a.abs(), b.abs()))
    return {"max_abs": float(d.max()), "rel_l2": float(d.norm() / (b.norm() + 1e-30)), "frac_beyond_1e-4": float(bad.double().mean()),
            "bit_exact": bool(torch.equal(a, b))}


def scene(B, tex_res, seed=0, subdiv=3):
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(subdiv)
    fv = synth.raster_space_faces(synth.bird_like(v, rng, B), f, synth.cameras(rng, B))
    tex = rng.uniform(0, 1, size=(B, f.shape[0], tex_res ** 2, 3)).astype(np.float32)
    return torch.from_numpy(fv).cuda(), torch.from_numpy(tex).cuda()


def main():
    out = {}
    mods = {"ref_fma": load("soft_rasterize_ref"), "ref_nofma": load("soft_rasterize_ref_nofma")}
    if not any(mods.values()):
        print(json.dumps({"unavailable": "oracle/_ref/soft_rasterize_ref*.so not built"}))
        return
    IS, S = 256, 512
    kw = dict(sigma_val=1e-5, dist_eps=1e-10, gamma_val=1e-4, anti_aliasing=True)
    # ---------------- parity ----------------
    for tex_res in (1, 6):
        for rgb_name, rgb in (("softmax", 1), ("hard", 0)):
            fv, tex = scene(2, tex_res, seed=3)
            a = fv.clone().requires_grad_(True)
            t = tex.clone().requires_grad_(True)
            img, p2f, aggr = raster.soft_rasterize(a, t, IS, aggr_func_rgb=rgb_name, **kw)
            g = torch.randn(img.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
            img.backward(g)
            for name, mod in mods.items():
                if mod is None:
                    continue
                colors, rp2f, raggr, finfo = ref_forward(mod, fv, tex, S, rgb)
                rimg = F.avg_pool2d(colors, 2, 2)
                ghi = (g / 4).repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
                rgf, rgt = ref_backward(mod, fv, tex, colors, finfo, raggr, ghi, S, rgb)
                key = "%s_T%d_%s" % (rgb_name, tex_res * tex_res, name)
                out[key] = {"images": stats(img.detach(), rimg), "aggrs": stats(aggr, raggr), "p2f": stats(p2f, rp2f),
                            "grad_faces": stats(a.grad, rgf)}
                if rgb == 0:
                    out[key]["face_id_plane_mismatches"] = int((aggr[:, 1] != raggr[:, 1]).sum())
                if tex_res == 1:
                    out[key]["grad_tex"] = stats(t.grad, rgt)
    # ---------------- timing (C2: B=16, T2=36, softmax) ----------------
    fv, tex = scene(16, 6, seed=0)
    g = torch.randn(16, 4, IS, IS, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]

    def time_ours():
        a = fv.clone().requires_grad_(True)
        t = tex.clone().requires_grad_(True)
        ev[0].record()
        img, _, _ = raster.soft_rasterize(a, t, IS, **kw)
        ev[1].record()
        img.backward(g)
        ev[2].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])

    def time_ref(mod):
        ev[0].record()
        colors, _, aggr, finfo = ref_forward(mod, fv, tex, S, 1)
        img = F.avg_pool2d(colors, 2, 2)
        ev[1].record()
        ghi = (g / 4).repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
        ref_backward(mod, fv, tex, colors, finfo, aggr, ghi, S, 1)
        ev[2].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])

    for _ in range(3):
        time_ours()
    ours = np.array([time_ours() for _ in range(10)]).mean(0)
    out["timing_ms_C2_B16"] = {"ours": {"fwd": float(ours[0]), "bwd": float(ours[1])}}
    if mods["ref_fma"] is not None:
        time_ref(mods["ref_fma"])
        ref = np.array([time_ref(mods["ref_fma"]) for _ in range(3)]).mean(0)
        out["timing_ms_C2_B16"]["reference_cuda_sm90a"] = {"fwd": float(ref[0]), "bwd": float(ref[1])}
        out["timing_ms_C2_B16"]["speedup_fwd_bwd"] = float(ref.sum() / ours.sum())
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
