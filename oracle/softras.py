"""CPU oracles for the soft rasteriser -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may import
this module; the product path (umr_b200/) never does.

Two implementations behind one numpy interface:
  impl="A"  the reference's own device code compiled for the host (oracle/ref_host_shim.cpp,
            built from the reference checkout into oracle/_ref/ by oracle/build_oracle.py);
  impl="B"  our independent restatement (oracle/softras_oracle.cpp).

The host glue below restates external/SoftRas/soft_renderer/functional/soft_rasterize.py:12-108
(buffer allocation/fill :47-55, the torch-1.1 `affine_grid` = align_corners=True grid :57-62,
dist_eps -> log(1/dist_eps - 1) :35, p2f normalisation :73) and rasterizer.py:42-55 (2x
supersampling + avg_pool2d).
"""
import ctypes
import os
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, _HERE)
import build_oracle  # noqa: E402

DIST = {"hard": 0, "barycentric": 1, "euclidean": 2}
RGB = {"hard": 0, "softmax": 1}
ALPHA = {"hard": 0, "sum": 1, "prod": 2}
TEX = {"surface": 0, "vertex": 1}

_libs = {}
_fp = ctypes.POINTER(ctypes.c_float)
_dp = ctypes.POINTER(ctypes.c_double)


def _lib(impl):
    if impl not in _libs:
        if impl == "A":
            path = build_oracle.build_a()
            if path is None:
                raise RuntimeError("oracle A unavailable: no reference checkout and no prebuilt oracle/_ref")
        else:
            path = build_oracle.build_b()
        _libs[impl] = ctypes.CDLL(path)
    return _libs[impl]


def have_oracle_a():
    try:
        _lib("A")
        return True
    except Exception:
        return False


def host_threads(cap=64):
    """Threads the oracle may use: the CPUs this process can actually run on -- the scheduler affinity mask, further
    limited by a cgroup CPU quota (cpu.max / cfs_quota) -- NOT os.cpu_count(), which on a shared GPU box reports
    every core of the machine and oversubscribes OpenMP (round-1 VERDICT: 3.4 vs 20 images/s on "128 cores")."""
    import math
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        with open("/sys/fs/cgroup/cpu.max") as fh:  # cgroup v2: "<quota> <period>" or "max <period>"
            q, per = fh.read().split()[:2]
            if q != "max":
                n = min(n, max(1, int(math.ceil(int(q) / float(per)))))
    except Exception:
        try:
            with open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us") as fq, open("/sys/fs/cgroup/cpu/cpu.cfs_period_us") as fp:
                q, per = int(fq.read()), int(fp.read())
                if q > 0:
                    n = min(n, max(1, int(math.ceil(q / float(per)))))
        except Exception:
            pass
    return max(1, min(n, cap))


def max_threads():
    return host_threads()


def _nt(nthreads):
    return host_threads() if nthreads <= 0 else nthreads


def _p(a):
    return a.ctypes.data_as(_fp if a.dtype == np.float32 else _dp)


def standard_grid(image_size, dtype=np.float32):
    """`affine_grid(identity, (1,1,S,S))` of torch 1.1 (== align_corners=True): [S,S,2] (x,y).  At S = 1 torch 1.1 takes
    linspace(-1, 1, 1) = [-1], so the one pixel is (-1, -1); torch >= 1.3 returns 0 there instead."""
    if int(image_size) == 1:
        return np.full((1, 1, 2), -1.0, dtype)
    import torch
    theta = torch.tensor([[1, 0, 0], [0, 1, 0]], dtype=torch.float)
    g = torch.nn.functional.affine_grid(theta.unsqueeze(0), (1, 1, image_size, image_size),
                                        align_corners=True)
    return np.ascontiguousarray(g.view(image_size, image_size, 2).numpy().astype(dtype))


class RasterCfg:
    """Scalar arguments of `soft_rasterize` with the defaults UMR uses (nnutils/smr.py:53-56)."""

    def __init__(self, image_size, background_color=(0, 0, 0), near=1.0, far=100.0, fill_back=True,
                 eps=1e-3, sigma_val=1e-5, dist_func="euclidean", dist_eps=1e-10, gamma_val=1e-4,
                 aggr_func_rgb="softmax", aggr_func_alpha="prod", texture_type="surface"):
        self.image_size = int(image_size)
        self.background_color = tuple(float(c) for c in background_color)
        self.near, self.far, self.eps = float(near), float(far), float(eps)
        self.sigma_val, self.gamma_val = float(sigma_val), float(gamma_val)
        self.dist = DIST[dist_func]
        self.dist_eps_log = float(np.log(1.0 / dist_eps - 1.0))  # soft_rasterize.py:35
        self.rgb, self.alpha, self.tex = RGB[aggr_func_rgb], ALPHA[aggr_func_alpha], TEX[texture_type]
        self.fill_back = bool(fill_back)

    def scalars(self):
        return (ctypes.c_float(self.near), ctypes.c_float(self.far), ctypes.c_float(self.eps),
                ctypes.c_float(self.sigma_val), ctypes.c_int(self.dist),
                ctypes.c_float(self.dist_eps_log), ctypes.c_float(self.gamma_val),
                ctypes.c_int(self.rgb), ctypes.c_int(self.alpha), ctypes.c_int(self.tex),
                ctypes.c_int(1 if self.fill_back else 0))


def forward(face_vertices, textures, cfg, impl="B", nthreads=0, dtype=np.float32):
    """soft_rasterize forward. face_vertices [B,F,9|3,3], textures [B,F,T2,3].
    Returns dict(soft_colors[B,4,S,S], p2f_info[B,F,2], aggrs_info[B,2,S,S], faces_info, p2f_raw, p2f_sum)."""
    fv = np.ascontiguousarray(np.asarray(face_vertices, dtype=dtype).reshape(face_vertices.shape[0], -1, 9))
    tex = np.ascontiguousarray(np.asarray(textures, dtype=dtype))
    B, F = fv.shape[:2]
    T2 = tex.shape[2]
    S = cfg.image_size
    faces_info = np.zeros((B, F, 27), dtype)
    aggrs = np.zeros((B, 2, S, S), dtype)
    p2f = np.zeros((B, F, 2), dtype)
    p2f_sum = np.zeros((B, F, 2), dtype)
    colors = np.ones((B, 4, S, S), dtype)
    for k in range(3):
        colors[:, k] *= dtype(cfg.background_color[k])
    grid = standard_grid(S, dtype)
    lib = _lib(impl)
    sfx = "f32" if dtype == np.float32 else "f64"
    fn = getattr(lib, ("ref_" if impl == "A" else "oracle_") + "forward_soft_rasterize_" + sfx)
    fn(_p(fv), _p(tex), _p(faces_info), _p(aggrs), _p(grid), _p(p2f), _p(p2f_sum), _p(colors),
       B, F, S, T2, *cfg.scalars(), ctypes.c_int(_nt(nthreads)))
    p2f_info = p2f / np.maximum(p2f_sum, dtype(1e-12))  # soft_rasterize.py:73
    return dict(soft_colors=colors, p2f_info=p2f_info, aggrs_info=aggrs, faces_info=faces_info,
                p2f_raw=p2f, p2f_sum=p2f_sum, face_vertices=fv, textures=tex)


def backward(fwd, grad_soft_colors, cfg, impl="B", ub_texgrad=False, nthreads=0):
    """soft_rasterize backward given the dict returned by forward(). Returns (grad_faces[B,F,9],
    grad_textures[B,F,T2,3]).  `ub_texgrad` (oracle B only) reproduces the as-compiled behaviour of
    kernel.cu:199-218 (gradient added to every texel) instead of the intended one."""
    fv, tex = fwd["face_vertices"], fwd["textures"]
    dtype = fv.dtype.type
    B, F = fv.shape[:2]
    T2 = tex.shape[2]
    S = cfg.image_size
    g = np.ascontiguousarray(np.asarray(grad_soft_colors, dtype=dtype))
    gf = np.zeros((B, F, 9), dtype)
    gt = np.zeros((B, F, T2, 3), dtype)
    lib = _lib(impl)
    sfx = "f32" if dtype == np.float32 else "f64"
    if impl == "A":
        fn = getattr(lib, "ref_backward_soft_rasterize_" + sfx)
        fn(_p(fv), _p(tex), _p(fwd["soft_colors"]), _p(fwd["faces_info"]), _p(fwd["aggrs_info"]),
           _p(gf), _p(gt), _p(g), B, F, S, T2, *cfg.scalars(), ctypes.c_int(_nt(nthreads)))
    else:
        fn = getattr(lib, "oracle_backward_soft_rasterize_" + sfx)
        fn(_p(fv), _p(tex), _p(fwd["soft_colors"]), _p(fwd["faces_info"]), _p(fwd["aggrs_info"]),
           _p(gf), _p(gt), _p(g), B, F, S, T2, *cfg.scalars(), ctypes.c_int(1 if ub_texgrad else 0),
           ctypes.c_int(_nt(nthreads)))
    return gf, gt


def avg_pool2(x):
    """F.avg_pool2d(x, 2, 2) (rasterizer.py:52-53): window summed row-major, then divided by 4."""
    a = x[..., 0::2, 0::2] + x[..., 0::2, 1::2]
    a = a + x[..., 1::2, 0::2]
    a = a + x[..., 1::2, 1::2]
    return a / x.dtype.type(4)


def avg_pool2_backward(g):
    """Gradient of avg_pool2: each hi-res pixel receives g/4."""
    q = g / g.dtype.type(4)
    return np.repeat(np.repeat(q, 2, axis=-2), 2, axis=-1)


def render(face_vertices, textures, image_size, anti_aliasing=True, impl="B", nthreads=0, **kw):
    """SoftRasterizer.forward (rasterizer.py:42-55): returns (images[B,4,is,is], fwd-dict, cfg)."""
    S = image_size * (2 if anti_aliasing else 1)
    cfg = RasterCfg(S, **kw)
    fwd = forward(face_vertices, textures, cfg, impl=impl, nthreads=nthreads)
    images = avg_pool2(fwd["soft_colors"]) if anti_aliasing else fwd["soft_colors"]
    return images, fwd, cfg


def render_backward(fwd, cfg, grad_images, anti_aliasing=True, impl="B", ub_texgrad=False, nthreads=0):
    g = avg_pool2_backward(np.asarray(grad_images, np.float32)) if anti_aliasing else grad_images
    return backward(fwd, g, cfg, impl=impl, ub_texgrad=ub_texgrad, nthreads=nthreads)
