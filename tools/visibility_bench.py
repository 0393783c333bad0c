"""Kernel time (library events) of the visibility passes at a C3-like shape: visible-face bytes (k_visible_faces, face-parallel)
vs planes (k_raster_fwd3<2>, per pixel).

--lib A.so --lib B.so: the same calls through two builds of the library, alternating A, B, A, B ... in one process
(medians per build and mode), with the card's name and power limit, e.g. to compare a kernel change with its parent."""
import argparse, ctypes, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from umr_b200 import _lib, raster, synth

ap = argparse.ArgumentParser()
ap.add_argument("--lib", action="append", default=[], help="a libumr_b200.so to time (twice or more: alternated)")
ap.add_argument("--rounds", type=int, default=10)
ap.add_argument("--calls", type=int, default=20)
a = ap.parse_args()
rng = np.random.default_rng(0)
v, f = synth.icosphere(3)
B, IS = 32, 1024
verts = synth.bird_like(v, rng, B); cams = synth.cameras(rng, B)
fv = torch.from_numpy(synth.raster_space_faces(verts, f, cams)).cuda()
kw = dict(sigma_val=1e-5, dist_eps=1e-10, gamma_val=1e-4, anti_aliasing=True)
if not a.lib:
    for mode in ("faces", "planes"):
        sink = []
        for it in range(8):
            if it == 3: raster.set_profile_sink(sink)
            raster.visibility(fv, IS, want_faces=(mode == "faces"), **kw)
        torch.cuda.synchronize(); raster.set_profile_sink(None)
        pr = raster.collect_profile(sink)
        print("visibility %s: %.3f ms (32 x 2048^2, F=1280)" % (mode, sum(pr["fwd"]) / len(pr["fwd"])))
    sys.exit(0)

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip())
libs = []
for path in a.lib:
    lib = ctypes.CDLL(os.path.abspath(path))
    for name, (res, args) in _lib.EXPORTS.items():
        fn = getattr(lib, name); fn.restype, fn.argtypes = res, args
    libs.append(lib)
F = fv.shape[1]
S = 2 * IS
p = raster.make_params(B, F, 1, IS, True, (0, 0, 0), 1, 100, True, 1e-3, kw["sigma_val"], "euclidean", kw["dist_eps"],
                       kw["gamma_val"], "hard", "prod", "surface")
ws = torch.empty(libs[0].umr_raster_workspace_bytes(B, F, IS, 1), dtype=torch.uint8, device="cuda")
aggrs = torch.empty(B, 2, S, S, device="cuda")
outs = {lib_i: torch.empty(B, F, dtype=torch.uint8, device="cuda") for lib_i in range(len(libs))}
st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def time_calls(i, mode, n):
    lib = libs[i]
    e0, e1 = ctypes.c_void_p(), ctypes.c_void_p()
    lib.umr_event_create(ctypes.byref(e0)); lib.umr_event_create(ctypes.byref(e1))
    p.ev_kernel_start, p.ev_kernel_stop = e0, e1
    ms = []
    for _ in range(n):
        vis = outs[i].data_ptr() if mode == "faces" else None
        pl = aggrs.data_ptr() if mode == "planes" else None
        _lib.check(lib.umr_raster_visibility(fv.data_ptr(), pl, vis, ctypes.byref(p), ws.data_ptr(), st), "umr_raster_visibility")
        t = ctypes.c_float()
        lib.umr_event_elapsed_ms(e0, e1, ctypes.byref(t))
        ms.append(t.value)
    p.ev_kernel_start = p.ev_kernel_stop = None
    lib.umr_event_destroy(e0); lib.umr_event_destroy(e1)
    return ms


for mode in ("faces", "planes"):
    res = {i: [] for i in range(len(libs))}
    for i in range(len(libs)):
        time_calls(i, mode, 5)   # warm-up
    for _ in range(a.rounds):
        for i in range(len(libs)):
            res[i] += time_calls(i, mode, a.calls)
    for i in range(len(libs)):
        q = np.percentile(res[i], [10, 50, 90])
        print("visibility %s %s: median %.4f ms (p10 %.4f, p90 %.4f; %d calls, 32 x 2048^2, F=%d)"
              % (mode, a.lib[i], q[1], q[0], q[2], len(res[i]), F))
if len(libs) > 1:
    assert torch.equal(outs[0], outs[1]), "the builds' visible-face bytes differ"
    print("visible-face bytes identical across builds")
