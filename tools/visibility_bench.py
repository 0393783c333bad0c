"""Kernel time (library events) of the visibility passes at a C3-like shape: visible-face bytes (k_visible_faces, face-parallel)
vs planes (k_raster_fwd3<2>, per pixel)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from umr_b200 import raster, synth
rng = np.random.default_rng(0)
v, f = synth.icosphere(3)
B, IS = 32, 1024
verts = synth.bird_like(v, rng, B); cams = synth.cameras(rng, B)
fv = torch.from_numpy(synth.raster_space_faces(verts, f, cams)).cuda()
kw = dict(sigma_val=1e-5, dist_eps=1e-10, gamma_val=1e-4, anti_aliasing=True)
for mode in ("faces", "planes"):
    sink = []
    for it in range(8):
        if it == 3: raster.set_profile_sink(sink)
        raster.visibility(fv, IS, want_faces=(mode == "faces"), **kw)
    torch.cuda.synchronize(); raster.set_profile_sink(None)
    pr = raster.collect_profile(sink)
    print("visibility %s: %.3f ms (32 x 2048^2, F=1280)" % (mode, sum(pr["fwd"]) / len(pr["fwd"])))
