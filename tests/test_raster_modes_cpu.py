"""Oracle B (our restatement) against oracle A (the reference's own device code compiled for the host) in EVERY mode
combination soft_rasterize accepts: 3 distance x 3 alpha x 2 texture x 2 colour aggregations x single / double-sided.
Single-threaded both run the same IEEE operation sequence, so all five outputs (colours, aggregation planes, p2f,
vertex and texel gradients) must be bit-identical.  The GPU mode sweep (test_raster_modes_gpu.py) is held against
oracle B, so this pins what it is held to."""
import numpy as np
import pytest

import softras
from util import scene

pytestmark = pytest.mark.skipif(not softras.have_oracle_a(), reason="oracle A (reference on host) not built")

SOFT = dict(sigma_val=1e-4, dist_eps=1e-4, gamma_val=1e-3)
COMBOS = [(d, a, t, r, fb) for d in ("hard", "barycentric", "euclidean") for a in ("hard", "sum", "prod")
          for t in ("surface", "vertex") for r in ("softmax", "hard") for fb in (True, False)]


def _inputs(textype, tex_res, seed):
    fv, tex = scene(2, 2, tex_res, seed=seed)    # 320 faces
    if textype == "vertex":
        tex = np.random.default_rng(seed + 1).uniform(0, 1, size=(2, fv.shape[1], 3, 3)).astype(np.float32)
    return fv, tex


@pytest.mark.parametrize("dist,alpha,textype,rgb,fill_back", COMBOS)
def test_every_mode_bit_exact_with_reference_on_host(dist, alpha, textype, rgb, fill_back):
    # S = 37: odd, partial tiles; S = 32: whole 16x16 tiles.  Surface textures at T2 = 1 and 9: with T2 > 1 the
    # reference's texel gradient is undefined (SURVEY.md App. B-1), so grad_textures is compared at T2 = 1 only.
    variants = [(1, True), (3, False)] if textype == "surface" else [(1, True)]
    for S in (37, 32):
        for tex_res, cmp_tex_grad in variants:
            fv, tex = _inputs(textype, tex_res, seed=40 + S + tex_res)
            kw = dict(SOFT, dist_func=dist, aggr_func_alpha=alpha, texture_type=textype, aggr_func_rgb=rgb,
                      fill_back=fill_back, background_color=(0.25, 0.5, 0.75))
            res = {}
            for impl in "AB":
                cfg = softras.RasterCfg(S, **kw)
                fwd = softras.forward(fv, tex, cfg, impl=impl, nthreads=1)
                g = np.random.default_rng(S).normal(size=fwd["soft_colors"].shape).astype(np.float32)
                gf, gt = softras.backward(fwd, g, cfg, impl=impl, nthreads=1)
                res[impl] = dict(soft_colors=fwd["soft_colors"], aggrs_info=fwd["aggrs_info"], p2f_info=fwd["p2f_info"],
                                 grad_faces=gf, grad_textures=gt)
            for k in res["A"]:
                if k == "grad_textures" and not cmp_tex_grad:
                    continue
                assert np.array_equal(res["A"][k], res["B"][k]), "%s differs at S=%d, T2=%d" % (k, S, tex.shape[2])
            # the comparison is not vacuous: the mesh is on screen and the backward produced gradients
            assert (res["B"]["aggrs_info"][:, 1] != res["B"]["aggrs_info"][:, 1, :1, :1]).any()
            assert np.abs(res["B"]["grad_faces"]).max() > 0 or (rgb == "hard" and dist == "hard")
