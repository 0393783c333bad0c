"""The 32-byte pair record (csrc/raster_stream.cuh): the streamed backward re-derives the z-gradient factors
w_clip_k / z_k^2 from the face record instead of reading them from the pair buffer.  At the C2 shape (and one
32x32-tile shape) its gradients must match the recompute backward, the forward must not depend on whether records are
saved, and the pair buffer raster.py sizes for C2 must keep every tile's records."""
import numpy as np
import pytest
import torch

from umr_b200 import _lib, raster
from util import rel_report, scene
from test_raster_gpu import UMR

DEV = "cuda:0"


def _render(fv, tex, image_size, g, cand, tile):
    old = raster.PAIR_CAND_PER_PIXEL, raster.FORWARD_TILE, raster.PAIR_ADAPTIVE
    raster.PAIR_CAND_PER_PIXEL, raster.FORWARD_TILE, raster.PAIR_ADAPTIVE = cand, tile, False
    try:
        tfv = torch.from_numpy(fv).to(DEV).requires_grad_(True)
        ttex = torch.from_numpy(tex).to(DEV).requires_grad_(True)
        img, p2f, aggr = raster.soft_rasterize(tfv, ttex, image_size, anti_aliasing=True, **UMR)
        saved = img.grad_fn.saved_tensors
        stats = saved[4][:8].view(torch.int32).cpu().tolist() if len(saved) == 5 else None
        img.backward(torch.from_numpy(g).to(DEV))
        torch.cuda.synchronize()
        return dict(images=img.detach().cpu().numpy(), p2f=p2f.cpu().numpy(), aggrs=aggr.cpu().numpy(),
                    grad_faces=tfv.grad.cpu().numpy(), grad_tex=ttex.grad.cpu().numpy(), stats=stats)
    finally:
        raster.PAIR_CAND_PER_PIXEL, raster.FORWARD_TILE, raster.PAIR_ADAPTIVE = old


@pytest.mark.gpu
@pytest.mark.parametrize("B,subdiv,tex_res,image_size,tile", [(16, 3, 6, 256, 16),   # C2 (16x16-tile forward)
                                                              (2, 3, 3, 128, 32)])  # 32x32-tile forward
def test_streamed_backward_matches_recompute(B, subdiv, tex_res, image_size, tile):
    fv, tex = scene(B, subdiv, tex_res, seed=23)
    g = np.random.default_rng(4).normal(size=(B, 4, image_size, image_size)).astype(np.float32)
    saved = _render(fv, tex, image_size, g, 32.0, tile)
    recomputed = _render(fv, tex, image_size, g, 0.0, tile)
    assert saved["stats"][1] == 0 and saved["stats"][0] > 0, saved["stats"]
    assert recomputed["stats"] is None
    for k in ("images", "aggrs"):   # every forward plane, bit for bit, whether records are saved or not
        assert np.array_equal(saved[k], recomputed[k]), k
    np.testing.assert_allclose(saved["p2f"], recomputed["p2f"], rtol=1e-5, atol=1e-6)   # p2f sums are float REDs
    for k in ("grad_faces", "grad_tex"):
        ref = recomputed[k]
        ok, msg = rel_report(k, saved[k], ref, 1e-4, 1e-6 * float(np.abs(ref).max()) + 1e-7)
        print(msg)
        assert ok, msg


def test_pair_buffer_bytes_reserve_1540_per_block():
    lib = _lib.load()
    for B, image_size, aa in ((16, 256, 1), (2, 64, 0)):
        a = lib.umr_raster_pair_buffer_bytes(B, image_size, aa, 1024)   # (multiples of 64: the headers are 256-byte aligned)
        b = lib.umr_raster_pair_buffer_bytes(B, image_size, aa, 3072)
        assert b - a == 2048 * 1540, (a, b)


@pytest.mark.gpu
def test_raster_py_sizing_saves_every_tile_at_c2(monkeypatch):
    """The first C2 render (fixed budget) and the next one (sized from the measured need) leave no tile unsaved."""
    monkeypatch.setattr(raster, "PAIR_ADAPTIVE", True)
    monkeypatch.setattr(raster, "PAIR_CAND_PER_PIXEL", 8.0)
    monkeypatch.setattr(raster, "FORWARD_TILE", 0)
    monkeypatch.setattr(raster, "_pair_need", {})
    monkeypatch.setattr(raster, "_pair_pending", [])
    B, image_size = 16, 256
    fv, tex = scene(B, 3, 6, seed=29)
    g = torch.ones(B, 4, image_size, image_size, device=DEV)
    sizes = []
    for _ in range(2):
        tfv = torch.from_numpy(fv).to(DEV).requires_grad_(True)
        img, _, _ = raster.soft_rasterize(tfv, torch.from_numpy(tex).to(DEV), image_size, anti_aliasing=True, **UMR)
        pairs = img.grad_fn.saved_tensors[4]
        img.backward(g)
        torch.cuda.synchronize()
        wanted, unsaved = pairs[:8].view(torch.int32).cpu().tolist()
        assert wanted > 0 and unsaved == 0, (wanted, unsaved)
        sizes.append(pairs.numel())
    assert sizes[1] < sizes[0], sizes   # the second buffer was sized from the first render's counters
