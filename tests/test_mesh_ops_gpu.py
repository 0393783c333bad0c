"""GPU parity of the SoftRas natives / regularisers / distance transform (csrc/mesh_ops.cu, SURVEY.md §8f-3, §8f-4)
against the CPU oracles of oracle/mesh_oracle.py: the two texture-atlas kernels BIT-EXACT, the regularisers at 1e-5
relative (their dense / ~40-kernel torch forms sum in another order), the distance transform at float32 rounding."""
import os

import numpy as np
import pytest
import torch

import mesh_oracle as O  # oracle/mesh_oracle.py (test infrastructure)
from umr_b200 import ops, synth
from umr_b200 import soft_renderer as sr
from util import rel_report

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("F,R,res", [(20, 2, 8), (320, 6, 16), (7, 3, 5)])
def test_create_texture_image_bit_exact(F, R, res):
    rng = np.random.default_rng(F)
    tex = rng.uniform(0, 1, size=(F, R * R, 3)).astype(np.float32)
    img, vt = sr.functional.create_texture_image(torch.from_numpy(tex).to(DEV), res)
    # restate the host glue of save_obj.py:9-27 for the oracle
    tile_width = int((F - 1.) ** 0.5) + 1
    tile_height = int((F - 1.) / tile_width) + 1
    n = np.arange(F)
    col, row = (n % tile_width).astype(np.float32), (n // tile_width).astype(np.float32)
    v = np.zeros((F, 3, 2), np.float32)
    v[:, 0, 0] = col * res + res / 2; v[:, 0, 1] = row * res + 1
    v[:, 1, 0] = col * res + 1;       v[:, 1, 1] = (row + 1) * res - 1 - 1
    v[:, 2, 0] = (col + 1) * res - 1 - 1; v[:, 2, 1] = (row + 1) * res - 1 - 1
    ref = O.create_texture_image_np(v, tex, np.ones((tile_height * res, tile_width * res, 3), np.float32))[::-1]
    assert img.shape == ref.shape
    assert np.array_equal(img, ref), "max diff %g at %d px" % (np.abs(img - ref).max(), int((img != ref).any(-1).sum()))
    assert vt.shape == (F, 3, 2) and vt.min() >= 0 and vt.max() <= 1


@pytest.mark.parametrize("F,R,H,W", [(30, 4, 64, 48), (320, 6, 128, 256)])
def test_load_textures_bit_exact(F, R, H, W):
    rng = np.random.default_rng(R)
    image = rng.uniform(0, 1, size=(H, W, 3)).astype(np.float32)
    uv = rng.uniform(0.02, 0.95, size=(F, 3, 2)).astype(np.float32)
    # the edges of the uv range (whole faces on u or v = 0 or 1, negative uv): the kernel clamps its corners there
    uv[:4] = np.float32([[[0, 1], [0.5, 1], [1, 1]], [[1, 0], [1, 0.3], [1, 1]], [[0, 0], [0, 0], [0, 0]],
                         [[-0.4, -1.2], [-0.1, 0.5], [0.2, -0.3]]])
    upd = (rng.uniform(size=F) > 0.3).astype(np.int32)
    upd[:4] = 1
    base = rng.uniform(0, 1, size=(F, R * R, 3)).astype(np.float32)
    got = ops.load_textures(torch.from_numpy(image).to(DEV), torch.from_numpy(uv).to(DEV), torch.from_numpy(base.copy()).to(DEV),
                            torch.from_numpy(upd).to(DEV)).cpu().numpy()
    ref = O.load_textures_np(image, uv, upd, base)
    assert np.array_equal(got, ref), "max diff %g" % np.abs(got - ref).max()
    assert np.array_equal(got[upd == 0], base[upd == 0])


def test_save_obj_with_texture_round_trips_through_load_textures(tmp_path):
    v, f = synth.icosphere(1)
    tex = torch.rand(1, f.shape[0], 16, 3, generator=torch.Generator().manual_seed(0))
    m = sr.Mesh(torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV), tex.to(DEV), texture_res=4)
    path = str(tmp_path / "ico.obj")
    m.save_obj(path, save_texture=True, texture_res_out=16)
    assert os.path.exists(path[:-4] + ".png") and os.path.exists(path[:-4] + ".mtl")
    m2 = sr.Mesh.from_obj(path, load_texture=True, texture_res=4)
    assert m2.textures.shape == (1, f.shape[0], 16, 3)
    # atlas (8-bit PNG, nearest texel per atlas pixel) -> bilinear reload: same colours up to quantisation / blending
    assert float((m2.textures.cpu() - tex).abs().mean()) < 0.12
    assert torch.equal(m2.faces.cpu(), torch.from_numpy(f)[None])


@pytest.mark.parametrize("subdiv,B,average", [(2, 3, False), (3, 2, True)])
def test_laplacian_and_flatten_losses(subdiv, B, average):
    rng = np.random.default_rng(subdiv)
    v, f = synth.icosphere(subdiv)
    verts = torch.from_numpy(synth.bird_like(v, rng, B))
    faces = torch.from_numpy(f.astype(np.int64))
    w = torch.from_numpy(rng.uniform(0.5, 1.5, size=(B,)).astype(np.float32))
    for name, mod, ref_fn in (("laplacian", sr.LaplacianLoss(torch.from_numpy(v), faces, average=average), O.laplacian_loss),
                              ("flatten", sr.FlattenLoss(faces, average=average), O.flatten_loss)):
        xr = verts.clone().requires_grad_(True)
        ref = ref_fn(xr, f, average=average)
        (ref if average else (ref * w).sum()).backward()
        xg = verts.clone().to(DEV).requires_grad_(True)
        got = mod.to(DEV)(xg)
        (got if average else (got * w.to(DEV)).sum()).backward()
        ok, msg = rel_report(name, got.detach().cpu().numpy(), ref.detach().numpy(), 2e-5, 1e-6)
        print(msg)
        assert ok, msg
        ok, msg = rel_report(name + " grad", xg.grad.cpu().numpy(), xr.grad.numpy(), 1e-4, 2e-5 * float(xr.grad.abs().max()))
        print(msg)
        assert ok, msg


@pytest.mark.parametrize("size", [64, 256, (48, 80)])
def test_dt_barrier_matches_scipy(size):
    rng = np.random.default_rng(0)
    H, W = (size, size) if isinstance(size, int) else size
    masks = np.stack([synth.ellipse_masks(rng, 1, max(H, W))[0][:H, :W] for _ in range(3)])
    masks[2, : H // 3] = 0
    masks[2, 5:9, 3:7] = 1  # a second blob
    got = ops.dt_barrier(torch.from_numpy(masks).to(DEV)).cpu().numpy()
    ref = np.stack([O.dt_barrier(m) for m in masks]).astype(np.float32)   # train_s2.py:196 casts to FloatTensor
    assert np.abs(got - ref).max() <= 2e-7, np.abs(got - ref).max()
    # degenerate masks (no object / no background): scipy's virtual-pixel behaviour is reproduced as well
    deg = np.stack([np.zeros((H, W), np.float32), np.ones((H, W), np.float32)])
    got = ops.dt_barrier(torch.from_numpy(deg).to(DEV)).cpu().numpy()
    ref = np.stack([O.dt_barrier(m) for m in deg]).astype(np.float32)
    assert np.abs(got - ref).max() <= 2e-7
