"""Pins the float64 reference of the fused vertex kernels (oracle/vertex_ref.py) before the GPU tests lean on it.

* Its forward is the existing float32 chain (`OracleSoftRenderer.face_vertices` and the closed-form light of
  tests/test_dropin_gpu.py) up to float32 rounding, and its bound: each float32 value lies within
  gamma_n * (magnitude evaluation) of the float64 one, n the longest chain of roundings (oracle/vertex_ref.py).
* Its projection is the existing float64 oracle `losses.orthographic_proj_withz` bit for bit.
* Its gradients pass `torch.autograd.gradcheck` for vertices and cameras, with the light on, H > 1 camera
  hypotheses, and a face small enough to take the eps branch of the normalisation.
* `corr_chamfer_ref` is `train_step.corr_loss_chamfer` (values and gradients) at UMR's weights.
"""
import numpy as np
import torch

import losses as L
import train_step as O
import vertex_ref as R
from umr_b200 import synth

from vertex_ref import gamma

DEFAULT_LIGHT = (0.8, (1, 1, 1), 0.5, (1, 1, 1), (0, 1, 0))   # smr.py:63, renderer.py:57-60


def _mesh(B=2, subdiv=1, seed=0):
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(subdiv)
    verts = torch.from_numpy(synth.bird_like(v, rng, B))
    cams = torch.from_numpy(synth.cameras(rng, B))
    faces = torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1)
    return verts, cams, faces


def test_projection_is_the_float64_oracle():
    verts, cams, _ = _mesh(B=3)
    got = R.project_vertices(verts.double(), cams.double(), 5.0)
    assert torch.equal(got, L.orthographic_proj_withz(verts.double(), cams.double(), offset_z=5.0))


def test_forward_matches_the_float32_chain_within_its_rounding_bound():
    verts, cams, faces = _mesh(B=3, subdiv=2)
    fv32, pre32 = O.OracleSoftRenderer(32).face_vertices(verts, faces, cams)   # float32 torch chain
    vd, cd = verts.double(), cams.double()
    fv, lt, pre = R.project_faces_ref(vd, cd, faces, 5.0, float(np.float32(-2.732)), 1.0, True, DEFAULT_LIGHT,
                                      with_pre=True)
    mag, _ = R.project_faces_ref(vd.abs(), cd.abs(), faces, 5.0, float(np.float32(-2.732)), 1.0, True, None,
                                 magnitude=True)
    # 11 roundings: 4 in (0,X) (x) conj(q), 4 in q (x) t, scale, translate / offset, then look_at or orthogonal
    err = (fv32.double() - fv).abs()
    assert (err <= gamma(11) * mag).all(), float((err / (gamma(11) * mag)).max())
    assert float(err.max()) > 0   # the chains are not the same computation
    # closed-form light of the float32 chain (test_dropin_gpu.py) against the reference's light
    n = torch.nn.functional.normalize(torch.cross(pre32[:, :, 2] - pre32[:, :, 1], pre32[:, :, 0] - pre32[:, :, 1],
                                                  dim=2), p=2, dim=2, eps=1e-6)
    light32 = 0.8 + 0.5 * torch.relu(n[:, :, 1])
    bound = R.light_error_bound(vd, cd, faces, 5.0, True, DEFAULT_LIGHT)
    err = (light32.double()[..., None] - lt).abs()
    assert (err <= bound).all(), float((err / bound).max())
    assert float(lt.min()) < 0.81 and float(lt.max()) > 1.2   # shadowed and lit faces both occur


def _small_case(H, seed):
    torch.manual_seed(seed)
    Bv, V = 2, 6
    verts = (torch.rand(Bv, V, 3, dtype=torch.float64) - 0.5)
    cams = torch.cat([0.6 + 0.2 * torch.rand(Bv * H, 1), 0.1 * torch.randn(Bv * H, 2),
                      torch.nn.functional.normalize(torch.randn(Bv * H, 4), dim=1)], 1).double()
    faces = torch.stack([torch.tensor([[0, 1, 2], [2, 3, 4], [1, 4, 5], [5, 0, 3]]),
                         torch.tensor([[3, 4, 5], [0, 2, 4], [1, 3, 5], [2, 1, 0]])])
    return verts, cams, faces


def test_gradcheck_with_light_and_hypotheses():
    verts, cams, faces = _small_case(H=3, seed=1)
    light = (0.3, (0.9, 0.5, 0.2), 0.7, (0.4, 1.0, 0.6), (0.3, 1.1, -0.4))
    v = verts.clone().requires_grad_(True)
    c = cams.clone().requires_grad_(True)

    def fn(v, c):
        fv, lt = R.project_faces_ref(v, c, faces, 5.0, -2.732, 0.75, True, light)
        return fv, lt
    _, lt = fn(v, c)
    assert (lt > 0.3 * torch.tensor([0.9, 0.5, 0.2]) + 1e-3).any()      # some faces lit: the light backward runs
    assert torch.autograd.gradcheck(fn, (v, c), eps=1e-6, atol=1e-7, rtol=1e-6)


def test_gradcheck_on_the_eps_branch_of_the_normalisation():
    # legs of 2^-10: |cross| = 2^-20 < 1e-6, so n_hat = n / 1e-6 (F.normalize's clamp) and is no unit vector
    verts = torch.tensor([[[0.25, 0.5, 0.125], [0.25 + 2 ** -10, 0.5, 0.125], [0.25, 0.5 + 2 ** -10, 0.125]]],
                         dtype=torch.float64)
    cams = torch.tensor([[1.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]], dtype=torch.float64)
    faces = torch.tensor([[0, 2, 1]])
    light = (0.5, (1, 1, 1), 0.5, (1, 1, 1), (0.2, 0.3, 1.0))
    _, _, pre = R.project_faces_ref(verts, cams, faces, 5.0, -2.732, 1.0, True, light, with_pre=True)
    n = torch.cross(pre[:, :, 2] - pre[:, :, 1], pre[:, :, 0] - pre[:, :, 1], dim=2)
    assert float(n.norm()) < 1e-6
    _, lt = R.project_faces_ref(verts, cams, faces, 5.0, -2.732, 1.0, True, light)
    assert float(lt[0, 0, 0]) > 0.5                  # lit, so the gradient goes through the eps branch
    v = verts.clone().requires_grad_(True)
    c = cams.clone().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda v, c: R.project_faces_ref(v, c, faces, 5.0, -2.732, 1.0, True, light)[1],
                                    (v, c), eps=1e-8, atol=1e-4, rtol=1e-5)   # entries are O(1)


def test_face_layouts_agree():
    verts, cams, faces = _mesh(B=2, subdiv=1)
    cams = torch.cat([cams, cams.flip(0)]).double()      # H = 2
    vd = verts.double()
    a, _ = R.project_faces_ref(vd, cams, faces[0], 5.0, -2.732)
    b, _ = R.project_faces_ref(vd, cams, faces[:1], 5.0, -2.732)
    c, _ = R.project_faces_ref(vd, cams, faces, 5.0, -2.732)
    assert torch.equal(a, b) and torch.equal(a, c)
    # per-mesh face lists: render b gathers mesh b // H's faces from mesh b // H's vertices
    perm = faces.clone()
    perm[1] = faces[1][torch.randperm(faces.shape[1], generator=torch.Generator().manual_seed(0))]
    d, _ = R.project_faces_ref(vd, cams, perm, 5.0, -2.732)
    assert torch.equal(d[:2], a[:2]) and not torch.equal(d[2:], a[2:])
    full, _ = R.project_faces_ref(vd.repeat_interleave(2, 0), cams, perm.repeat_interleave(2, 0), 5.0, -2.732)
    assert torch.equal(d, full)


def test_corr_chamfer_ref_matches_the_oracle_composition():
    rng = np.random.default_rng(4)
    B = 3
    v, _ = synth.icosphere(2)
    verts0 = torch.from_numpy(synth.bird_like(v, rng, B)).double()
    cams0 = torch.from_numpy(synth.cameras(rng, B)).double()
    parts = [torch.from_numpy(p) for p in synth.part_vertex_sets(rng, v.shape[0], sizes=(20, 30, 10, 15))]
    targets = [torch.from_numpy(t).double() for t in synth.part_points(rng, B, sizes=(7, 33, 5, 12))]
    outs = []
    for ref in (True, False):
        verts, cams = verts0.clone().requires_grad_(True), cams0.clone().requires_grad_(True)
        if ref:
            loss, vert2d, _ = R.corr_chamfer_ref(verts, cams, parts, targets)
        else:
            loss = O.corr_loss_chamfer(O.OracleSoftRenderer(32), parts, *targets, verts, cams, avg=False)
            vert2d = None
        (loss * torch.tensor([0.5, 1.0, 2.0], dtype=torch.float64)).sum().backward()
        outs.append((loss.detach(), verts.grad, cams.grad, vert2d))
    for a, b in zip(outs[0][:3], outs[1][:3]):
        assert torch.allclose(a, b, rtol=1e-12, atol=1e-14)
    sel = torch.cat(parts)
    assert torch.equal(outs[0][3].detach(), L.orthographic_proj_withz(verts0[:, sel], cams0)[:, :, :2])
