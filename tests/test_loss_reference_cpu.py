"""Pins the float64 reference of the loss and mesh-op kernels (oracle/loss_ref.py) before tests/test_loss_range_gpu.py
relies on it: it agrees with the existing float32 oracles (oracle/losses.py, oracle/mesh_oracle.py) within their
rounding bound, its gradients pass gradcheck, and the brute-force distance transform equals scipy on tall, wide,
one-pixel-thin, empty, full and non-binary masks."""
import numpy as np
import pytest
import torch

import loss_ref as R
import losses as O
import mesh_oracle as MO
from loss_ref import gamma
from umr_b200 import synth
from umr_b200 import soft_renderer as sr


def _within(name, got, ref, bound):
    got, ref, bound = (torch.as_tensor(x).double() for x in (got, ref, bound))
    err = (got - ref).abs()
    ratio = float((err / bound.clamp_min(1e-300)).max())
    print("%-36s max err/bound = %.3e" % (name, ratio))
    assert bool((err <= bound).all()), "%s: worst err/bound %.3g" % (name, ratio)


def test_sampler_matches_grid_sample():
    g = torch.Generator().manual_seed(0)
    for C, H, W in ((1, 5, 7), (3, 1, 6), (4, 6, 1), (2, 9, 9)):
        img = torch.rand(2, C, H, W, generator=g) * 2 - 1
        flow = torch.rand(2, 37, 2, generator=g) * 2.4 - 1.2
        flow[0, :4] = torch.tensor([[-1.0, -1.0], [1.0, 1.0], [1.0, -1.0], [0.0, 0.0]])
        ref32 = O.sample_textures(flow.view(2, 37, 1, 1, 2), img).reshape(2, 37, C)
        out = R.sample_ref(img.double(), flow)
        mag, _, _, _ = R.sample_magnitude(img.double(), flow, torch.ones(2, 37, C))
        _within("sampler C=%d %dx%d" % (C, H, W), ref32, out, gamma(9) * mag)


def test_sampler_gradients():
    g = torch.Generator().manual_seed(1)
    img = torch.rand(1, 2, 5, 9, generator=g, dtype=torch.float64).requires_grad_(True)
    flow = (torch.randint(-1100, 1100, (1, 23, 2), generator=g).double() / 1024)   # dyadic: exact in float32
    assert torch.autograd.gradcheck(lambda im: R.sample_ref(im, flow), (img,))
    # flow: bilinear within a cell, so a central difference whose two points share the cell is exact
    fl = flow.clone().requires_grad_(True)
    w = torch.rand(1, 23, 2, generator=g, dtype=torch.float64)
    gf, = torch.autograd.grad((R.sample_ref(img.detach(), fl) * w).sum(), fl)
    h = 2.0 ** -14
    for n in range(23):
        for d in range(2):
            lo, hi = flow.clone(), flow.clone()
            lo[0, n, d] -= h
            hi[0, n, d] += h
            ix = lambda f: np.floor(((f.float()[0, n] + 1) / 2 * torch.tensor([8.0, 4.0])).numpy())   # noqa: E731
            if not np.array_equal(ix(lo), ix(hi)):
                continue
            fd = ((R.sample_ref(img.detach(), hi) - R.sample_ref(img.detach(), lo)) * w).sum() / (2 * h)
            assert abs(float(fd) - float(gf[0, n, d])) <= 1e-9 * max(1.0, abs(float(fd)))


def test_iou_l1_loss_head_match_float32_oracles():
    g = torch.Generator().manual_seed(2)
    B, H, W = 3, 23, 31
    rgba = torch.rand(B, 4, H, W, generator=g)
    gt = torch.rand(B, 3, H, W, generator=g)
    m = (torch.rand(B, H, W, generator=g) > 0.5).float()
    N = H * W
    li, I, U = R.iou_ref(rgba[:, 3].double(), m.double())
    _, Im, Um = R.iou_ref(rgba[:, 3].double(), m.double(), magnitude=True)
    ref32 = O.neg_iou_loss(rgba[:, 3], m, avg=False)
    eI, eU = gamma(3 + N) * Im, gamma(4 + N) * Um
    _within("iou", ref32, li, (eI + I / U * eU) / U + gamma(2) * (I / U + li.abs()))
    l1 = R.masked_l1_ref(rgba[:, :3].double(), gt.double(), m.double(), rgba[:, 3].double())
    l1m = R.masked_l1_ref(rgba[:, :3].double(), gt.double(), m.double(), rgba[:, 3].double(), magnitude=True)
    _within("masked l1", O.texture_loss_masks(rgba[:, :3], gt, m, rgba[:, 3], avg=False), l1, gamma(5 + 3 * N) * l1m)
    loss, per = R.loss_head_ref(rgba.double(), gt.double(), m.double(), 2.5, 3.0)
    assert torch.allclose(per[:, 0], li) and torch.allclose(per[:, 1], l1)
    assert abs(float(loss) - float(2.5 * li.mean() + 3.0 * l1.mean())) < 1e-15


def test_chamfer_matches_float32_oracle():
    g = torch.Generator().manual_seed(3)
    for D in (2, 3):
        a = torch.rand(2, 40, D, generator=g) - 0.5
        b = torch.rand(2, 29, D, generator=g) - 0.5
        b[:, 7] = b[:, 3]                                                           # duplicate points
        n = O.dist_chamfer_np(a.numpy(), b.numpy())
        r = R.chamfer_ref(a.double(), b.double())
        mag = R.chamfer_ref(a.double().abs(), b.double().abs(), r[2], r[3], magnitude=True)
        assert R.near_tie(a.double(), b.double(), torch.from_numpy(n[2]), r[2], 2).all()
        assert R.near_tie(b.double(), a.double(), torch.from_numpy(n[3]), r[3], 2).all()
        r = R.chamfer_ref(a.double(), b.double(), torch.from_numpy(n[2]), torch.from_numpy(n[3]))
        _within("chamfer d_ab D=%d" % D, n[0], r[0], gamma(6) * mag[0])
        _within("chamfer d_ba D=%d" % D, n[1], r[1], gamma(6) * mag[1])
        ri = R.chamfer_ref(a.double(), b.double())
        assert (ri[3][:, 7] == ri[3][:, 3]).all() and (torch.argmin(R._sqdist(a.double(), b.double()), 2) != 7).all()


def test_texcycle_matches_oracle_and_visibility_rule():
    g = torch.Generator().manual_seed(4)
    B, F, T, P = 2, 20, 3, 50
    flow = torch.rand(B, F, T, T, 2, generator=g) * 2 - 1
    prob = torch.rand(B, F, 2, generator=g) * 2 - 1
    ids = torch.randint(-1, F, (B, P), generator=g).float()
    ref32, _ = O.tex_cycle(flow, prob, ids)
    vis = R.visible_ref(ids, F)
    r = R.texcycle_ref(flow.double().reshape(B, F, T * T, 2), prob.double(), vis)
    rm = R.texcycle_ref(flow.double().reshape(B, F, T * T, 2), prob.double(), vis, magnitude=True)
    _within("texcycle", ref32, r, gamma(T * T + 6 + B * F) * rm)
    odd = torch.tensor([[-1.0, -2.0, float(F), float(F + 3), -float(F), -float(F) - 1, 2.0]])
    assert R.visible_ref(odd, F).nonzero()[:, 1].tolist() == [0, 2, F - 2, F - 1]


def test_mesh_helper_is_closed_with_a_wide_valence_spread():
    v, f = R.spiked_uv_sphere(12, 12, 5)
    val = np.bincount(f.reshape(-1), minlength=len(v))
    assert val.min() == 3 and val.max() >= 12
    fl = sr.FlattenLoss(torch.from_numpy(f))
    assert fl.edge_table.shape[0] * 2 == 3 * len(f)                                 # closed: every edge has two faces


def test_laplacian_flatten_match_oracles_and_gradcheck():
    v, f = R.spiked_uv_sphere(6, 7, 3)
    rng = np.random.default_rng(5)
    x = torch.from_numpy((v[None] * rng.uniform(0.8, 1.2, (2, len(v), 1))).astype(np.float32))
    lap = sr.LaplacianLoss(torch.from_numpy(v), torch.from_numpy(f))
    ref32 = MO.laplacian_loss(x, f)
    r, _ = R.laplacian_ref(x.double(), lap.csr_rowptr, lap.csr_col, lap.csr_coef)
    rm, _ = R.laplacian_ref(x.double().abs(), lap.csr_rowptr, lap.csr_col, lap.csr_coef, magnitude=True)
    _within("laplacian", ref32, r, gamma(2 * len(v) + 8) * rm)            # the dense matmul sums over a whole row
    fl = sr.FlattenLoss(torch.from_numpy(f))
    ref32 = MO.flatten_loss(x, f)
    r = R.flatten_ref(x.double(), fl.edge_table)
    lb, _ = R.flatten_error_bound(x, fl.edge_table, 1e-6, torch.ones(2), 8 + fl.edge_table.shape[0])
    _within("flatten", ref32, r, lb)
    xd = x.double().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda t: R.laplacian_ref(t, lap.csr_rowptr, lap.csr_col, lap.csr_coef)[0], (xd,))
    assert torch.autograd.gradcheck(lambda t: R.flatten_ref(t, fl.edge_table), (xd,))


def test_loss_gradcheck():
    g = torch.Generator().manual_seed(6)
    p = torch.rand(2, 30, generator=g, dtype=torch.float64).requires_grad_(True)
    t = (torch.rand(2, 30, generator=g) > 0.5).double()
    assert torch.autograd.gradcheck(lambda q: R.iou_ref(q, t)[0], (p,))
    rgba = (torch.rand(2, 4, 3, 5, generator=g, dtype=torch.float64) * 0.9 + 0.05).requires_grad_(True)
    gt = torch.rand(2, 3, 3, 5, generator=g, dtype=torch.float64)
    m = torch.rand(2, 3, 5, generator=g, dtype=torch.float64)
    assert torch.autograd.gradcheck(lambda x: R.loss_head_ref(x, gt, m, 2.5, 3.0)[0], (rgba,))
    assert torch.autograd.gradcheck(lambda x: R.masked_l1_ref(x[:, :3], gt, m, x[:, 3]), (rgba,))
    a = torch.rand(2, 9, 3, generator=g, dtype=torch.float64).requires_grad_(True)
    b = torch.rand(2, 5, 3, generator=g, dtype=torch.float64).requires_grad_(True)
    ia, ib = R.chamfer_ref(a, b)[2:]
    assert torch.autograd.gradcheck(lambda x, y: R.chamfer_ref(x, y, ia, ib)[:2], (a, b))
    fl = torch.rand(2, 4, 9, 2, generator=g, dtype=torch.float64).requires_grad_(True)
    pr = torch.rand(2, 4, 2, generator=g, dtype=torch.float64)
    vis = torch.tensor([[True, False, True, True], [False, True, True, False]])
    assert torch.autograd.gradcheck(lambda x: R.texcycle_ref(x, pr, vis), (fl,))


def _masks():
    rng = np.random.default_rng(7)
    out = {"tall": (rng.uniform(size=(23, 7)) > 0.6).astype(np.float32),
           "wide": (rng.uniform(size=(5, 29)) > 0.7).astype(np.float32),
           "row": (rng.uniform(size=(1, 17)) > 0.5).astype(np.float32),
           "column": (rng.uniform(size=(13, 1)) > 0.5).astype(np.float32),
           "empty": np.zeros((9, 12), np.float32), "full": np.ones((12, 9), np.float32),
           "dot": np.zeros((11, 8), np.float32), "half": np.full((6, 10), 0.5, np.float32),
           "nonbinary": rng.choice(np.float32([0, 0.25, 0.5, 1, 2]), size=(14, 10)).astype(np.float32),
           "ellipse": synth.ellipse_masks(rng, 1, 24)[0][:19]}
    out["dot"][7, 2] = 1
    return out


@pytest.mark.parametrize("name", list(_masks()))
def test_brute_force_edt_equals_scipy(name):
    from scipy.ndimage import distance_transform_edt
    m = _masks()[name]
    d2o, d2i = R.edt_sq_brute(m)
    assert np.array_equal(np.sqrt(d2o.astype(np.float64)), distance_transform_edt(1 - m))
    assert np.array_equal(np.sqrt(d2i.astype(np.float64)), distance_transform_edt(m))
    assert np.allclose(R.dt_barrier_ref(m), MO.dt_barrier(m), rtol=0, atol=1e-15)


def test_load_textures_oracle_clamps_at_the_image_edge():
    img = np.arange(2 * 3 * 3, dtype=np.float32).reshape(2, 3, 3)
    uv = np.float32([[[1, 1], [1, 1], [1, 1]], [[0, 0], [0, 0], [0, 0]], [[-0.6, -2], [-0.6, -2], [-0.6, -2]],
                     [[1, 0], [1, 0], [1, 0]]])
    out = MO.load_textures_np(img, uv, np.ones(4, np.int32), np.zeros((4, 1, 3), np.float32))
    assert np.array_equal(out[0, 0], img[1, 2]) and np.array_equal(out[1, 0], img[0, 0])
    assert np.array_equal(out[3, 0], img[0, 2]) and np.isfinite(out).all()
