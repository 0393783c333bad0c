"""SCOPS part centres and part points (csrc/part_points.cu, DESIGN.md §17) against the numpy restatement
(tests/part_points_oracle.py) across the accepted input range.

With the uniforms injected, the drawn pixel sets and the kept points equal the restatement bit for bit; the restatement
selects around the kernel's own centres, which are checked separately against float64 within their stated bound."""
import ctypes

import numpy as np
import pytest
import torch

import part_points_oracle as ppo
from umr_b200 import _lib, synth
from umr_b200.nnutils import loss_utils
from umr_b200.raster import _stream_ptr
from umr_b200.utils import image

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
DTYPES = {np.float32: torch.float32, np.float64: torch.float64}
CH, NS = (1, 2, 3, 4), (10, 10, 30, 30)


def _call(prob, mask, u, channels, ns, dtype, centers_in=None):
    t = DTYPES[dtype]
    c_in = torch.as_tensor(centers_in, device=DEV) if centers_in is not None else None
    centers, points, drawn = image._part_points(torch.as_tensor(prob, device=DEV).to(t), torch.as_tensor(mask, device=DEV),
                                                torch.as_tensor(u, device=DEV).to(t), ns, channels, centers_in=c_in,
                                                drawn=True)
    return centers.cpu().numpy(), [p.cpu().numpy() for p in points], [d.cpu().numpy() for d in drawn]


def _uniforms(rng, B, K, S, dtype):
    return rng.random((B, K, S * S)).astype(dtype)


def check(prob, mask, u, channels, ns, dtype):
    """One call against the restatement: drawn sets and points exactly, centres within the bound.  Returns the outputs."""
    centers, points, drawn = _call(prob, mask, u, channels, ns, dtype)
    assert centers.dtype == dtype and all(p.dtype == dtype for p in points)
    dr_ref, pts_ref = ppo.part_points(prob, mask, u, channels, ns, dtype, centers)
    for k in range(len(channels)):
        np.testing.assert_array_equal(drawn[k], dr_ref[k])
        np.testing.assert_array_equal(points[k], pts_ref[k])
    for b in range(prob.shape[0]):
        for k, ch in enumerate(channels):
            want = ppo.centre(prob[b], mask[b], ch)
            bound = ppo.centre_bound(prob[b], mask[b], ch, dtype)
            assert (np.abs(centers[b, k] - want) <= bound).all(), (b, k, centers[b, k], want, bound)
    return centers, points, drawn


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("S", [256, 64])
def test_injected_uniforms_match_the_restatement(S, dtype):
    rng = np.random.default_rng(S)
    prob, mask = ppo.scops_like(rng, 3, S)
    check(prob, mask, _uniforms(rng, 3, 4, S, dtype), CH, NS, dtype)


@pytest.mark.parametrize("B", [1, 512])
def test_batch_sizes(B):
    rng = np.random.default_rng(B)
    prob, mask = ppo.scops_like(rng, min(B, 8), 64)
    idx = rng.integers(0, prob.shape[0], B)
    prob, mask = prob[idx], mask[idx]
    check(prob, mask, _uniforms(rng, B, 4, 64, np.float32), CH, NS, np.float32)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_one_sample_and_the_largest_draw(dtype):
    # n = 1 draws int(1.5) = 1 pixel; n = 683 draws 1024, the most one call takes
    rng = np.random.default_rng(3)
    prob, mask = ppo.scops_like(rng, 2, 64)
    prob[..., 2] = np.maximum(prob[..., 2], 0.01)
    mask[:] = 1                                  # 4096 positive pixels for the 1024 draws
    check(prob, mask, _uniforms(rng, 2, 3, 64, dtype), (1, 2, 4), (1, 683, 5), dtype)


def test_exactly_m_positive_pixels_are_all_drawn():
    rng = np.random.default_rng(4)
    prob, mask = ppo.scops_like(rng, 2, 64)
    mask[:] = 0
    pix = rng.choice(64 * 64, 15, replace=False)
    mask.reshape(2, -1)[:, pix] = 1.0                 # 15 = int(1.5 * 10) positive pixels
    _, _, drawn = check(prob, mask, _uniforms(rng, 2, 2, 64, np.float32), (1, 2), (10, 10), np.float32)
    for d in drawn:
        np.testing.assert_array_equal(d, np.sort(np.broadcast_to(pix, d.shape), axis=1))


def test_one_pixel_wide_part():
    rng = np.random.default_rng(5)
    prob, mask = ppo.scops_like(rng, 2, 64)
    prob[..., 1:3] = 0
    prob[:, 8:56, 30, 1] = rng.uniform(0.1, 1.0, (2, 48))      # one column
    prob[:, 20, 4:60, 2] = rng.uniform(0.1, 1.0, (2, 56))      # one row
    mask[:] = 1
    _, points, _ = check(prob, mask, _uniforms(rng, 2, 2, 64, np.float32), (1, 2), (30, 30), np.float32)
    assert (points[0][:, :, 0] == 30 / 128 - 1).all() and (points[1][:, :, 1] == 20 / 128 - 1).all()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_distance_ties_take_the_lower_pixel_index(dtype):
    # a disc of pixels round pixel (32, 32) with the centre given at that pixel, (0, 0): rings of equidistant pixels,
    # kept by pixel index across the cut
    S = 64
    yy, xx = np.mgrid[0:S, 0:S]
    prob = np.zeros((1, S, S, 2), np.float32)
    prob[0, :, :, 1] = np.where((xx - 32) ** 2 + (yy - 32) ** 2 <= 25, 1.0, 0.0)
    mask = np.ones((1, S, S))
    zero = np.zeros((1, 1, 2), dtype)
    rng = np.random.default_rng(6)
    for n in (5, 13, 40):
        u = _uniforms(rng, 1, 1, S, dtype)
        _, points, drawn = _call(prob, mask, u, (1,), (n,), dtype, centers_in=zero)
        dr_ref, pts_ref = ppo.part_points(prob, mask, u, (1,), (n,), dtype, zero)
        np.testing.assert_array_equal(drawn[0], dr_ref[0])
        np.testing.assert_array_equal(points[0], pts_ref[0])
        xy = ppo.coords(drawn[0][0], S, dtype)
        d = xy[:, 0] * xy[:, 0] + xy[:, 1] * xy[:, 1]
        assert len(np.unique(d)) < len(d)        # the draw holds ties


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_refusals_raise_value_error(dtype):
    rng = np.random.default_rng(7)
    prob, mask = ppo.scops_like(rng, 2, 32)
    mask[:] = 1
    u = _uniforms(rng, 2, 4, 32, dtype)
    zero = prob.copy()
    zero[1, :, :, 3] = 0
    with pytest.raises(ValueError, match="image 1, channel 3: a NaN"):
        _call(zero, mask, u, CH, NS, dtype)
    few = prob.copy()
    few[0, :, :, 2] = 0
    few[0, 5, :14, 2] = 0.5                      # 14 positive pixels, 15 drawn
    with pytest.raises(ValueError, match="image 0, channel 2: fewer"):
        _call(few, mask, u, CH, NS, dtype)
    nan = prob.copy()
    nan[1, 3, 3, 4] = np.nan
    with pytest.raises(ValueError, match="image 1, channel 4"):
        _call(nan, mask, u, CH, NS, dtype)
    neg = prob.copy()
    neg[0, 9, 9, 1] = -0.25
    with pytest.raises(ValueError, match="image 0, channel 1"):
        _call(neg, mask, u, CH, NS, dtype)
    check(prob, mask, u, CH, NS, dtype)           # the inputs themselves are accepted


GUARD = 64


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_guard_bands_round_every_output_and_two_launches(dtype):
    rng = np.random.default_rng(8)
    B, S, K = 3, 64, 4
    prob, mask = ppo.scops_like(rng, B, S)
    u = _uniforms(rng, B, K, S, dtype)
    t = DTYPES[dtype]
    p = torch.as_tensor(prob, device=DEV).to(t).contiguous()
    m = torch.as_tensor(mask, device=DEV).to(t).contiguous()
    uu = torch.as_tensor(u, device=DEV).contiguous()
    sentinel = -12345.0

    def guarded(n, dt):
        return torch.full((2 * GUARD + n,), sentinel, device=DEV, dtype=dt)
    cen = guarded(B * K * 2, t)
    pts = [guarded(B * n * 2, t) for n in NS]
    drn = [guarded(B * ppo.n_draws(n), torch.int32) for n in NS]
    st = guarded(B * K, torch.int32)
    lib = _lib.load()
    args = lambda: (p.data_ptr(), m.data_ptr(), uu.data_ptr(), B, S, 5, K, (ctypes.c_int32 * K)(*CH), (ctypes.c_int32 * K)(*NS),
                    0 if dtype is np.float32 else 1, None, cen[GUARD:].data_ptr(),
                    (ctypes.c_void_p * K)(*[q[GUARD:].data_ptr() for q in pts]),
                    (ctypes.c_void_p * K)(*[d[GUARD:].data_ptr() for d in drn]), st[GUARD:].data_ptr(), _stream_ptr(DEV))
    torch.cuda.synchronize()
    before = lib.umr_launch_count()
    assert lib.umr_part_points(*args()) == 0
    assert lib.umr_launch_count() - before == 2
    torch.cuda.synchronize()
    for buf, n in [(cen, B * K * 2), (st, B * K)] + list(zip(pts, [B * n * 2 for n in NS])) + \
            list(zip(drn, [B * ppo.n_draws(n) for n in NS])):
        assert (buf[:GUARD] == sentinel).all() and (buf[GUARD + n:] == sentinel).all()
        assert not (buf[GUARD:GUARD + n] == sentinel).any()
    assert (st[GUARD:GUARD + B * K] == 0).all()
    centers = cen[GUARD:GUARD + B * K * 2].reshape(B, K, 2).cpu().numpy()
    dr_ref, pts_ref = ppo.part_points(prob, mask, u, CH, NS, dtype, centers)
    for k, n in enumerate(NS):
        np.testing.assert_array_equal(pts[k][GUARD:GUARD + B * n * 2].reshape(B, n, 2).cpu().numpy(), pts_ref[k])
        np.testing.assert_array_equal(drn[k][GUARD:GUARD + B * ppo.n_draws(n)].reshape(B, -1).cpu().numpy(), dr_ref[k])


def test_launch_count_per_call():
    rng = np.random.default_rng(9)
    prob, mask = ppo.scops_like(rng, 2, 64)
    p, m = torch.as_tensor(prob, device=DEV), torch.as_tensor(mask, device=DEV)
    image.part_points(p, m)
    lib = _lib.load()
    before = lib.umr_launch_count()
    image.part_points(p, m)
    assert lib.umr_launch_count() - before == 2


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_bitwise_repeatable_and_a_seeded_generator_reproduces_a_call(dtype):
    rng = np.random.default_rng(10)
    prob, mask = ppo.scops_like(rng, 4, 256)
    p, m = torch.as_tensor(prob, device=DEV).to(dtype), torch.as_tensor(mask, device=DEV)
    outs = []
    for _ in range(2):
        g = torch.Generator(device=DEV).manual_seed(1234)
        outs.append(image.part_points(p, m, generator=g))
    for a, b in zip([outs[0][0], *outs[0][1]], [outs[1][0], *outs[1][1]]):
        assert torch.equal(a, b)
    other = image.part_points(p, m, generator=torch.Generator(device=DEV).manual_seed(99))
    assert torch.equal(other[0], outs[0][0]) and not all(torch.equal(a, b) for a, b in zip(other[1], outs[0][1]))
    # the points are what the restatement keeps from those uniforms
    g = torch.Generator(device=DEV).manual_seed(1234)
    u = torch.rand(4, 4, 256 * 256, generator=g, device=DEV, dtype=dtype).cpu().numpy()
    dt = np.float32 if dtype == torch.float32 else np.float64
    _, pts_ref = ppo.part_points(prob, mask, u, CH, NS, dt, outs[0][0].cpu().numpy())
    for k in range(4):
        np.testing.assert_array_equal(outs[0][1][k].cpu().numpy(), pts_ref[k])


def test_single_image_wrappers():
    rng = np.random.default_rng(11)
    prob, mask = ppo.scops_like(rng, 1, 64)
    p, m = torch.as_tensor(prob[0], device=DEV), torch.as_tensor(mask[0], device=DEV)
    for ch in CH:
        c = image.prob2center(p, m, ch=ch)
        assert c.shape == (2,) and (np.abs(c.cpu().numpy() - ppo.centre(prob[0], mask[0], ch))
                                    <= ppo.centre_bound(prob[0], mask[0], ch, np.float32)).all()
    # sample_prob keeps the points nearest the centre it is given
    c = torch.tensor([0.3, -0.6], device=DEV)
    pts = image.sample_prob(p, m, c, num_samples=30, ch=3, generator=torch.Generator(device=DEV).manual_seed(5))
    u = torch.rand(1, 1, 64 * 64, generator=torch.Generator(device=DEV).manual_seed(5), device=DEV).cpu().numpy()
    drawn = ppo.draw(prob[0], mask[0], u[0, 0], 3, 30, np.float32)
    np.testing.assert_array_equal(pts.cpu().numpy(), ppo.nearest(drawn, c.cpu().numpy(), 64, 30, np.float32))


def test_kernel_draw_has_the_law_of_multinomial_without_replacement():
    # 3 x 3 map, m = 3 (n = 2): the subset frequencies of 40000 images against the exact law
    import scipy.stats
    rng = np.random.default_rng(12)
    q = rng.uniform(0.05, 1.0, 9)
    q[4] = 0
    B = 40000
    prob = np.broadcast_to(q.reshape(1, 3, 3, 1), (B, 3, 3, 2)).astype(np.float32).copy()
    mask = np.ones((B, 3, 3))
    _, _, drawn = _call(prob, mask, _uniforms(rng, B, 1, 3, np.float32), (1,), (2,), np.float32)
    exact = ppo.subset_probabilities(q.astype(np.float32).astype(np.float64), 3)
    subsets = sorted(exact)
    index = {s: j for j, s in enumerate(subsets)}
    observed = np.bincount([index[tuple(r)] for r in drawn[0].tolist()], minlength=len(subsets))
    expected = np.array([exact[s] for s in subsets]) * B
    assert scipy.stats.chisquare(observed, expected * observed.sum() / expected.sum()).pvalue > 1e-3


def test_corr_loss_step_on_part_points_equals_the_restatements_points():
    rng = np.random.default_rng(13)
    B, S = 4, 256
    prob, mask = ppo.scops_like(rng, B, S)
    u = _uniforms(rng, B, 4, S, np.float32)
    centers, points, _ = _call(prob, mask, u, CH, NS, np.float32)
    _, pts_ref = ppo.part_points(prob, mask, u, CH, NS, np.float32, centers)
    v, _ = synth.icosphere(3)
    parts = [torch.from_numpy(p) for p in synth.part_vertex_sets(rng, v.shape[0], sizes=(20, 40, 20, 40))]
    corr = loss_utils.CorrLossChamfer(None, S, part_vertices=parts)
    verts = torch.from_numpy(synth.bird_like(v, rng, B)).to(DEV)
    cams = torch.from_numpy(synth.cameras(rng, B)).to(DEV)

    def step(pts):
        head, neck, back, belly = [torch.as_tensor(p, device=DEV) for p in pts]
        vv = verts.clone().requires_grad_(True)
        loss, _ = corr(head, belly, neck, back, vv, cams)      # avg=True: (mean loss, projected vertices)
        loss.backward()
        return loss.detach(), vv.grad
    l1, g1 = step(points)
    l2, g2 = step(pts_ref)
    assert torch.isfinite(l1) and torch.equal(l1, l2) and torch.equal(g1, g2)
