"""Keypoint transfer kernels (csrc/kp_transfer.cu) against the CPU oracle (tests/kp_transfer_oracle.py) across their
accepted input range, and `sample_textures` with more than 4 channels against grid_sample(align_corners=True).

The oracle restates the kernels' float32 operation order, so outputs agree bit for bit.  A decision whose margin over
the runner-up is at most BOUND but not zero (a near-tie that another summation order could flip) is reported and not
required to agree; exact ties (margin 0) must, by the lowest index."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import kp_transfer_oracle as ko
from umr_b200 import _lib
from umr_b200.nnutils import geom_utils, kp_transfer, smr
from umr_b200.raster import _stream_ptr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
BOUND = 1e-6   # float32: a few ulps of the heat-map means (<= 1) and of the squared distances (<= 8)


def _flow_scene(P, K, F, T, S, sigma, seed):
    """Faces whose T^2 flow points cluster around a centre in [-1.1, 1.1] (some past the border), keypoints in
    [-1.05, 1.05] plus one on the border and one whose heat map is all zero, and a duplicated face (exact ties)."""
    rng = np.random.default_rng(seed)
    T2 = T * T
    centre = rng.uniform(-1.1, 1.1, (P, F, 1, 2))
    fs = (centre + rng.uniform(-0.04, 0.04, (P, F, T2, 2))).astype(np.float32)
    ft = (rng.uniform(-1.1, 1.1, (P, F, 1, 2)) + rng.uniform(-0.04, 0.04, (P, F, T2, 2))).astype(np.float32)
    if F >= 4:
        fs[:, F - 1] = fs[:, 1]
    kps = rng.uniform(-1.05, 1.05, (P, K, 2)).astype(np.float32)
    if F >= 4:
        kps[:, 0] = fs[:, 1].mean(axis=1)     # on the duplicated face: an exact tie between faces 1 and F-1
    if K >= 3:
        kps[:, 1] = [1.0, -1.0]                # on the border
        kps[:, 2] = [2.5, 0.0]                 # window outside the image: all-zero heat map -> face 0
    wide = ko.wide_window_keypoints(sigma, S)
    if K >= 5 and wide:                        # windows one pixel wider than the table before the clamp
        kps[:, 3] = [wide[0], wide[-1]]
        kps[:, 4, 0] = wide[len(wide) // 2]
        if F >= 3:
            fs[:, 2] = heat_flow(kps[:, 3], T2, rng)   # a face on that keypoint, so its window decides the choice
    return kps, fs, ft


def heat_flow(kp, T2, rng):
    """[P,T2,2] flow points within a few heat-map pixels of the keypoints kp [P,2]."""
    return (kp[:, None, :] + rng.uniform(-0.06, 0.06, (kp.shape[0], T2, 2))).astype(np.float32)


def _soft_masks(P, S, seed):
    """Soft ellipses with a tail of tiny non-zero alphas, plus an empty, a one-pixel and a full mask."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:S, 0:S] / (S - 1) * 2 - 1
    m = np.zeros((P, S, S), np.float32)
    for p in range(P):
        cx, cy, r = rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), rng.uniform(0.2, 0.6)
        d = np.sqrt((x - cx) ** 2 + (y - cy) ** 2) - r
        m[p] = np.where(d < 0, 1.0, np.where(d < 0.1, np.exp(-d * 200), 0.0)).astype(np.float32)
    if P >= 4:
        m[1] = 0
        m[2] = 0
        m[2, S // 3, S // 5] = 1e-20
        m[3] = 0.5
    return m


def _cam_scene(P, K, V, S, seed):
    rng = np.random.default_rng(seed)
    ps = rng.uniform(-0.9, 0.9, (P, V, 2)).astype(np.float32)
    pt = rng.uniform(-0.9, 0.9, (P, V, 2)).astype(np.float32)
    if V >= 2:
        ps[:, V - 1] = ps[:, 0]                  # duplicated vertex: exact tie, lowest index
    kps = rng.uniform(-1.0, 1.0, (P, K, 2)).astype(np.float32)
    if K >= 2:
        kps[:, 1] = ps[:, 0]
    return kps, ps, pt, _soft_masks(P, S, seed + 1)


def _cuda(*a):
    return [torch.from_numpy(np.ascontiguousarray(x)).to(DEV) for x in a]


def _cam_raw(kps, ps, pt, mask):
    """umr_kp_transfer_cam on given projections (the kernel without the projection step)."""
    k, s, t, m = _cuda(kps, ps, pt, mask)
    P, K = kps.shape[:2]
    S = mask.shape[1]
    grid = kp_transfer._grid(S, DEV)
    out = torch.empty(P, K, 2, device=DEV)
    p = lambda x: ctypes.c_void_p(x.data_ptr())
    _lib.check(_lib.load().umr_kp_transfer_cam(p(k), p(s), p(t), p(m), p(grid), p(out), P, K, ps.shape[1], S,
                                               _stream_ptr(DEV)), "cam")
    return out.cpu().numpy()


def _agree(got, want, margin, what):
    ok = (margin > BOUND) | (margin == 0)
    same = np.all((got == want) | (np.isnan(got) & np.isnan(want)), axis=-1)
    bad = ok & ~same
    assert not bad.any(), "%s: %d of %d (pair, keypoint) differ, first %s: got %s want %s (margin %g)" % (
        what, bad.sum(), bad.size, np.argwhere(bad)[0], got[bad][0], want[bad][0], margin[bad][0])
    return int((~ok & ~same).sum())


FLOW_BASE = dict(P=7, K=15, F=1280, T=6, S=256, sigma=3)
FLOW_RANGE = ([dict(S=s) for s in (64, 255, 256, 257)] + [dict(sigma=s) for s in (1, 3, 7, 18)]
              + [dict(K=k) for k in (1, 15, 33)] + [dict(F=f) for f in (1, 1280, 5120)] + [dict(T=t) for t in (1, 6)]
              + [dict(P=1), dict(P=7), dict(P=1000, F=64, T=2)])


@pytest.mark.parametrize("over", FLOW_RANGE, ids=lambda d: "-".join("%s%d" % kv for kv in d.items()))
def test_flow_matches_oracle(over):
    a = dict(FLOW_BASE, **over)
    kps, fs, ft = _flow_scene(a["P"], a["K"], a["F"], a["T"], a["S"], a["sigma"], seed=sum(a.values()))
    want, face, margin = ko.transfer_flow(kps, fs, ft, a["sigma"], a["S"])
    k, s, t = _cuda(kps, fs, ft)
    got = kp_transfer.transfer_flow(k, s, t, sigma=a["sigma"], image_size=a["S"]).cpu().numpy()
    near = _agree(got, want, margin, "flow %s" % a)
    if a["K"] >= 3:
        assert (face[:, 2] == 0).all() and (got[:, 2] == want[:, 2]).all()   # all-zero heat map -> face 0
    print("flow %s: %d near-ties differ, min margin %g" % (a, near, margin[margin > 0].min() if (margin > 0).any() else 0))


def test_flow_wide_windows_are_exercised_and_sigma_past_the_table_is_refused():
    kps, fs, ft = _flow_scene(3, 15, 64, 3, 256, 3, seed=6)
    pt = ko.heat_center(kps[0, 3])
    assert int((pt[0] + np.float32(9)) + np.float32(1)) - int(pt[0] - np.float32(9)) == 20
    k, s, t = _cuda(kps, fs, ft)
    kp_transfer.transfer_flow(k, s, t, sigma=18)
    with pytest.raises(RuntimeError, match="umr_kp_transfer_flow"):
        kp_transfer.transfer_flow(k, s, t, sigma=19)


def test_flow_takes_five_dimensional_flows_and_visibility_columns():
    kps, fs, ft = _flow_scene(3, 15, 64, 3, 256, 3, seed=5)
    k3 = np.concatenate([kps, np.ones((3, 15, 1), np.float32)], axis=2)
    k, s, t, k3 = _cuda(kps, fs, ft, k3)
    a = kp_transfer.transfer_flow(k, s, t)
    b = kp_transfer.transfer_flow(k3, s.view(3, 64, 3, 3, 2), t.view(3, 64, 3, 3, 2))
    assert torch.equal(a, b) and not a.requires_grad


CAM_BASE = dict(P=7, K=15, V=642, S=256)
CAM_RANGE = ([dict(S=s) for s in (64, 255, 256, 257)] + [dict(K=k) for k in (1, 15, 33)] + [dict(V=v) for v in (1, 642)]
             + [dict(P=1), dict(P=7), dict(P=1000, S=64)])


@pytest.mark.parametrize("over", CAM_RANGE, ids=lambda d: "-".join("%s%d" % kv for kv in d.items()))
def test_cam_matches_oracle(over):
    a = dict(CAM_BASE, **over)
    kps, ps, pt, mask = _cam_scene(a["P"], a["K"], a["V"], a["S"], seed=sum(a.values()))
    want, margin = ko.transfer_cam(kps, ps, pt, mask, a["S"])
    got = _cam_raw(kps, ps, pt, mask)
    _agree(got, want, margin, "cam %s" % a)
    if a["P"] >= 4:
        assert np.isnan(got[1]).all()                        # empty mask
        g = ko.grid_table(a["S"])
        assert (got[2] == [g[a["S"] // 5], g[a["S"] // 3]]).all()   # the one foreground pixel, however faint


@pytest.mark.parametrize("S", [64, 255, 256, 257])
def test_cam_exact_pixel_ties_take_the_lowest_flat_index(S):
    """Two foreground pixels mirrored about 0 (linspace is symmetric, so their distances to a projection on the axis are
    bitwise equal): in one row (pair 0) and in one column (pair 1); the lower flat index wins, as `nonzero` orders it."""
    g = ko.grid_table(S)
    r, c = S // 3, S // 5
    mask = np.zeros((2, S, S), np.float32)
    mask[0, r, c] = mask[0, r, S - 1 - c] = 0.3
    mask[1, c, r] = mask[1, S - 1 - c, r] = 1.0
    ps = np.zeros((2, 1, 2), np.float32)
    pt = np.array([[[0.0, g[r]]], [[g[r], 0.0]]], np.float32)
    kps = np.zeros((2, 3, 2), np.float32)
    want, margin = ko.transfer_cam(kps, ps, pt, mask, S)
    assert (margin == 0).all()
    got = _cam_raw(kps, ps, pt, mask)
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(got[0], np.tile([g[c], g[r]], (3, 1)))
    np.testing.assert_array_equal(got[1], np.tile([g[r], g[c]], (3, 1)))


def test_cam_through_the_renderer_projection():
    P, K, V, S = 5, 15, 642, 128
    rng = np.random.default_rng(9)
    verts = torch.from_numpy(rng.uniform(-0.6, 0.6, (1, V, 3)).astype(np.float32)).to(DEV)
    q = rng.normal(size=(2 * P, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    cams = np.concatenate([rng.uniform(0.8, 1.2, (2 * P, 1)), rng.uniform(-0.1, 0.1, (2 * P, 2)), q], axis=1)
    cams = torch.from_numpy(cams.astype(np.float32)).to(DEV)
    renderer = smr.SoftRenderer(S, "softmax")
    kps = torch.from_numpy(rng.uniform(-1, 1, (P, K, 3)).astype(np.float32)).to(DEV)
    mask = torch.from_numpy(_soft_masks(P, S, 3)).to(DEV)
    got = kp_transfer.transfer_cam(kps, verts, cams[:P], cams[P:], mask, renderer).cpu().numpy()
    ps = renderer.project_points(verts.expand(P, -1, -1), cams[:P]).cpu().numpy()
    pt = renderer.project_points(verts.expand(P, -1, -1), cams[P:]).cpu().numpy()
    want, margin = ko.transfer_cam(kps[..., :2].cpu().numpy(), ps, pt, mask.cpu().numpy(), S)
    _agree(got, want, margin, "cam via project_points")


def _raw_flow(k, s, t, out_ptr, P, K, F, T2, S, sigma):
    gauss, grid = kp_transfer._gauss(sigma, DEV), kp_transfer._grid(S, DEV)
    p = lambda x: ctypes.c_void_p(x.data_ptr())
    return _lib.load().umr_kp_transfer_flow(p(k), p(s), p(t), p(gauss), p(grid), ctypes.c_void_p(out_ptr), P, K, F, T2, S,
                                            sigma, _stream_ptr(DEV))


def test_guard_values_around_the_outputs():
    P, K, F, T, S = 3, 15, 100, 3, 256
    kps, fs, ft = _flow_scene(P, K, F, T, S, 3, seed=11)
    k, s, t = _cuda(kps, fs, ft)
    buf = torch.full((P * K * 2 + 64,), 12345.0, device=DEV)
    assert _raw_flow(k, s, t, buf.data_ptr() + 32 * 4, P, K, F, T * T, S, 3) == 0
    _, ps, pt, mask = _cam_scene(P, K, 50, S, seed=12)
    cbuf = torch.full((P * K * 2 + 64,), 12345.0, device=DEV)
    c, sp, tp, m = _cuda(kps, ps, pt, mask)
    grid = kp_transfer._grid(S, DEV)
    p = lambda x: ctypes.c_void_p(x.data_ptr())
    assert _lib.load().umr_kp_transfer_cam(p(c), p(sp), p(tp), p(m), p(grid), ctypes.c_void_p(cbuf.data_ptr() + 32 * 4),
                                           P, K, 50, S, _stream_ptr(DEV)) == 0
    for b, want in ((buf, kp_transfer.transfer_flow(k, s, t)), (cbuf, torch.from_numpy(_cam_raw(kps, ps, pt, mask)).to(DEV))):
        h = b.cpu()
        assert (h[:32] == 12345.0).all() and (h[-32:] == 12345.0).all()
        assert torch.equal(h[32:-32].view(P, K, 2), want.cpu())


def test_bitwise_reproducible_and_one_launch_per_call():
    kps, fs, ft = _flow_scene(20, 15, 1280, 6, 256, 3, seed=13)
    k, s, t = _cuda(kps, fs, ft)
    _, ps, pt, mask = _cam_scene(20, 15, 642, 256, seed=14)
    verts = torch.rand(1, 642, 3, device=DEV) - 0.5
    cams = torch.tensor([[1.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]], device=DEV).repeat(20, 1)
    m = torch.from_numpy(mask).to(DEV)
    renderer = smr.SoftRenderer(256, "softmax")
    lib = _lib.load()
    runs = []
    for _ in range(2):
        n0 = lib.umr_launch_count()
        a = kp_transfer.transfer_flow(k, s, t)
        n1 = lib.umr_launch_count()
        b = kp_transfer.transfer_cam(k, verts, cams, cams, m, renderer)
        n2 = lib.umr_launch_count()
        assert (n1 - n0, n2 - n1) == (1, 1)
        runs.append((a, b))
    assert torch.equal(runs[0][0], runs[1][0])
    assert torch.equal(torch.nan_to_num(runs[0][1], 7.0), torch.nan_to_num(runs[1][1], 7.0))


def test_cuda_graph_capture():
    kps, fs, ft = _flow_scene(7, 15, 1280, 6, 256, 3, seed=15)
    k, s, t = _cuda(kps, fs, ft)
    m = torch.from_numpy(_soft_masks(7, 256, 16)).to(DEV)
    verts = torch.rand(1, 642, 3, device=DEV) - 0.5
    cams = torch.tensor([[1.0, 0.05, 0.0, 1.0, 0.0, 0.0, 0.0]], device=DEV).repeat(7, 1)
    renderer = smr.SoftRenderer(256, "softmax")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):   # warm-up: the tables are made (and cached) outside the capture
        eager = (kp_transfer.transfer_flow(k, s, t), kp_transfer.transfer_cam(k, verts, cams, cams, m, renderer))
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        captured = (kp_transfer.transfer_flow(k, s, t), kp_transfer.transfer_cam(k, verts, cams, cams, m, renderer))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured[0], eager[0])
    assert torch.equal(torch.nan_to_num(captured[1], 7.0), torch.nan_to_num(eager[1], 7.0))


# ---------------------------------------------------------------------------------------------------------------------
# sample_textures with C > 4 channels (channel groups of at most 4)
# ---------------------------------------------------------------------------------------------------------------------
def _reference(img, flow):
    """grid_sample(align_corners=True) in float64 with its gradients: img [B,C,H,W], flow [B,N,2]."""
    i = img.detach().double().requires_grad_(True)
    f = flow.detach().double().requires_grad_(True)
    out = Fn.grid_sample(i, f[:, None], mode="bilinear", padding_mode="zeros", align_corners=True)[:, :, 0].permute(0, 2, 1)
    return out, i, f


@pytest.mark.parametrize("C", [5, 8, 15])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("det", [False, True])
def test_sample_textures_many_channels(C, dtype, det):
    torch.manual_seed(C)
    B, H, W, F, T = 2, 37, 41, 60, 3
    img = torch.rand(B, C, H, W, device=DEV, dtype=dtype)
    tf = (torch.rand(B, F, T, T, 2, device=DEV, dtype=dtype) * 2.2 - 1.1)
    go = torch.randn(B, F, T, T, C, device=DEV, dtype=dtype)
    ref, ri, rf = _reference(img, tf.view(B, -1, 2))
    (ref * go.double().view(B, -1, C)).sum().backward()
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        i, f = img.clone().requires_grad_(True), tf.clone().requires_grad_(True)
        out = geom_utils.sample_textures(f, i)
        (out * go).sum().backward()
        # each group's output is the 4-channel sampler's; the flow gradient is the groups' summed in ascending order
        outs, parts = [], []
        for c0 in range(0, C, 4):
            fp = tf.clone().requires_grad_(True)
            o = geom_utils.sample_textures(fp, img[:, c0:c0 + 4].contiguous())
            (o * go[..., c0:c0 + 4]).sum().backward()
            outs.append(o.detach())
            parts.append(fp.grad)
    finally:
        torch.use_deterministic_algorithms(old)
    tol = 1e-12 if dtype == torch.float64 else 2e-5
    assert out.shape == (B, F, T, T, C) and out.dtype == dtype
    torch.testing.assert_close(out.double().view(B, -1, C), ref.detach(), rtol=tol, atol=tol)
    torch.testing.assert_close(i.grad.double(), ri.grad, rtol=tol, atol=tol * 10)
    torch.testing.assert_close(f.grad.double().view(B, -1, 2), rf.grad, rtol=tol * 10, atol=tol * 100)
    total = parts[0]
    for p in parts[1:]:
        total = total + p
    assert torch.equal(f.grad, total)
    assert torch.equal(out.detach(), torch.cat(outs, dim=-1))


def test_avg_uv_part_probabilities():
    """avg_uv.py:191 samples SCOPS's 5 part probabilities [1,5,256,256] at the texture flow."""
    torch.manual_seed(0)
    segs = torch.softmax(torch.randn(1, 5, 256, 256, device=DEV), dim=1)
    tf = torch.rand(1, 1280, 6, 6, 2, device=DEV) * 2 - 1
    out = geom_utils.sample_textures(tf, segs)
    ref, _, _ = _reference(segs, tf.view(1, -1, 2))
    assert out.shape == (1, 1280, 6, 6, 5)
    # float32 rounds the pixel coordinate (x + 1) / 2 * 255 to a few ulps of 256; probabilities change by at most 1 per
    # pixel, so the samples may differ from the float64 reference by that much
    torch.testing.assert_close(out.double().view(1, -1, 5), ref.detach(), rtol=0, atol=4 * 256 * 2.0 ** -24)
    torch.testing.assert_close(out.sum(-1), torch.ones_like(out[..., 0]), rtol=0, atol=1e-5)
