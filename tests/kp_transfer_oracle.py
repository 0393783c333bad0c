"""CPU oracle of the keypoint transfer (experiments/test_kp.py:125-193, utils/kp_utils.py:13-69), restated in numpy float32
with the sampling convention written out: grid_sample(bilinear, zeros padding, align_corners=True), the torch-1.1
semantics the texture flow was trained with.  Every product and sum is one float32 operation in the order the kernels
of csrc/kp_transfer.cu use (nw, ne, sw, se corners; T^2 samples summed in order, then divided by T^2; k_chamfer_nn's
distance (|q|^2 + |k|^2) - 2 q.k), so the two agree bit for bit; each decision also reports its margin over the
runner-up, so a test can tell a real disagreement from a near-tie that a different summation order would flip."""
import numpy as np
import torch

f32 = np.float32
HEATMAP_SCALE = f32(256)   # test_kp.py:146, whatever the image size


def gauss_table(sigma):
    """draw_labelmap's unnormalised Gaussian [(6 sigma + 1)^2] (kp_utils.py:53-58): float64 exp, then float32."""
    n = 6 * sigma + 1
    x = np.arange(0, n, 1, float)
    y = x[:, np.newaxis]
    c = n // 2
    return np.exp(- ((x - c) ** 2 + (y - c) ** 2) / (2 * sigma ** 2)).astype(f32)


def grid_table(S):
    """The identity grid's coordinate table: torch.linspace(-1, 1, S), as torch-1.1 affine_grid yields it."""
    return torch.linspace(-1, 1, S, dtype=torch.float32).numpy()


def heat_center(kp):
    """(kp + 1) / 2 * 256 in float32."""
    kp = np.asarray(kp, f32)
    return ((kp + f32(1)) / f32(2)) * HEATMAP_SCALE


def heatmap(kp, sigma, S):
    """draw_labelmap(zeros(S, S), pt, sigma) with pt = (kp + 1) / 2 * 256, restated: window corners truncated toward
    zero like Python int(); an all-zero map when the window misses the image (or the keypoint is not finite).  Where
    float32 rounding makes br - ul = 6 sigma + 2 (the reference's slice assignment fails there), the window is clamped
    to the table: br = min(br, ul + 6 sigma + 1)."""
    pt = heat_center(kp)
    img = np.zeros((S, S), f32)
    a = pt - f32(3 * sigma)
    b = (pt + f32(3 * sigma)) + f32(1)
    if not (np.all(a < f32(S)) and np.all(b > f32(-1))):
        return img
    ul = [int(a[0]), int(a[1])]
    n = 6 * sigma + 1
    br = [min(int(b[0]), ul[0] + n), min(int(b[1]), ul[1] + n)]
    g = gauss_table(sigma).reshape(n, n)
    g_x = max(0, -ul[0]), min(br[0], S) - ul[0]
    g_y = max(0, -ul[1]), min(br[1], S) - ul[1]
    img_x = max(0, ul[0]), min(br[0], S)
    img_y = max(0, ul[1]), min(br[1], S)
    img[img_y[0]:img_y[1], img_x[0]:img_x[1]] = g[g_y[0]:g_y[1], g_x[0]:g_x[1]]
    return img


def sample(images, flow):
    """images [C,H,W] float32, flow [N,2] (x, y) in [-1, 1] -> [N,C]: bilinear, zeros padding, align_corners=True, in the
    sampler's float32 arithmetic."""
    images = np.asarray(images, f32)
    C, H, W = images.shape
    flow = np.asarray(flow, f32)
    ix = ((flow[:, 0] + f32(1)) / f32(2)) * f32(W - 1)
    iy = ((flow[:, 1] + f32(1)) / f32(2)) * f32(H - 1)
    x0 = np.floor(ix).astype(np.int64)
    y0 = np.floor(iy).astype(np.int64)
    x1, y1 = x0 + 1, y0 + 1
    fx0, fy0, fx1, fy1 = x0.astype(f32), y0.astype(f32), x1.astype(f32), y1.astype(f32)
    corners = [(x0, y0, (fx1 - ix) * (fy1 - iy)), (x1, y0, (ix - fx0) * (fy1 - iy)),
               (x0, y1, (fx1 - ix) * (iy - fy0)), (x1, y1, (ix - fx0) * (iy - fy0))]
    acc = np.zeros((flow.shape[0], C), f32)
    for x, y, w in corners:
        ok = (x >= 0) & (x < W) & (y >= 0) & (y < H)
        v = images[:, np.clip(y, 0, H - 1), np.clip(x, 0, W - 1)].T
        acc = np.where(ok[:, None], acc + v * w[:, None], acc)
    return acc


def face_means(vals):
    """vals [F,T2,C] -> [F,C]: the T^2 samples summed in order, then divided by T^2."""
    s = np.zeros((vals.shape[0], vals.shape[2]), f32)
    for t in range(vals.shape[1]):
        s = s + vals[:, t]
    return s / f32(vals.shape[1])


def _first_max(v):
    """(index, margin over the runner-up) of torch.max's choice: NaN first, then the largest, lowest index on ties."""
    nan = np.isnan(v)
    if nan.any():
        return int(np.argmax(nan)), np.inf
    i = int(np.argmax(v))
    rest = np.delete(v, i)
    return i, (float(v[i]) - float(rest.max())) if rest.size else np.inf


def transfer_flow(kps, flow_src, flow_tgt, sigma, S):
    """kps [P,K,2], flows [P,F,T2,2] -> (out [P,K,2], face [P,K], margin [P,K]) of test_kp.py:125-158."""
    kps = np.asarray(kps, f32)
    flow_src, flow_tgt = np.asarray(flow_src, f32), np.asarray(flow_tgt, f32)
    P, K = kps.shape[:2]
    F, T2 = flow_src.shape[1:3]
    grid = grid_table(S)
    gx = np.broadcast_to(grid[None, :], (S, S))
    gy = np.broadcast_to(grid[:, None], (S, S))
    out = np.zeros((P, K, 2), f32)
    face = np.zeros((P, K), np.int64)
    margin = np.zeros((P, K))
    for p in range(P):
        heat = np.stack([heatmap(kps[p, k], sigma, S) for k in range(K)])
        means = face_means(sample(heat, flow_src[p].reshape(-1, 2)).reshape(F, T2, K))   # [F,K]
        for k in range(K):
            face[p, k], margin[p, k] = _first_max(means[:, k])
        pf = face_means(sample(np.stack([gx, gy]), flow_tgt[p].reshape(-1, 2)).reshape(F, T2, 2))   # p2face [F,2]
        out[p] = pf[face[p]]
    return out, face, margin


def p2face(flow_tgt, S):
    """The identity grid sampled at every face's target flow, T^2 mean: flow_tgt [F,T2,2] -> [F,2]."""
    grid = grid_table(S)
    img = np.stack([np.broadcast_to(grid[None, :], (S, S)), np.broadcast_to(grid[:, None], (S, S))])
    F, T2 = flow_tgt.shape[:2]
    return face_means(sample(img, np.asarray(flow_tgt, f32).reshape(-1, 2)).reshape(F, T2, 2))


def chamfer_dist(q, keys):
    """k_chamfer_nn's distance of one 2-D query to keys [N,2], float32, defined order."""
    q = np.asarray(q, f32)
    keys = np.asarray(keys, f32)
    qq = q[0] * q[0] + q[1] * q[1]
    kk = keys[:, 0] * keys[:, 0] + keys[:, 1] * keys[:, 1]
    zz = q[0] * keys[:, 0] + q[1] * keys[:, 1]
    return (qq + kk) - f32(2) * zz


def _first_min(d):
    """(index, margin) of the nearest key: lowest index on ties, NaN and +inf never chosen; (None, inf) if none is."""
    d = np.where(np.isnan(d), np.inf, d)
    if d.size == 0 or not np.any(d < np.inf):
        return None, np.inf
    i = int(np.argmin(d))
    rest = np.delete(d, i)
    return i, (float(rest.min()) - float(d[i])) if rest.size else np.inf


def transfer_cam(kps, proj_src, proj_tgt, mask, S):
    """kps [P,K,2], projections [P,V,2], mask [P,S,S] -> (out [P,K,2], margin [P,K]) of test_kp.py:160-193: the smaller of
    the two decisions' margins; NaN where the reference fails (empty mask)."""
    kps = np.asarray(kps, f32)
    P, K = kps.shape[:2]
    grid = grid_table(S)
    out = np.full((P, K, 2), np.nan, f32)
    margin = np.full((P, K), np.inf)
    for p in range(P):
        fg = np.flatnonzero(np.asarray(mask[p]).reshape(-1) != 0)
        coords = np.stack([grid[fg % S], grid[fg // S]], axis=1)
        for k in range(K):
            v, m1 = _first_min(chamfer_dist(kps[p, k], proj_src[p]))
            if v is None:
                continue
            j, m2 = _first_min(chamfer_dist(proj_tgt[p, v], coords))
            if j is None:
                continue
            out[p, k] = coords[j]
            margin[p, k] = min(m1, m2)
    return out, margin


def wide_window_keypoints(sigma, S):
    """float32 keypoint coordinates in [-1, 1] whose heat-map window comes out 6 sigma + 2 wide before the clamp (float32
    pt + 3 sigma rounds up to a power of two, so br = int((pt + 3 sigma) + 1) is one too large) and lies in the image.
    The crossings are searched a few hundred float32 steps around pt + 3 sigma = 2^e."""
    out = []
    for e in range(1, 16):
        c = 2.0 ** e - 3 * sigma
        if not 0 <= c < S:
            continue
        v = f32(c / 128.0 - 1.0)
        for _ in range(64):
            v = np.nextafter(v, f32(-2))
        for _ in range(128):
            pt = heat_center(v)
            a, b = pt - f32(3 * sigma), (pt + f32(3 * sigma)) + f32(1)
            if a < f32(S) and b > f32(-1) and int(b) - int(a) == 6 * sigma + 2 and -1 <= v <= 1:
                out.append(f32(v))
            v = np.nextafter(v, f32(2))
    return out
