"""Numpy restatement of the part centres and part points of DESIGN.md §17 (utils/image.py:143-206 `prob2center` /
`sample_prob`, data/base.py:155-166), the oracle of tests/test_part_points_{cpu,gpu}.py.

`centre` is the contract in float64.  `keys`, `draw` and `nearest` take the kernels' precision (`dtype`) and perform the
same IEEE operations they do, one rounding each, so the drawn pixel sets and the kept points are compared bit for bit:
  key   = log(u) / q for q = p * mask > 0 (log in float64, rounded once to dtype), q <= 0 never drawn;
  draw  = the m = floor(1.5 n) largest keys, ties to the lower pixel index, as ascending pixel indices;
  point = ((x / 256) * 2 - 1, (y / 256) * 2 - 1) of pixel k = y * S + x;
  keep  = the n drawn pixels of least (dx * dx + dy * dy, pixel index) from the given centre.
"""
import itertools

import numpy as np


def n_draws(n):
    return int(1.5 * n)


def scops_like(rng, B, S, C=5, ring=True):
    """SCOPS-like inputs: part_prob [B,S,S,C] float32 (softmax over C of a few Gaussian blobs per channel), mask [B,S,S]
    float64, an ellipse with a soft rim, as cv2.resize leaves the loader's mask."""
    yy, xx = np.mgrid[0:S, 0:S] / S
    logits = np.zeros((B, S, S, C))
    for b in range(B):
        for c in range(C):
            for _ in range(3):
                cx, cy, w = rng.uniform(0.2, 0.8), rng.uniform(0.2, 0.8), rng.uniform(0.05, 0.2)
                logits[b, :, :, c] += 3 * np.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / (2 * w * w))
    logits += 0.3 * rng.standard_normal(logits.shape)
    e = np.exp(logits - logits.max(-1, keepdims=True))
    prob = (e / e.sum(-1, keepdims=True)).astype(np.float32)
    mask = np.zeros((B, S, S))
    for b in range(B):
        r = ((xx - rng.uniform(0.4, 0.6)) / rng.uniform(0.25, 0.4)) ** 2 + ((yy - rng.uniform(0.4, 0.6)) / rng.uniform(0.25, 0.4)) ** 2
        mask[b] = np.clip((1.1 - r) * 4, 0, 1) if ring else (r <= 1)
    return prob, mask


def coordinate_maps(S):
    """get_coordinate_tensors (utils/image.py:143-150) for a square map, in float64: x_map[i, j] = j / S * 2 - 1."""
    x_map = np.tile(np.arange(S), (S, 1)) / S * 2 - 1.0
    return x_map, x_map.T.copy()


def centre(prob, mask, ch):
    """prob2center in float64: prob [S,S,C], mask [S,S] -> (x, y)."""
    q = prob[:, :, ch].astype(np.float64) * mask.astype(np.float64)
    pdf = q / q.sum()
    x_map, y_map = coordinate_maps(prob.shape[0])
    return np.array([(pdf * x_map).sum(), (pdf * y_map).sum()])


def centre_bound(prob, mask, ch, dtype, threads=256):
    """A bound on |kernel centre - centre()| per coordinate: gamma_k * sum |pdf * coordinate|, k = 2 (L + 8) + 4 for
    L = ceil(S^2 / threads) terms per thread and an 8-level tree in both sums (sum q, then sum pdf * coordinate), and one
    rounding each for q, pdf, the coordinate and the product."""
    q = prob[:, :, ch].astype(np.float64) * mask.astype(np.float64)
    pdf = q / q.sum()
    x_map, y_map = coordinate_maps(prob.shape[0])
    L = -(-prob.shape[0] ** 2 // threads)
    k = 2 * (L + 8) + 4
    u = np.finfo(dtype).eps / 2
    gamma = k * u / (1 - k * u)
    return gamma * np.array([np.abs(pdf * x_map).sum(), np.abs(pdf * y_map).sum()])


def keys(prob, mask, u, ch, dtype):
    """Flat keys [S*S] in dtype and the drawable pixels (q > 0)."""
    q = (prob[:, :, ch].astype(dtype) * mask.astype(dtype)).reshape(-1)
    valid = q > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        lg = np.log(np.asarray(u, np.float64).reshape(-1)).astype(dtype)
        key = np.where(valid, lg / np.where(valid, q, dtype(1)), -np.inf).astype(dtype)
    return key, valid


def draw(prob, mask, u, ch, n, dtype):
    """The m = floor(1.5 n) drawn pixel indices, ascending."""
    key, valid = keys(prob, mask, u, ch, dtype)
    cand = np.nonzero(valid)[0]
    order = np.lexsort((cand, -key[cand].astype(np.float64)))
    return np.sort(cand[order[:n_draws(n)]])


def coords(idx, S, dtype):
    idx = np.asarray(idx)
    x, y = (idx % S).astype(dtype), (idx // S).astype(dtype)
    two, one, scale = dtype(2), dtype(1), dtype(256)
    return np.stack([(x / scale) * two - one, (y / scale) * two - one], axis=-1)


def nearest(drawn, c, S, n, dtype):
    """The n points of `drawn` (pixel indices, any order) nearest the centre c, ascending (distance, pixel index)."""
    drawn = np.asarray(drawn)
    xy = coords(drawn, S, dtype)
    c = np.asarray(c).astype(dtype)
    dx, dy = xy[:, 0] - c[0], xy[:, 1] - c[1]
    d = dx * dx + dy * dy
    order = np.lexsort((drawn, d))
    return xy[order[:n]]


def part_points(prob, mask, u, channels, num_samples, dtype, centres):
    """The batched call on given uniforms u [B,K,S*S] and centres [B,K,2] -> (drawn tuple of [B,m], points tuple of
    [B,n,2])."""
    B, S = prob.shape[:2]
    drawn, points = [], []
    for k, (ch, n) in enumerate(zip(channels, num_samples)):
        dr = np.stack([draw(prob[b], mask[b], u[b, k], ch, n, dtype) for b in range(B)])
        drawn.append(dr)
        points.append(np.stack([nearest(dr[b], centres[b, k], S, n, dtype) for b in range(B)]))
    return tuple(drawn), tuple(points)


def subset_probabilities(pdf, m):
    """Exact probability of each m-subset (sorted tuple of indices) under sequential drawing without replacement, the law
    of torch.multinomial(pdf, m, replacement=False)."""
    pdf = np.asarray(pdf, np.float64) / np.sum(pdf)
    out = {}
    for seq in itertools.permutations(range(len(pdf)), m):
        p, left = 1.0, 1.0
        for i in seq:
            if pdf[i] == 0:
                p = 0.0
                break
            p *= pdf[i] / left
            left -= pdf[i]
        if p > 0:
            key = tuple(sorted(seq))
            out[key] = out.get(key, 0.0) + p
    return out

