"""numpy restatement of the SCOPS semantic template (experiments/avg_uv.py:203-293, DESIGN.md §18), the oracle of
tests/test_semantic_template_{cpu,gpu}.py.

The UV samples are the sampler's torch-1.1 arithmetic in float32 with every operation rounded once, as the -fmad=false
kernels compute them, so sums over the same samples in the same order are bitwise the kernels'.  Distances are restated
in float64 over those samples; `dist_bound` is the rounding bound of the kernels' float32 summation order."""
import itertools
import math

import numpy as np

F32 = np.float32
U32 = 2.0 ** -24


def _corner_index(f):
    """(int) of a float32 floor as the device converts it: NaN -> 0, saturating at the int32 range."""
    with np.errstate(invalid="ignore"):
        return np.where(np.isnan(f), 0, np.clip(f, -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)


def bilinear(img, x, y):
    """img [C,H,W] float32 sampled at float32 coordinates x, y (any equal shapes) -> [C, *shape] float32: grid_sample,
    bilinear, zeros padding, align_corners=True, in losses.cuh's operation order (corners nw, ne, sw, se)."""
    C, H, W = img.shape
    x, y = np.asarray(x, F32), np.asarray(y, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        ix = ((x + F32(1)) / F32(2)) * F32(W - 1)
        iy = ((y + F32(1)) / F32(2)) * F32(H - 1)
        x0, y0 = _corner_index(np.floor(ix)), _corner_index(np.floor(iy))
        x1, y1 = x0 + 1, y0 + 1
        wx1, wx0 = x1.astype(F32) - ix, ix - x0.astype(F32)
        wy1, wy0 = y1.astype(F32) - iy, iy - y0.astype(F32)
        acc = np.zeros((C,) + x.shape, F32)
        for cx, cy, w in ((x0, y0, wx1 * wy1), (x1, y0, wx0 * wy1), (x0, y1, wx1 * wy0), (x1, y1, wx0 * wy0)):
            ok = (cx >= 0) & (cx < W) & (cy >= 0) & (cy < H)
            v = img[:, np.clip(cy, 0, H - 1), np.clip(cx, 0, W - 1)]
            acc = np.where(ok, acc + v * w.astype(F32), acc)
    return acc


def uv_parts(part_segs, uvimage_pred):
    """part_segs [B,C,S,S], uvimage_pred [B,2,H,W] -> [B,C,H,W] float32, grid_sample(part_segs, uv.permute(0,2,3,1))."""
    return np.stack([bilinear(part_segs[b], uvimage_pred[b, 0], uvimage_pred[b, 1]) for b in range(part_segs.shape[0])])


def distances(parts, exemplar):
    """float64 sum over (c, y, x) of (uv_parts[b] - exemplar)^2 over the float32 samples -> [B]."""
    d = parts.astype(np.float64) - exemplar.astype(np.float64)[None]
    return (d * d).reshape(parts.shape[0], -1).sum(axis=1)


def gamma(n):
    return n * U32 / (1 - n * U32)


def dist_bound(dist64, C, H, W):
    """|float32 kernel distance - float64 restatement| <= gamma(L + 3) * dist64: each term (v - e)^2 has relative error
    gamma(3), and each passes through at most L = 4 C (a thread's serial sum) + 8 (the 256-wide tree) + tiles (the
    serial finish over 1024-pixel tiles) additions of non-negative numbers."""
    tiles = -(-(H * W) // 1024)
    return gamma(4 * C + 8 + tiles + 3) * dist64


def select(dist, k):
    """The first k images in ascending (distance, index) order, NaN after every number."""
    d = np.asarray(dist, np.float64)
    key = np.where(np.isnan(d), np.inf, d)
    order = np.lexsort((np.arange(len(d)), np.isnan(d), key))
    return order[:k]


def accumulate(acc, parts, selected):
    """acc [C,H,W] float32 + (the selected maps summed in selection order), all float32."""
    s = np.zeros_like(acc)
    for b in selected:
        s = s + parts[b]
    return acc + s


def mean(acc, count):
    """avg_prob [H,W,C] = acc / count, float32."""
    return (acc / F32(count)).transpose(1, 2, 0).copy()


def average(batches, exemplar, k=5):
    """The averaging pass over [(part_segs, uvimage_pred)] -> (avg_prob [H,W,C], [(dist64, selected)] per batch), the
    selection taken from the float64 distances."""
    acc = np.zeros_like(exemplar)
    log = []
    for segs, uv in batches:
        parts = uv_parts(segs, uv)
        d = distances(parts, exemplar)
        sel = select(d, k)
        acc = accumulate(acc, parts, sel)
        log.append((d, sel))
    return mean(acc, k * len(batches)), log


def argmax(values, axis):
    """The first NaN if any, else the first largest: numpy's (and torch's) argmax."""
    return np.argmax(values, axis=axis)


def mode(labels, C):
    """Most frequent label in [0, C), ties to the smallest; -1 for no labels (`most_freq`'s first-max argmax)."""
    if len(labels) == 0:
        return -1
    return int(np.argmax(np.bincount(labels, minlength=C)))


def label(avg_prob, uv_sampler, faces, num_sym_faces, num_vertices=None):
    """The labelling pass: avg_prob [H,W,C], uv_sampler [F',T2,2], faces [F,3] -> dict of label_image [H,W] uint8,
    texel_labels [F,T2], face_labels [F], vertex_labels [V] and part_vertices (labels 1..C-1)."""
    H, W, C = avg_prob.shape
    Fs, T2, _ = uv_sampler.shape
    faces = np.asarray(faces, np.int64)
    V = int(faces.max()) + 1 if num_vertices is None else num_vertices
    img = np.ascontiguousarray(avg_prob.transpose(2, 0, 1))
    src = np.concatenate([np.arange(Fs), np.arange(Fs - num_sym_faces, Fs)])
    uv = uv_sampler[src]
    tex = bilinear(img, uv[..., 0], uv[..., 1])                       # [C,F,T2]
    texel = argmax(tex, axis=0)
    face = np.array([mode(t, C) for t in texel])
    incident = [set() for _ in range(V)]
    for f, tri in enumerate(faces):
        for v in tri:
            incident[v].add(f)
    vert = np.array([mode(face[sorted(s)], C) for s in incident])
    return dict(label_image=argmax(avg_prob, axis=2).astype(np.uint8), texel_labels=texel, face_labels=face,
                vertex_labels=vert, part_vertices=[np.nonzero(vert == p)[0] for p in range(1, C)])


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def spherical_coords(X):
    """utils/mesh.py:232-244 `get_spherical_coords`: points [N,3] -> (u, v) in [-1, 1]."""
    rad = np.linalg.norm(X, axis=1)
    theta = np.arccos(X[:, 2] / rad)
    phi = np.arctan2(X[:, 1], X[:, 0])
    return np.stack([((phi + np.pi) / (2 * np.pi)) * 2 - 1, (theta / np.pi) * 2 - 1], 1)


def uv_sampler(verts, faces, tex_size):
    """utils/mesh.py:247-272 `compute_uvsampler` -> [F,T*T,2] float32: the spherical coordinates of the T x T
    barycentric grid of every face.  T = 1 (which divides by zero there) takes each face's centroid."""
    if tex_size == 1:
        samples = verts[faces].mean(axis=1)[:, None, :]
    else:
        a = np.arange(tex_size, dtype=np.float64) / (tex_size - 1)
        coords = np.stack([p for p in itertools.product(a, a)])
        vs = verts[faces].astype(np.float64)
        v2, v0v2, v1v2 = vs[:, 2], vs[:, 0] - vs[:, 2], vs[:, 1] - vs[:, 2]
        samples = np.dstack([v0v2, v1v2]).dot(coords.T) + v2.reshape(-1, 3, 1)
        samples = np.transpose(samples, (0, 2, 1))
    uv = spherical_coords(samples.reshape(-1, 3))
    return uv.reshape(len(faces), tex_size * tex_size, 2).astype(F32)


def smooth_field(rng, shape_hw, n_modes=3, amp=1.0):
    """A smooth random float32 field [H,W], quantised to multiples of 2^-12."""
    H, W = shape_hw
    ys, xs = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    acc = np.zeros((H, W))
    for _ in range(n_modes):
        fx, fy = rng.uniform(0.3, 2.5, 2)
        acc += np.cos(2 * math.pi * (fx * xs + fy * ys) + rng.uniform(0, 2 * math.pi))
    return (np.round(amp * acc / n_modes * 4096) / 4096).astype(F32)


def part_segs(rng, B, C, S):
    """SCOPS-like part probabilities [B,C,S,S]: a softmax over smooth fields, quantised to multiples of 2^-12."""
    logits = np.stack([[smooth_field(rng, (S, S), amp=4.0) for _ in range(C)] for _ in range(B)]).astype(np.float64)
    p = np.exp(logits - logits.max(axis=1, keepdims=True))
    p /= p.sum(axis=1, keepdims=True)
    return (np.round(p * 4096) / 4096).astype(F32)


def uvimage_pred(rng, B, H, W, spread=1.0):
    """A texture-flow UV image [B,2,H,W]: the identity grid, perturbed smoothly, scaled by `spread` (> 1 reaches past
    [-1, 1]), quantised to multiples of 2^-12."""
    ys, xs = np.meshgrid(np.linspace(-1, 1, H), np.linspace(-1, 1, W), indexing="ij")
    out = np.empty((B, 2, H, W), F32)
    for b in range(B):
        out[b, 0] = spread * (0.8 * xs + 0.2 * smooth_field(rng, (H, W)))
        out[b, 1] = spread * (0.8 * ys + 0.2 * smooth_field(rng, (H, W)))
    return (np.round(out * 4096) / 4096).astype(F32)
