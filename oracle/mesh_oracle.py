"""CPU oracles for the SoftRas natives / regularisers around the render path -- TEST INFRASTRUCTURE ONLY.

* create_texture_image_np / load_textures_np: numpy float32 restatements of the reference CUDA kernels
  (external/SoftRas/soft_renderer/cuda/create_texture_image_cuda_kernel.cu:10-70, load_textures_cuda_kernel.cu:8-66),
  one rounding per operation in the reference's order (numpy never contracts to FMA), double where the kernel's
  literals promote to double.
* laplacian_loss / flatten_loss: the reference modules' own formulas (SoftRas/losses.py:6-114) on torch CPU, with the
  reference's O(E*F) edge scan.
* dt_barrier: utils/image.py:130-141 (scipy).
"""
import numpy as np
import torch

f32 = np.float32


def create_texture_image_np(faces_uv, textures, image, eps=1e-5):
    faces_uv = np.asarray(faces_uv, f32)
    textures = np.asarray(textures, f32)
    image = np.array(image, f32, copy=True)
    H, W = image.shape[:2]
    F_ = textures.shape[0]
    R = int(np.sqrt(textures.shape[1]))
    tile_width = int(np.sqrt(F_ - 1)) + 1
    R_out = W // tile_width
    eps = f32(eps)
    i = np.arange(H * W)
    x = (i % (tile_width * R_out)).astype(np.int64)
    y = (i // (tile_width * R_out)).astype(np.int64)
    fn = x // R_out + (y // R_out) * tile_width
    ok = fn < F_
    fnc = np.minimum(fn, F_ - 1)
    p0, p1, p2 = faces_uv[fnc, 0], faces_uv[fnc, 1], faces_uv[fnc, 2]
    fi = [p1[:, 1] - p2[:, 1], p2[:, 0] - p1[:, 0], p1[:, 0] * p2[:, 1] - p2[:, 0] * p1[:, 1],
          p2[:, 1] - p0[:, 1], p0[:, 0] - p2[:, 0], p2[:, 0] * p0[:, 1] - p0[:, 0] * p2[:, 1],
          p0[:, 1] - p1[:, 1], p1[:, 0] - p0[:, 0], p0[:, 0] * p1[:, 1] - p1[:, 0] * p0[:, 1]]
    den = p2[:, 0] * (p0[:, 1] - p1[:, 1]) + p0[:, 0] * (p1[:, 1] - p2[:, 1]) + p1[:, 0] * (p2[:, 1] - p0[:, 1])
    fi = [(v / (den + eps)).astype(f32) for v in fi]
    xf, yf = x.astype(f32), y.astype(f32)
    w = []
    w_sum = np.zeros_like(xf)
    for k in range(3):
        wk = (fi[3 * k] * xf + fi[3 * k + 1] * yf + fi[3 * k + 2]).astype(f32)
        wk = np.maximum(np.minimum(wk, f32(1)), f32(0))
        w.append(wk)
        w_sum = (w_sum + wk).astype(f32)
    w = [(wk / (w_sum + eps)).astype(f32) for wk in w]
    w_x = (w[0] * f32(R)).astype(np.int64)
    w_y = (w[1] * f32(R)).astype(np.int64)
    low = ((w[0] + w[1]).astype(f32) * f32(R) - w_x.astype(f32) - w_y.astype(f32)).astype(f32) <= 1
    idx = np.where(low, w_y * R + w_x, (R - 1 - w_y) * R + (R - 1 - w_x))
    out = image.reshape(-1, 3)
    vals = textures[fnc, np.clip(idx, 0, R * R - 1)]
    out[ok] = vals[ok]
    return out.reshape(H, W, 3)


def load_textures_np(image, faces_uv, is_update, textures):
    image = np.asarray(image, f32)
    faces_uv = np.asarray(faces_uv, f32)
    out = np.array(textures, f32, copy=True)
    F_, RR, _ = out.shape
    R = int(np.sqrt(RR))
    H, W = image.shape[:2]
    i = np.arange(F_ * RR)
    fn = i // RR
    w_y = (i % RR) // R
    w_x = i % R
    lower = (w_x + w_y) < R
    w0 = np.where(lower, (w_x + 1. / 3.) / R, ((R - 1. - w_x) + 2. / 3.) / R).astype(f32)
    w1 = np.where(lower, (w_y + 1. / 3.) / R, ((R - 1. - w_y) + 2. / 3.) / R).astype(f32)
    w2 = (1. - w0.astype(np.float64) - w1.astype(np.float64)).astype(f32)
    face = faces_uv[fn]
    pos_x = ((face[:, 0, 0] * w0 + face[:, 1, 0] * w1).astype(f32) + face[:, 2, 0] * w2).astype(f32) * f32(W - 1)
    pos_y = ((face[:, 0, 1] * w0 + face[:, 1, 1] * w1).astype(f32) + face[:, 2, 1] * w2).astype(f32) * f32(H - 1)
    ix, iy = pos_x.astype(np.int64), pos_y.astype(np.int64)
    iy1 = (pos_y + f32(1)).astype(np.int64)
    wx1 = (pos_x - ix.astype(f32)).astype(f32)
    wx0 = (f32(1) - wx1).astype(f32)
    wy1 = (pos_y - iy.astype(f32)).astype(f32)
    wy0 = (f32(1) - wy1).astype(f32)
    # the four corners clamped into the image (the reference reads outside it at uv = 1 and uv < 0; DESIGN.md §2)
    x0, x1 = np.clip(ix, 0, W - 1), np.clip(ix + 1, 0, W - 1)
    y0, y1 = np.clip(iy, 0, H - 1), np.clip(iy1, 0, H - 1)
    flat = out.reshape(-1, 3)
    upd = np.asarray(is_update)[fn] != 0
    c = np.zeros((F_ * RR, 3), f32)
    c = (c + image[y0, x0] * (wx0 * wy0)[:, None]).astype(f32)
    c = (c + image[y1, x0] * (wx0 * wy1)[:, None]).astype(f32)
    c = (c + image[y0, x1] * (wx1 * wy0)[:, None]).astype(f32)
    c = (c + image[y1, x1] * (wx1 * wy1)[:, None]).astype(f32)
    flat[upd] = c[upd]
    return flat.reshape(F_, RR, 3)


def laplacian_matrix(nv, faces):
    """SoftRas/losses.py:12-27."""
    faces = np.asarray(faces)
    laplacian = np.zeros([nv, nv]).astype(np.float32)
    laplacian[faces[:, 0], faces[:, 1]] = -1
    laplacian[faces[:, 1], faces[:, 0]] = -1
    laplacian[faces[:, 1], faces[:, 2]] = -1
    laplacian[faces[:, 2], faces[:, 1]] = -1
    laplacian[faces[:, 2], faces[:, 0]] = -1
    laplacian[faces[:, 0], faces[:, 2]] = -1
    r, c = np.diag_indices(laplacian.shape[0])
    laplacian[r, c] = -laplacian.sum(1)
    for i in range(nv):
        laplacian[i, :] /= laplacian[i, i]
    return torch.from_numpy(laplacian)


def laplacian_loss(x, faces, average=False):
    """SoftRas/losses.py:31-37."""
    L = laplacian_matrix(x.size(1), faces)
    y = torch.matmul(L, x)
    y = y.pow(2).sum(tuple(range(y.ndimension())[1:]))
    return y.sum() / x.size(0) if average else y


def flatten_edges(faces):
    """SoftRas/losses.py:45-64 (the reference's O(E*F) scan)."""
    faces = np.asarray(faces)
    vertices = list(set([tuple(v) for v in np.sort(np.concatenate((faces[:, 0:2], faces[:, 1:3]), axis=0))]))
    v0s = np.array([v[0] for v in vertices], 'int32')
    v1s = np.array([v[1] for v in vertices], 'int32')
    v2s, v3s = [], []
    for v0, v1 in zip(v0s, v1s):
        count = 0
        for face in faces:
            if v0 in face and v1 in face:
                v = np.copy(face)
                v = v[v != v0]
                v = v[v != v1]
                if count == 0:
                    v2s.append(int(v[0]))
                    count += 1
                else:
                    v3s.append(int(v[0]))
    return [torch.from_numpy(np.asarray(a, 'int64')) for a in (v0s, v1s, v2s, v3s)]


def flatten_loss(vertices, faces, average=False, eps=1e-6):
    """SoftRas/losses.py:71-114."""
    i0, i1, i2, i3 = flatten_edges(faces)
    v0s, v1s, v2s, v3s = vertices[:, i0, :], vertices[:, i1, :], vertices[:, i2, :], vertices[:, i3, :]
    a1 = v1s - v0s
    b1 = v2s - v0s
    a1l2 = a1.pow(2).sum(-1)
    b1l2 = b1.pow(2).sum(-1)
    a1l1 = (a1l2 + eps).sqrt()
    b1l1 = (b1l2 + eps).sqrt()
    ab1 = (a1 * b1).sum(-1)
    cos1 = ab1 / (a1l1 * b1l1 + eps)
    sin1 = (1 - cos1.pow(2) + eps).sqrt()
    c1 = a1 * (ab1 / (a1l2 + eps))[:, :, None]
    cb1 = b1 - c1
    cb1l1 = b1l1 * sin1
    a2 = v1s - v0s
    b2 = v3s - v0s
    a2l2 = a2.pow(2).sum(-1)
    b2l2 = b2.pow(2).sum(-1)
    a2l1 = (a2l2 + eps).sqrt()
    b2l1 = (b2l2 + eps).sqrt()
    ab2 = (a2 * b2).sum(-1)
    cos2 = ab2 / (a2l1 * b2l1 + eps)
    sin2 = (1 - cos2.pow(2) + eps).sqrt()
    c2 = a2 * (ab2 / (a2l2 + eps))[:, :, None]
    cb2 = b2 - c2
    cb2l1 = b2l1 * sin2
    cos = (cb1 * cb2).sum(-1) / (cb1l1 * cb2l1 + eps)
    loss = (cos + 1).pow(2).sum(tuple(range(cos.ndimension())[1:]))
    return loss.sum() / vertices.size(0) if average else loss


def dt_barrier(mask, k=50):
    """utils/image.py:130-141."""
    from scipy.ndimage import distance_transform_edt
    dist_out = distance_transform_edt(1 - mask)
    dist_in = distance_transform_edt(mask)
    dist_diff = (dist_out - dist_in) / max(mask.shape)
    return 1. / (1 + np.exp(k * -dist_diff))
