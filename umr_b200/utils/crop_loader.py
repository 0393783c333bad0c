"""The host half of the training loader's `forward_img` (data/base.py:88-186): scalar work and slicing only.

The reference crops, resizes and mirrors every image in float64 on the host (`crop`, `resize_img`, `mirror_image`) and
`set_input` normalises it on the CPU.  Here the loader keeps the scalar work -- the perturbed square box, the flip draw,
the keypoint and sfm-pose arithmetic -- and cuts the uint8 window of the source that the box overlaps.  `collate` packs
a batch's windows into one flat uint8 tensor and an int32 table, which `umr_b200.utils.image.crop_batch` turns into the
batch's images, masks and part maps on the GPU (DESIGN.md §19).

The random draws are the reference's, in its order: four `np.random.random()` in `peturb_bbox`, then
`np.random.rand(1) > 0.5` where `mirror_image` draws it, so a seeded loader gives the reference's boxes and flips.  The
keypoint and pose arithmetic is the reference's, operation for operation, in float64.
"""
import collections
import math

import numpy as np
import torch
from torch.utils.data.dataloader import default_collate

TABLE_COLS = 8   # UMR_CROP_TABLE_COLS: offset, h, w, ch, x0, y0, L, flip

# The uint8 window of one image: img [h,w,ch] (ch 1 or 3) and mask [h,w] sit at (x0, y0) in an L x L crop frame
CropWindow = collections.namedtuple("CropWindow", "img mask x0 y0 L flip")


def peturb_bbox(bbox, pf=0, jf=0):
    """utils/image.py:45-65: pad the zero-indexed box by pf and jitter it by jf of its size, four np.random.random()
    draws in the reference's order (drawn even when jf = 0)."""
    pet_bbox = [coord for coord in bbox]
    bwidth = bbox[2] - bbox[0] + 1
    bheight = bbox[3] - bbox[1] + 1
    pet_bbox[0] -= (pf * bwidth) + (1 - 2 * np.random.random()) * jf * bwidth
    pet_bbox[1] -= (pf * bheight) + (1 - 2 * np.random.random()) * jf * bheight
    pet_bbox[2] += (pf * bwidth) + (1 - 2 * np.random.random()) * jf * bwidth
    pet_bbox[3] += (pf * bheight) + (1 - 2 * np.random.random()) * jf * bheight
    return pet_bbox


def square_bbox(bbox):
    """utils/image.py:68-85: grow the shorter side to a square box; [x0, y0] ints, [x1, y1] floats, as the reference."""
    sq_bbox = [int(round(coord)) for coord in bbox]
    bwidth = sq_bbox[2] - sq_bbox[0] + 1
    bheight = sq_bbox[3] - sq_bbox[1] + 1
    maxdim = float(max(bwidth, bheight))
    dw_b_2 = int(round((maxdim - bwidth) / 2.0))
    dh_b_2 = int(round((maxdim - bheight) / 2.0))
    sq_bbox[0] -= dw_b_2
    sq_bbox[1] -= dh_b_2
    sq_bbox[2] = sq_bbox[0] + maxdim - 1
    sq_bbox[3] = sq_bbox[1] + maxdim - 1
    return sq_bbox


def draw_flip():
    """mirror_image's coin (data/base.py:226)."""
    return bool(np.random.rand(1) > 0.5)


def crop_window(img, mask, bbox):
    """The part of `crop(img, bbox)` (utils/image.py:88-119) that reads the source: the uint8 window the box overlaps.

    img: uint8 [H,W] (grey) or [H,W,3]; mask: [H,W] with values in 0..255.  Returns CropWindow with flip False.  A box
    that overlaps no pixel gives a 1 x 1 window of image 255 and mask 0, which are the frame's background values exactly
    (the reference's crop gives that frame too, where its slicing does not raise)."""
    img = np.asarray(img)
    mask = np.asarray(mask)
    if img.dtype != np.uint8 or img.ndim not in (2, 3) or (img.ndim == 3 and img.shape[2] != 3):
        raise ValueError("crop_window: img must be uint8 [H,W] or [H,W,3], got %s %s" % (img.dtype, img.shape))
    if mask.shape != img.shape[:2] or not (mask.dtype == np.uint8 or mask.dtype == np.bool_):
        raise ValueError("crop_window: mask must be uint8 or bool %s, got %s %s" % (img.shape[:2], mask.dtype, mask.shape))
    b = [int(round(c)) for c in bbox]
    L = b[2] - b[0] + 1
    if L <= 0 or b[3] - b[1] + 1 != L:
        raise ValueError("crop_window: the box must be square with a positive side, got %r" % (bbox,))
    im_h, im_w = img.shape[:2]
    xs, xe = max(0, b[0]), min(im_w, b[2] + 1)
    ys, ye = max(0, b[1]), min(im_h, b[3] + 1)
    if xe <= xs or ye <= ys:
        return CropWindow(np.full((1, 1, 1), 255, np.uint8), np.zeros((1, 1), np.uint8), 0, 0, L, False)
    win = img[ys:ye, xs:xe]
    return CropWindow(win[:, :, None] if win.ndim == 2 else win, mask[ys:ye, xs:xe].astype(np.uint8, copy=False),
                      xs - b[0], ys - b[1], L, False)


def quaternion_matrix(quaternion):
    """Homogeneous rotation matrix of a quaternion (utils/transformations.py:1254-1278, same numpy operations)."""
    q = np.array(quaternion, dtype=np.float64, copy=True)
    n = np.dot(q, q)
    if n < np.finfo(float).eps * 4.0:
        return np.identity(4)
    q *= math.sqrt(2.0 / n)
    q = np.outer(q, q)
    return np.array([
        [1.0 - q[2, 2] - q[3, 3], q[1, 2] - q[3, 0], q[1, 3] + q[2, 0], 0.0],
        [q[1, 2] + q[3, 0], 1.0 - q[1, 1] - q[3, 3], q[2, 3] - q[1, 0], 0.0],
        [q[1, 3] - q[2, 0], q[2, 3] + q[1, 0], 1.0 - q[1, 1] - q[2, 2], 0.0],
        [0.0, 0.0, 0.0, 1.0]])


def quaternion_from_matrix(matrix):
    """Quaternion of a precise rotation matrix: utils/transformations.py:1281-1363 with isprecise=True."""
    M = np.asarray(matrix, dtype=np.float64)[:4, :4]
    q = np.empty((4, ))
    t = np.trace(M)
    if t > M[3, 3]:
        q[0] = t
        q[3] = M[1, 0] - M[0, 1]
        q[2] = M[0, 2] - M[2, 0]
        q[1] = M[2, 1] - M[1, 2]
    else:
        i, j, k = 0, 1, 2
        if M[1, 1] > M[0, 0]:
            i, j, k = 1, 2, 0
        if M[2, 2] > M[i, i]:
            i, j, k = 2, 0, 1
        t = M[i, i] - (M[j, j] + M[k, k]) + M[3, 3]
        q[i] = t
        q[j] = M[i, j] + M[j, i]
        q[k] = M[k, i] + M[i, k]
        q[3] = M[k, j] - M[j, k]
        q = q[[3, 0, 1, 2]]
    q *= 0.5 / math.sqrt(t * M[3, 3])
    if q[0] < 0.0:
        np.negative(q, q)
    return q


def transform_points(kp, vis, sfm_pose, bbox, img_size, flip, kp_perm):
    """The keypoint and sfm-pose arithmetic of crop_image, scale_image, mirror_image and normalize_kp
    (data/base.py:188-251), in float64 as the reference does it.  kp [K,3] float64, vis [K] bool, sfm_pose
    [scale, trans [2], quaternion [4]] (updated in place, as in the reference), bbox the square box.  Returns
    (kp_norm, sfm_pose)."""
    kp = np.copy(kp)
    # crop_image
    kp[vis, 0] -= bbox[0]
    kp[vis, 1] -= bbox[1]
    sfm_pose[1][0] -= bbox[0]
    sfm_pose[1][1] -= bbox[1]
    # scale_image: the crop's side is the box's, resized to round(L * scale)
    L = int(round(bbox[2])) - int(round(bbox[0])) + 1
    scale = img_size / float(max(L, L))
    side = int(np.round(L * scale))
    if side != img_size:
        raise ValueError("transform_points: a %d box resizes to %d, not %d" % (L, side, img_size))
    kp[vis, :2] *= scale
    sfm_pose[0] *= scale
    sfm_pose[1] *= scale
    # mirror_image
    if flip:
        new_x = side - kp[:, 0] - 1
        kp = np.hstack((new_x[:, None], kp[:, 1:]))[kp_perm, :]
        R = quaternion_matrix(sfm_pose[2])
        flip_R = np.diag([-1, 1, 1, 1]).dot(R.dot(np.diag([-1, 1, 1, 1])))
        sfm_pose[2] = quaternion_from_matrix(flip_R)
        sfm_pose[1][0] = side - sfm_pose[1][0] - 1
    # normalize_kp
    v = kp[:, 2, None] > 0
    new_kp = np.stack([2 * (kp[:, 0] / side) - 1, 2 * (kp[:, 1] / side) - 1, kp[:, 2]]).T
    sfm_pose[0] *= (1.0 / side + 1.0 / side)
    sfm_pose[1][0] = 2.0 * (sfm_pose[1][0] / side) - 1
    sfm_pose[1][1] = 2.0 * (sfm_pose[1][1] / side) - 1
    return v * new_kp, sfm_pose


def crop_item(img, mask, bbox, kp, sfm_pose, img_size, padding_frac, jitter_frac, mirror, kp_perm):
    """forward_img's sequence (data/base.py:108-150) on the host: the perturbed square box, the window, the flip draw and
    the points, drawing np.random in the reference's order.  bbox is the zero-indexed tight box, kp [K,3] with 1-indexed
    visible points (the loader's `parts.T`), sfm_pose [scale, trans, quaternion].  jitter_frac is 0 outside training.
    Returns (CropWindow, kp_norm, sfm_pose, square box)."""
    kp = np.array(kp, dtype=float)
    vis = kp[:, 2] > 0
    kp[vis, :2] -= 1
    box = square_bbox(peturb_bbox(bbox, pf=padding_frac, jf=jitter_frac))
    win = crop_window(img, mask, box)
    flip = draw_flip() if mirror else False
    kp_norm, sfm_pose = transform_points(kp, vis, sfm_pose, box, img_size, flip, kp_perm)
    return win._replace(flip=flip), kp_norm, sfm_pose, box


def collate(batch):
    """DataLoader collate_fn: each item's 'crop' CropWindow goes into 'crop_pack' (uint8 [bytes]: per image its image
    window [h,w,ch] then its mask window [h,w]) and 'crop_table' (int32 [B,8]: offset, h, w, ch, x0, y0, L, flip);
    every other key goes through default_collate.  With pin_memory=True the DataLoader pins both."""
    wins = [item["crop"] for item in batch]
    rest = default_collate([{k: v for k, v in item.items() if k != "crop"} for item in batch])
    sizes = [w.img.size + w.mask.size for w in wins]
    total = int(sum(sizes))
    if total >= 2 ** 31:
        raise ValueError("collate: %d window bytes do not fit the table's int32 offsets" % total)
    pack = torch.empty(total, dtype=torch.uint8)
    table = torch.empty(len(wins), TABLE_COLS, dtype=torch.int32)
    buf = pack.numpy()
    off = 0
    for i, (w, n) in enumerate(zip(wins, sizes)):
        h, wd, ch = w.img.shape
        buf[off:off + w.img.size] = w.img.reshape(-1)
        buf[off + w.img.size:off + n] = w.mask.reshape(-1)
        table[i] = torch.tensor([off, h, wd, ch, w.x0, w.y0, w.L, int(w.flip)], dtype=torch.int32)
        off += n
    rest["crop_pack"] = pack
    rest["crop_table"] = table
    return rest
