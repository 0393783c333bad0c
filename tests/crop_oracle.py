"""numpy restatement of the batch crop (DESIGN.md §19): the crop frame, cv2.resize INTER_LINEAR on float64 as the
contract states it, the mirror, torchvision's ImageNet Normalize and set_input's part-map normalisation.  The kernels
are pinned to it bit for bit, and it to the reference's own float32 outputs (tests/golden/crop/reference.npz)."""
import numpy as np

MEAN = np.array([0.485, 0.456, 0.406], np.float32)
STD = np.array([0.229, 0.224, 0.225], np.float32)


def frame(win):
    """The L x L crop frame of a CropWindow in float64: (image [L,L,3], mask [L,L])."""
    L = win.L
    img = np.ones((L, L, 3))
    mask = np.zeros((L, L))
    h, w = win.mask.shape
    img[win.y0:win.y0 + h, win.x0:win.x0 + w] = win.img / 255.0   # a grey window broadcasts to RGB
    mask[win.y0:win.y0 + h, win.x0:win.x0 + w] = win.mask
    return img, mask


def taps(S, L):
    """Per output index: the two source indices and the float32 weights (cv2 resize.cpp, INTER_LINEAR)."""
    scale = 1.0 / (S / L)
    f = ((np.arange(S) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = f - s.astype(np.float32)
    low, high = s < 0, s >= L - 1
    s[low], f[low] = 0, 0
    s[high], f[high] = L - 1, 0
    return s, np.minimum(s + 1, L - 1), np.float32(1) - f, f


def resize(src, S):
    """src [L,L] or [L,L,ch] float64 -> [S,S(,ch)] float64: the horizontal pass then the vertical, each a*w0 + b*w1."""
    L = src.shape[0]
    x0, x1, a0, a1 = taps(S, L)
    sh = (1, -1) + (1,) * (src.ndim - 2)
    a0, a1 = a0.astype(np.float64).reshape(sh), a1.astype(np.float64).reshape(sh)
    r = src[:, x0] * a0 + src[:, x1] * a1
    y0, y1, b0, b1 = taps(S, L)
    sv = (-1, 1) + (1,) * (src.ndim - 2)
    return r[y0] * b0.astype(np.float64).reshape(sv) + r[y1] * b1.astype(np.float64).reshape(sv)


def crop(win, S, double=False):
    """imgs [3,S,S] and masks [S,S] of one CropWindow, mirrored when win.flip: float32, or the float64 resize results."""
    img, mask = frame(win)
    img, mask = resize(img, S), resize(mask, S)
    if win.flip:
        img, mask = img[:, ::-1], mask[:, ::-1]
    img = np.ascontiguousarray(img.transpose(2, 0, 1))
    mask = np.ascontiguousarray(mask)
    return (img, mask) if double else (img.astype(np.float32), mask.astype(np.float32))


def normalize(imgs):
    """torchvision Normalize: float32 subtract, then float32 divide, by channel ([...,3,S,S])."""
    return (imgs - MEAN[:, None, None]) / STD[:, None, None]


def part_maps(part_prob, mask, flip):
    """part_prob [S,S,C] float32, mask [S,S] float32 -> (part_prob mirrored [S,S,C], part_segs [C,S,S]):
    q = p * mask, q / max(q) per channel, a NaN max if any q is NaN."""
    p = np.ascontiguousarray(part_prob[:, ::-1] if flip else part_prob)
    q = p.transpose(2, 0, 1) * mask[None]
    with np.errstate(divide="ignore", invalid="ignore"):
        return p, q / q.reshape(q.shape[0], -1).max(axis=1)[:, None, None]


def batch(wins, S, part_prob=None):
    """The whole call: (imgs, input_imgs, masks, part_prob mirrored or None, part_segs or None)."""
    out = [crop(w, S) for w in wins]
    imgs = np.stack([o[0] for o in out])
    masks = np.stack([o[1] for o in out])
    if part_prob is None:
        return imgs, normalize(imgs), masks, None, None
    pm = [part_maps(part_prob[b], masks[b], w.flip) for b, w in enumerate(wins)]
    return imgs, normalize(imgs), masks, np.stack([p[0] for p in pm]), np.stack([p[1] for p in pm])


def bitwise_equal(a, b):
    """Equal bit for bit, any NaN equal to any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    both_nan = np.isnan(a) & np.isnan(b)
    ia = a.view(np.int32 if a.dtype == np.float32 else np.int64)
    ib = b.view(np.int32 if b.dtype == np.float32 else np.int64)
    return bool(((ia == ib) | both_nan).all())
