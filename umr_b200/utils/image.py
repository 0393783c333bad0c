"""`utils/image.py` pieces on the per-step path (reference: utils/image.py:120-206).

`compute_dt_barrier` is called once per image per training step on the host with scipy in the reference
(experiments/train_s2.py:196); here the whole batch is transformed by one pair of kernels (csrc/mesh_ops.cu `k_edt_*`).

`prob2center` and `sample_prob` (utils/image.py:168-206) build CorrLossChamfer's part points in the reference's data
loader, four channels per image on the CPU (data/base.py:155-166).  `part_points` does every channel of a whole batch in
two kernel launches (csrc/part_points.cu, DESIGN.md §17); `prob2center` and `sample_prob` keep the reference's
single-image signatures on top of it.

`crop_batch` is the pixel half of the loader's `forward_img` (crop, cv2.resize, mirror: data/base.py:88-186) and of
`set_input`'s ResNet normalisation and part-map normalisation (experiments/train_s2.py:166-192), for a whole batch in two
kernel launches (csrc/crop.cu, DESIGN.md §19); the loader's half is `umr_b200.utils.crop_loader`.
"""
import ctypes

import numpy as np
import torch

from .. import _lib, ops
from ..raster import _ptr, _stream_ptr


def compute_dt_barrier(mask, k=50):
    """Barrier distance transform.  mask: [H,W] or [B,H,W], numpy array or torch tensor (non-zero = object).
    Returns the same container type: numpy input -> numpy float64-compatible array (values computed on the GPU),
    cuda tensor -> cuda float32 tensor."""
    if isinstance(mask, np.ndarray):
        out = ops.dt_barrier(torch.from_numpy(np.ascontiguousarray(mask, dtype=np.float32)).cuda(), k)
        return out.cpu().numpy().astype(np.float64)
    if not mask.is_cuda:
        return ops.dt_barrier(mask.cuda(), k).to(mask.device)
    return ops.dt_barrier(mask, k)


_DTYPES = {torch.float32: 0, torch.float64: 1}   # UMR_DTYPE_FLOAT32 / UMR_DTYPE_FLOAT64
MAX_CHANNELS = 8      # UMR_PART_POINTS_MAX_CHANNELS
MAX_DRAWS = 1024      # UMR_PART_POINTS_MAX_DRAWS: floor(1.5 n) pixels drawn per channel
_STATUS = {1: "a NaN, infinite or negative probability, or a zero or non-finite sum",
           2: "fewer positive pixels than the floor(1.5 * num_samples) it draws"}


def _part_points(part_prob, mask, uniforms, num_samples, channels, centers_in=None, drawn=False):
    """The one library call behind part_points, prob2center and sample_prob.  part_prob [B,S,S,C], mask [B,S,S] and
    uniforms [B,K,S*S] on one CUDA device, K = len(channels) = len(num_samples); centers_in [B,K,2] replaces the centres
    of the nearest-n selection.  Returns (centers [B,K,2], points tuple of [B,n_k,2], drawn tuple of [B,m_k] int32 pixel
    indices in ascending order, or None).  Reads the status once (one host synchronisation) and raises ValueError for a
    channel torch.multinomial would refuse."""
    ts = [part_prob, mask, uniforms] + ([centers_in] if centers_in is not None else [])
    for t in ts:
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise TypeError("part_points: inputs must be CUDA tensors")
    if len({t.device for t in ts}) > 1:
        raise ValueError("part_points: inputs must be on one device, got %s" % sorted(str(t.device) for t in ts))
    if part_prob.dtype not in _DTYPES:
        raise TypeError("part_points: part_prob must be float32 or float64, got %s" % part_prob.dtype)
    if part_prob.dim() != 4 or part_prob.shape[1] != part_prob.shape[2]:
        raise ValueError("part_points: part_prob must be [B,S,S,C] with square maps, got %s" % (tuple(part_prob.shape),))
    B, S, _, C = part_prob.shape
    if tuple(mask.shape) != (B, S, S):
        raise ValueError("part_points: mask must be [B,S,S] = %s, got %s" % ((B, S, S), tuple(mask.shape)))
    channels, num_samples = tuple(channels), tuple(num_samples)
    K = len(channels)
    if not 1 <= K <= MAX_CHANNELS or len(num_samples) != K:
        raise ValueError("part_points: 1 to %d channels, one num_samples each, got %r and %r"
                         % (MAX_CHANNELS, channels, num_samples))
    for ch, n in zip(channels, num_samples):
        if isinstance(ch, bool) or int(ch) != ch or not 0 <= ch < C:
            raise ValueError("part_points: channel %r is not one of part_prob's %d" % (ch, C))
        if isinstance(n, bool) or int(n) != n or n < 1 or int(1.5 * n) > MAX_DRAWS:
            raise ValueError("part_points: num_samples must be integers with 1 <= n and floor(1.5 n) <= %d, got %r"
                             % (MAX_DRAWS, n))
    if tuple(uniforms.shape) != (B, K, S * S) or uniforms.dtype != part_prob.dtype:
        raise ValueError("part_points: uniforms must be %s [%d,%d,%d], got %s %s"
                         % (part_prob.dtype, B, K, S * S, uniforms.dtype, tuple(uniforms.shape)))
    if centers_in is not None and tuple(centers_in.shape) != (B, K, 2):
        raise ValueError("part_points: centres must be [%d,%d,2], got %s" % (B, K, tuple(centers_in.shape)))
    dt, dev = part_prob.dtype, part_prob.device
    prob = part_prob.detach().contiguous()
    msk = mask.detach().to(dt).contiguous()
    u = uniforms.detach().contiguous()
    cin = centers_in.detach().to(dt).contiguous() if centers_in is not None else None
    with torch.cuda.device(dev):
        centers = torch.empty(B, K, 2, device=dev, dtype=dt)
        points = tuple(torch.empty(B, int(n), 2, device=dev, dtype=dt) for n in num_samples)
        draws = tuple(torch.empty(B, int(1.5 * n), device=dev, dtype=torch.int32) for n in num_samples) if drawn else None
        status = torch.empty(B, K, device=dev, dtype=torch.int32)
        ch_arr = (ctypes.c_int32 * K)(*[int(c) for c in channels])
        n_arr = (ctypes.c_int32 * K)(*[int(n) for n in num_samples])
        pt_arr = (ctypes.c_void_p * K)(*[p.data_ptr() for p in points])
        dr_arr = (ctypes.c_void_p * K)(*[d.data_ptr() for d in draws]) if drawn else None
        _lib.check(_lib.load().umr_part_points(_ptr(prob), _ptr(msk), _ptr(u), B, S, C, K, ch_arr, n_arr, _DTYPES[dt],
                                               _ptr(cin), _ptr(centers), pt_arr, dr_arr, _ptr(status), _stream_ptr(dev)),
                   "umr_part_points")
        st = status.cpu()   # the call's one host synchronisation
    if st.any():
        b, k = [int(i) for i in st.nonzero()[0]]
        raise ValueError("part_points: image %d, channel %d: %s (%d of %d channels refused)"
                         % (b, channels[k], _STATUS[int(st[b, k])], int((st != 0).sum()), B * K))
    return centers, points, draws


def part_points(part_prob, mask, num_samples=(10, 10, 30, 30), channels=(1, 2, 3, 4), generator=None):
    """The SCOPS part centres and part points of a batch: data/base.py:155-166 for every image at once.

    part_prob [B,S,S,C] (float32 or float64) and mask [B,S,S] (cast to part_prob's dtype) are CUDA tensors on one
    device, with square maps.  For each channel ch = channels[k] and n = num_samples[k]: q = part_prob[..., ch] * mask,
    pdf = q / sum(q); the centre is `prob2center`'s; m = floor(1.5 n) distinct pixels are drawn with torch.multinomial's
    without-replacement law over pdf (Efraimidis-Spirakis keys over uniforms from torch.rand(..., generator=generator)
    on the device, so a seeded generator reproduces a call) and the n nearest the centre are kept, ascending by squared
    distance, ties to the lower pixel index.  Points are ((x / 256) * 2 - 1, (y / 256) * 2 - 1), the reference's
    constant, right at S = 256.  The draws are equal in distribution, not bitwise, to the reference's CPU stream.

    Returns (centers [B,K,2], points), points a tuple of [B,n_k,2]: with the defaults, the head, neck, back and belly
    points CorrLossChamfer takes.  Each call synchronises with the host once, to read the status: a channel with a NaN,
    infinite or negative q, a zero sum, or fewer than m positive pixels raises ValueError, as torch.multinomial does."""
    if not isinstance(part_prob, torch.Tensor) or part_prob.dim() != 4:
        raise ValueError("part_points: part_prob must be a [B,S,S,C] tensor")
    B, S = part_prob.shape[:2]
    u = torch.rand(B, len(tuple(channels)), S * S, generator=generator, device=part_prob.device, dtype=part_prob.dtype)
    centers, points, _ = _part_points(part_prob, mask, u, num_samples, channels)
    return centers, points


def prob2center(part_prob, mask, ch=1):
    """utils/image.py:168-181 for one image: part_prob [S,S,C] and mask [S,S] CUDA tensors -> the centre [2] of channel
    `ch`, in part_prob's dtype.  Raises ValueError where part_points does.  Synchronises once."""
    S = part_prob.shape[0]
    u = torch.zeros(1, 1, S * S, device=part_prob.device, dtype=part_prob.dtype)
    centers, _, _ = _part_points(part_prob[None], mask[None], u, (1,), (ch,))
    return centers[0, 0]


def sample_prob(part_prob, mask, center, num_samples=10, ch=1, generator=None):
    """utils/image.py:183-206 for one image: part_prob [S,S,C], mask [S,S] and center [2] CUDA tensors -> the
    num_samples points [n,2] nearest `center` among floor(1.5 num_samples) drawn from channel `ch`, as part_points draws
    them.  Raises ValueError where part_points does.  Synchronises once."""
    S = part_prob.shape[0]
    u = torch.rand(1, 1, S * S, generator=generator, device=part_prob.device, dtype=part_prob.dtype)
    c = torch.as_tensor(center, device=part_prob.device).reshape(1, 1, 2)
    _, points, _ = _part_points(part_prob[None], mask[None], u, (num_samples,), (ch,), centers_in=c)
    return points[0][0]


CROP_TABLE_COLS = 8       # UMR_CROP_TABLE_COLS
CROP_MAX_CHANNELS = 8     # UMR_CROP_MAX_CHANNELS


def crop_batch(pack, table, size, part_prob=None):
    """The batch `crop_loader.collate` packed, cropped, resized to size x size, mirrored and normalised on the GPU.

    pack: uint8 [bytes] ('crop_pack'), on a CUDA device or pinned on the host; table: int32 [B,8] on the host
    ('crop_table': offset, h, w, ch, x0, y0, L, flip per image), validated there and copied to the device without a
    host synchronisation; part_prob: optional float32 [B,size,size,C] CUDA tensor, C <= 8, the SCOPS maps as loaded.
    Returns (imgs [B,3,S,S], input_imgs [B,3,S,S], masks [B,S,S], part_prob [B,S,S,C] mirrored, part_segs [B,C,S,S]),
    float32, the last two None without part_prob: cv2.resize INTER_LINEAR on the float64 crop frame rounded once to
    float32, torchvision's ImageNet Normalize, and q / max(q) per (image, channel) for q = part_prob * masks.  One kernel
    launch, two with part_prob; bitwise reproducible."""
    if not isinstance(table, torch.Tensor) or table.is_cuda or table.dtype != torch.int32 or table.dim() != 2 \
            or table.shape[1] != CROP_TABLE_COLS or table.shape[0] < 1:
        raise ValueError("crop_batch: table must be a host int32 [B,%d] tensor" % CROP_TABLE_COLS)
    if not isinstance(pack, torch.Tensor) or pack.dtype != torch.uint8 or pack.dim() != 1 or pack.numel() < 1:
        raise ValueError("crop_batch: pack must be a non-empty uint8 [bytes] tensor")
    if isinstance(size, bool) or int(size) != size or size < 1:
        raise ValueError("crop_batch: size must be a positive integer, got %r" % (size,))
    B, S = table.shape[0], int(size)
    if part_prob is not None:
        if not isinstance(part_prob, torch.Tensor) or not part_prob.is_cuda:
            raise TypeError("crop_batch: part_prob must be a CUDA tensor")
        if part_prob.dtype != torch.float32:
            raise TypeError("crop_batch: part_prob must be float32, got %s" % part_prob.dtype)
        if part_prob.dim() != 4 or tuple(part_prob.shape[:3]) != (B, S, S) or not 1 <= part_prob.shape[3] <= CROP_MAX_CHANNELS:
            raise ValueError("crop_batch: part_prob must be [%d,%d,%d,C] with 1 <= C <= %d, got %s"
                             % (B, S, S, CROP_MAX_CHANNELS, tuple(part_prob.shape)))
        if pack.is_cuda and pack.device != part_prob.device:
            raise ValueError("crop_batch: pack and part_prob must be on one device, got %s and %s"
                             % (pack.device, part_prob.device))
    if pack.is_cuda:
        dev = pack.device
    elif part_prob is not None:
        dev = part_prob.device
    else:
        dev = torch.device("cuda", torch.cuda.current_device())
    tab = table.contiguous()
    with torch.cuda.device(dev):
        pk = pack.to(dev, non_blocking=True).contiguous()
        tab_dev = tab.to(dev, non_blocking=True)
        imgs = torch.empty(B, 3, S, S, device=dev)
        input_imgs = torch.empty(B, 3, S, S, device=dev)
        masks = torch.empty(B, S, S, device=dev)
        prob = segs = None
        C = 0
        if part_prob is not None:
            C = part_prob.shape[3]
            part_prob = part_prob.detach().contiguous()
            prob = torch.empty_like(part_prob)
            segs = torch.empty(B, C, S, S, device=dev)
        host = ctypes.cast(tab.data_ptr(), ctypes.POINTER(ctypes.c_int32))
        _lib.check(_lib.load().umr_crop_batch(_ptr(pk), pk.numel(), _ptr(tab_dev), host, B, S, _ptr(part_prob), C,
                                              _ptr(imgs), _ptr(input_imgs), _ptr(masks), _ptr(prob), _ptr(segs),
                                              _stream_ptr(dev)), "umr_crop_batch")
    return imgs, input_imgs, masks, prob, segs
