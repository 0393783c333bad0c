"""Keypoint transfer and PCK of UMR's keypoint evaluation (experiments/test_kp.py), batched over image pairs.

The reference transfers one pair at a time: `map_kp_img1_to_img2_flow` (test_kp.py:125-158) draws K heat maps on the
host and samples them with `grid_sample`; `map_kp_img1_to_img2_cam` (:160-193) runs `nonzero` (a host synchronisation)
and two `distChamfer` calls.  Here P pairs go through one kernel launch each mode (csrc/kp_transfer.cu), with the
torch-1.1 sampling convention (align_corners=True) the texture flow was trained with, which the reference's own calls
no longer use on torch >= 1.3.  Contract and deviations: DESIGN.md §16.

    pred = kp_transfer.transfer_flow(kps_src, tex_flow_src, tex_flow_tgt)          # [P,K,2]
    pck1, pck15 = kp_transfer.pck(pred, kps_tgt[..., :2], vis, err_scaling)

Evaluation only: the inputs are CUDA tensors, the outputs carry no gradient.
"""
import functools

import numpy as np
import torch

from .. import _lib
from ..ops import _pairs
from ..raster import _ptr, _stream_ptr

@functools.lru_cache(maxsize=None)
def _gauss(sigma, device):
    """The unnormalised Gaussian of draw_labelmap (kp_utils.py:53-58), [(6 sigma + 1)^2]: numpy float64 `exp`, then
    float32, on `device`.  Cached like `_grid`, so a call after the first makes no host-to-device copy (a CUDA graph can
    capture it)."""
    n = 6 * sigma + 1
    x = np.arange(0, n, 1, float)
    y = x[:, np.newaxis]
    c = n // 2
    g = np.exp(- ((x - c) ** 2 + (y - c) ** 2) / (2 * sigma ** 2))
    return torch.from_numpy(g.astype(np.float32).reshape(-1)).to(device)


@functools.lru_cache(maxsize=None)
def _grid(size, device):
    """The identity grid's coordinates [size] on `device`: torch.linspace(-1, 1, size), which torch-1.1 `affine_grid` with
    an identity theta yields along each axis (kp_utils.py:13-24)."""
    return torch.linspace(-1, 1, size, dtype=torch.float32).to(device)


def _need_cuda(*ts):
    """All CUDA tensors on one device: the kernel reads every buffer on the first one's device."""
    for t in ts:
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise TypeError("kp_transfer: inputs must be CUDA tensors")
    devices = {t.device for t in ts}
    if len(devices) > 1:
        raise ValueError("kp_transfer: inputs must be on one device, got %s" % sorted(str(d) for d in devices))


def _keypoints(kps):
    """[P,K,2] or [P,K,3] (the visibility column is ignored, as the reference ignores it) -> contiguous float32 [P,K,2]."""
    if kps.dim() != 3 or kps.shape[2] not in (2, 3):
        raise ValueError("kp_transfer: keypoints must be [P,K,2] or [P,K,3], got %s" % (tuple(kps.shape),))
    return _pairs(kps.detach()[:, :, :2].to(torch.float32).contiguous())


def _int(v, what, low):
    if isinstance(v, bool) or int(v) != v or v < low:
        raise ValueError("kp_transfer: %s must be an integer >= %d, got %r" % (what, low, v))
    return int(v)


def transfer_flow(kps_src, flow_src, flow_tgt, sigma=3, image_size=256):
    """Flow mode of test_kp.py:125-158 for P pairs: keypoints kps_src [P,K,2|3] of each source image, texture flows
    flow_src / flow_tgt [P,F,T,T,2] or [P,F,T*T,2] of the source and target images -> transferred keypoints [P,K,2] in
    the target image's [-1, 1] coordinates.  Each keypoint's heat map (Gaussian of `sigma`, on an image_size^2 image,
    centred at (kp + 1) / 2 * 256 whatever image_size is, as test_kp.py:146 writes it) picks the face whose source-flow samples it covers most; the result is that face's mean target-flow position on the
    identity grid."""
    _need_cuda(kps_src, flow_src, flow_tgt)
    sigma = _int(sigma, "sigma", 1)
    image_size = _int(image_size, "image_size", 1)
    kps = _keypoints(kps_src)
    P, K = kps.shape[:2]
    if flow_src.shape != flow_tgt.shape or flow_src.dim() < 3 or flow_src.shape[0] != P or flow_src.shape[-1] != 2:
        raise ValueError("kp_transfer: flows must both be [P,F,...,2] with P = %d, got %s and %s"
                         % (P, tuple(flow_src.shape), tuple(flow_tgt.shape)))
    F = flow_src.shape[1]
    fs = _pairs(flow_src.detach().reshape(P, F, -1, 2).to(torch.float32).contiguous())
    ft = _pairs(flow_tgt.detach().reshape(P, F, -1, 2).to(torch.float32).contiguous())
    dev = kps.device
    with torch.cuda.device(dev):
        gauss, grid = _gauss(sigma, dev), _grid(image_size, dev)
        out = torch.empty(P, K, 2, device=dev, dtype=torch.float32)
        _lib.check(_lib.load().umr_kp_transfer_flow(_ptr(kps), _ptr(fs), _ptr(ft), _ptr(gauss), _ptr(grid), _ptr(out), P, K,
                                                    F, fs.shape[2], image_size, sigma, _stream_ptr(dev)),
                   "umr_kp_transfer_flow")
    return out


def transfer_cam(kps_src, verts, cam_src, cam_tgt, mask_tgt, renderer):
    """Camera mode of test_kp.py:160-193 for P pairs: keypoints kps_src [P,K,2|3], mesh vertices verts [P,V,3] or
    [1,V,3] / [V,3] (the mean shape, shared), cameras cam_src / cam_tgt [P,7], target masks mask_tgt [P,S,S] (any non-zero
    value is foreground, as `nonzero` counts it) and the `SoftRenderer` whose `project_points` projects the vertices ->
    [P,K,2]: the grid coordinate of the target foreground pixel nearest to the target projection of the source vertex
    nearest to each keypoint.  A pair with an empty mask gives NaN (the reference fails there)."""
    _need_cuda(kps_src, verts, cam_src, cam_tgt, mask_tgt)
    kps = _keypoints(kps_src)
    P, K = kps.shape[:2]
    if mask_tgt.dim() != 3 or mask_tgt.shape[0] != P or mask_tgt.shape[1] != mask_tgt.shape[2]:
        raise ValueError("kp_transfer: mask_tgt must be [P,S,S] with P = %d, got %s" % (P, tuple(mask_tgt.shape)))
    if cam_src.shape != (P, 7) or cam_tgt.shape != (P, 7):
        raise ValueError("kp_transfer: cameras must be [P,7] with P = %d, got %s and %s"
                         % (P, tuple(cam_src.shape), tuple(cam_tgt.shape)))
    if verts.dim() == 2:
        verts = verts[None]
    if verts.dim() != 3 or verts.shape[2] != 3 or verts.shape[0] not in (1, P):
        raise ValueError("kp_transfer: verts must be [P,V,3], [1,V,3] or [V,3], got %s" % (tuple(verts.shape),))
    verts = verts.detach().expand(P, -1, -1)
    S = mask_tgt.shape[1]
    dev = kps.device
    with torch.no_grad(), torch.cuda.device(dev):
        proj_src = _pairs(renderer.project_points(verts, cam_src.detach()).to(torch.float32).contiguous())
        proj_tgt = _pairs(renderer.project_points(verts, cam_tgt.detach()).to(torch.float32).contiguous())
        mask = mask_tgt.detach().to(torch.float32).contiguous()
        grid = _grid(S, dev)
        out = torch.empty(P, K, 2, device=dev, dtype=torch.float32)
        _lib.check(_lib.load().umr_kp_transfer_cam(_ptr(kps), _ptr(proj_src), _ptr(proj_tgt), _ptr(mask), _ptr(grid),
                                                   _ptr(out), P, K, proj_src.shape[1], S, _stream_ptr(dev)),
                   "umr_kp_transfer_cam")
    return out


def pck(pred, gt, vis, err_scaling, thresholds=(0.1, 0.15)):
    """PCK of test_kp.py:254-258,316-322: pred / gt [N,K,2] keypoints, vis [N,K] visibility (0/1) -> one float per
    threshold: per keypoint, the fraction of its visible rows whose error sqrt(sum (pred - gt)^2) * err_scaling is below
    the threshold, then the mean over keypoints.  A keypoint visible in no row makes the mean NaN, as in the reference.
    Computed on the host in numpy float32, as the reference computes it."""
    def host(a):
        return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    pred, gt, vis = host(pred).astype(np.float32), host(gt).astype(np.float32), host(vis).astype(np.float32)
    if pred.shape != gt.shape or pred.ndim != 3 or pred.shape[2] != 2 or vis.shape != pred.shape[:2]:
        raise ValueError("pck: pred / gt must be [N,K,2] and vis [N,K], got %s, %s, %s" % (pred.shape, gt.shape, vis.shape))
    err = pred - gt
    err = np.sqrt(np.sum(err * err, axis=2)) * err_scaling
    n_vis = np.sum(vis, axis=0)
    with np.errstate(invalid="ignore", divide="ignore"):
        return tuple(float((np.sum((err < t) * vis, axis=0) / n_vis).mean()) for t in thresholds)
