"""torch.autograd bindings of the geometric-loss kernels (C ABI: include/umr_b200.h).

CUDA only: there is no CPU fallback (the CPU oracles live in oracle/ and are test infrastructure).

Under torch.use_deterministic_algorithms(True) the Functions whose default kernels sum with float atomics call the
`*_deterministic` symbols instead (bitwise reproducible, DESIGN.md §2).  The flag is read once in `forward` and kept in
`ctx`, so a backward runs in the mode of its forward.

Dtype rule of the loss Functions (DESIGN.md §10): an op computes in float64, with the `*_f64` symbols, when any of its
floating-point tensor inputs is float64.  It then returns float64 values and each input's gradient in that input's dtype.
The float64 kernels are always bitwise reproducible, so the deterministic flag does not change them.  Every other dtype
(float32, half) computes in float32 as before.  The choice is made in `forward` and kept in `ctx`.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .raster import _ptr, _stream_ptr


def _need_cuda(*ts):
    for t in ts:
        if not t.is_cuda:
            raise TypeError("umr_b200 ops support only cuda Tensors")


def _workspace(nbytes, device):
    """Device scratch of a deterministic call (an allocation, no fill: CUDA-graph safe)."""
    return torch.empty(nbytes, device=device, dtype=torch.uint8)


def vertex_incidence(index, num_vertices):
    """Transposed index table of the deterministic gathers: `index` (any shape, values in [0, num_vertices)) ->
    (rowptr [V+1], positions) int32 numpy arrays, where positions[rowptr[v]:rowptr[v+1]] are the flat positions k with
    index.flat[k] == v in ascending order.  The flatten loss passes its [E,4] edge table (position = edge * 4 + role), the
    part-chamfer loss its vertex selection [NS] (position = j)."""
    flat = np.asarray(index, dtype=np.int64).reshape(-1)
    if flat.size and (flat.min() < 0 or flat.max() >= num_vertices):
        raise IndexError("vertex index out of range for a mesh of %d vertices" % num_vertices)
    positions = np.argsort(flat, kind="stable").astype(np.int32)
    rowptr = np.zeros(num_vertices + 1, np.int64)
    np.cumsum(np.bincount(flat, minlength=num_vertices), out=rowptr[1:])
    return rowptr.astype(np.int32), positions


def device_incidence(keys, rows):
    """The same transposed table, built on the keys' device: keys (any shape, integer) -> (rowptr [rows+1],
    positions [keys.numel()]) int32 tensors, where positions[rowptr[r]:rowptr[r+1]] are the flat positions k with
    keys.flat[k] == r in ascending order.  Keys outside [0, rows) are dropped: they sort past the last row, so they sit
    after rowptr[rows].  Torch ops only (a stable sort and a searchsorted), which are deterministic, need no host
    synchronisation and can be captured in a CUDA graph.  Used by the deterministic backwards of the vertex pipeline
    (vertex -> face corners) and of the sampler's image gradient (pixel cell -> samples)."""
    flat = keys.reshape(-1).long()
    if flat.numel() > 2 ** 31 - 1 or rows > 2 ** 31 - 2:
        raise ValueError("device_incidence: %d positions over %d rows do not fit int32" % (flat.numel(), rows))
    flat = flat.masked_fill((flat < 0) | (flat >= rows), rows)
    sorted_keys, positions = torch.sort(flat, stable=True)
    rowptr = torch.searchsorted(sorted_keys, torch.arange(rows + 1, device=flat.device, dtype=torch.int64))
    return rowptr.to(torch.int32), positions.to(torch.int32)


def _incidence_on(index, num_vertices, device):
    rowptr, pos = vertex_incidence(index.detach().cpu().numpy(), num_vertices)
    return torch.from_numpy(rowptr).to(device), torch.from_numpy(pos).to(device)


def _batch_view(t, inner, dtype=torch.float32):
    """(tensor, batch stride in elements) if `t` [B, ...] is dense within each batch item, else a copy."""
    B = t.shape[0]
    if t[0].is_contiguous() and t.dtype == dtype:
        return t, (t.stride(0) if B > 1 else inner)
    t = t.contiguous().to(dtype)
    return t, inner


def _is_f64(*ts):
    """The dtype rule: float64 when any floating-point tensor among `ts` (None entries skipped) is float64."""
    return any(t is not None and t.dtype == torch.float64 for t in ts)


def _f64(t):
    """Detached, contiguous, float64."""
    return t.detach().contiguous().double()


# -------------------------------------------------------------------------------------------------
# bilinear texture-flow sampler
# -------------------------------------------------------------------------------------------------
class BilinearSampleFunction(torch.autograd.Function):
    """images [B,C,H,W], flow [B,N,2] -> out [B,N,C]; bilinear, zeros padding, align_corners=True
    (the torch-1.1 semantics the reference was written for: geom_utils.py:55, loss_utils.py:64)."""

    @staticmethod
    def forward(ctx, images, flow):
        _need_cuda(images, flow)
        ctx.f64 = _is_f64(images, flow)
        if ctx.f64:
            return BilinearSampleFunction._forward_f64(ctx, images, flow)
        lib = _lib.load()
        img = images.detach().contiguous().float()
        fl = flow.detach().contiguous().float()
        B, C, H, W = img.shape
        N = fl.shape[1]
        with torch.cuda.device(img.device):
            out = torch.empty(B, N, C, device=img.device, dtype=torch.float32)
            rc = lib.umr_bilinear_sample_forward(_ptr(img), _ptr(fl), _ptr(out), B, C, H, W, N,
                                                 _stream_ptr(img.device))
        _lib.check(rc, "umr_bilinear_sample_forward")
        ctx.save_for_backward(img, fl)
        ctx.img_grad = images.requires_grad
        ctx.det = torch.are_deterministic_algorithms_enabled()   # the forward has no atomics; the backward's mode
        return out

    @staticmethod
    def backward(ctx, grad_out):
        if ctx.f64:
            return BilinearSampleFunction._backward_f64(ctx, grad_out)
        lib = _lib.load()
        img, fl = ctx.saved_tensors
        B, C, H, W = img.shape
        N = fl.shape[1]
        g = grad_out.contiguous().float()
        with torch.cuda.device(img.device):
            gflow = torch.empty_like(fl)
            gimg = torch.empty_like(img) if ctx.img_grad else None
            if ctx.det:
                rowptr = samples = None
                if gimg is not None:   # samples keyed by their top-left cell, then the cell -> samples table
                    cells = torch.empty(B, N, device=img.device, dtype=torch.int32)
                    _lib.check(lib.umr_bilinear_sample_cells(_ptr(fl), _ptr(cells), B, H, W, N, _stream_ptr(img.device)),
                               "umr_bilinear_sample_cells")
                    rowptr, samples = device_incidence(cells, B * (H + 1) * (W + 1))
                rc = lib.umr_bilinear_sample_backward_deterministic(_ptr(img), _ptr(fl), _ptr(g), _ptr(gflow), _ptr(gimg),
                                                                    B, C, H, W, N, _ptr(rowptr), _ptr(samples),
                                                                    _stream_ptr(img.device))
            else:
                rc = lib.umr_bilinear_sample_backward(_ptr(img), _ptr(fl), _ptr(g), _ptr(gflow), _ptr(gimg),
                                                      B, C, H, W, N, _stream_ptr(img.device))
        _lib.check(rc, "umr_bilinear_sample_backward_deterministic" if ctx.det else "umr_bilinear_sample_backward")
        return gimg, gflow

    @staticmethod
    def _forward_f64(ctx, images, flow):
        lib = _lib.load()
        img, fl = _f64(images), _f64(flow)
        B, C, H, W = img.shape
        N = fl.shape[1]
        with torch.cuda.device(img.device):
            out = torch.empty(B, N, C, device=img.device, dtype=torch.float64)
            rc = lib.umr_bilinear_sample_forward_f64(_ptr(img), _ptr(fl), _ptr(out), B, C, H, W, N, _stream_ptr(img.device))
        _lib.check(rc, "umr_bilinear_sample_forward_f64")
        ctx.save_for_backward(img, fl)
        ctx.img_grad = images.requires_grad
        ctx.dtypes = (images.dtype, flow.dtype)
        return out

    @staticmethod
    def _backward_f64(ctx, grad_out):
        lib = _lib.load()
        img, fl = ctx.saved_tensors
        B, C, H, W = img.shape
        N = fl.shape[1]
        g = grad_out.contiguous().double()
        with torch.cuda.device(img.device):
            gflow = torch.empty_like(fl)
            gimg = rowptr = samples = None
            if ctx.img_grad:   # the image gradient is a gather over the cell -> samples table of the double coordinates
                gimg = torch.empty_like(img)
                cells = torch.empty(B, N, device=img.device, dtype=torch.int32)
                _lib.check(lib.umr_bilinear_sample_cells_f64(_ptr(fl), _ptr(cells), B, H, W, N, _stream_ptr(img.device)),
                           "umr_bilinear_sample_cells_f64")
                rowptr, samples = device_incidence(cells, B * (H + 1) * (W + 1))
            rc = lib.umr_bilinear_sample_backward_f64(_ptr(img), _ptr(fl), _ptr(g), _ptr(gflow), _ptr(gimg), B, C, H, W, N,
                                                      _ptr(rowptr), _ptr(samples), _stream_ptr(img.device))
        _lib.check(rc, "umr_bilinear_sample_backward_f64")
        return (gimg.to(ctx.dtypes[0]) if gimg is not None else None), gflow.to(ctx.dtypes[1])


def bilinear_sample(images, flow):
    return BilinearSampleFunction.apply(images, flow)


# -------------------------------------------------------------------------------------------------
# silhouette IoU
# -------------------------------------------------------------------------------------------------
class NegIouFunction(torch.autograd.Function):
    """predict/target [B, ...] -> per-image loss [B] = 1 - sum(p*t) / (sum(p+t-p*t) + 1e-6)."""

    @staticmethod
    def forward(ctx, predict, target):
        _need_cuda(predict, target)
        lib = _lib.load()
        B = predict.shape[0]
        if target.shape[0] != B or target.numel() != predict.numel():
            raise ValueError("neg_iou_loss: predict %s and target %s must hold the same number of elements per image"
                             % (tuple(predict.shape), tuple(target.shape)))
        ctx.f64 = _is_f64(predict, target)
        if ctx.f64:
            return NegIouFunction._forward_f64(ctx, predict, target)
        t = target.detach().contiguous().float().view(B, -1)
        N = t.shape[1]
        p, pbs = _batch_view(predict.detach(), N)  # e.g. the alpha plane of the RGBA render, read in place
        det = torch.are_deterministic_algorithms_enabled()
        with torch.cuda.device(p.device):
            inter = torch.empty(B, device=p.device, dtype=torch.float32)
            uni = torch.empty_like(inter)
            loss = torch.empty_like(inter)
            if det:
                ws = _workspace(lib.umr_iou_workspace_bytes_deterministic(B, N), p.device)
                rc = lib.umr_iou_forward_deterministic(_ptr(p), pbs, _ptr(t), _ptr(inter), _ptr(uni), _ptr(loss), B, N,
                                                       _ptr(ws), _stream_ptr(p.device))
            else:
                rc = lib.umr_iou_forward(_ptr(p), pbs, _ptr(t), _ptr(inter), _ptr(uni), _ptr(loss), B, N,
                                         _stream_ptr(p.device))
        _lib.check(rc, "umr_iou_forward_deterministic" if det else "umr_iou_forward")
        ctx.save_for_backward(t, inter, uni)
        ctx.shape = tuple(predict.shape)
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        if ctx.f64:
            return NegIouFunction._backward_f64(ctx, grad_loss)
        lib = _lib.load()
        t, inter, uni = ctx.saved_tensors
        B, N = t.shape
        g = grad_loss.contiguous().float()
        with torch.cuda.device(t.device):
            gp = torch.empty_like(t)
            rc = lib.umr_iou_backward(_ptr(t), _ptr(inter), _ptr(uni), _ptr(g), _ptr(gp), B, N,
                                      _stream_ptr(t.device))
        _lib.check(rc, "umr_iou_backward")
        return gp.view(ctx.shape), None

    @staticmethod
    def _forward_f64(ctx, predict, target):
        lib = _lib.load()
        B = predict.shape[0]
        t = _f64(target).view(B, -1)
        N = t.shape[1]
        p, pbs = _batch_view(predict.detach(), N, torch.float64)
        with torch.cuda.device(p.device):
            inter = torch.empty(B, device=p.device, dtype=torch.float64)
            uni = torch.empty_like(inter)
            loss = torch.empty_like(inter)
            ws = _workspace(lib.umr_iou_workspace_bytes_f64(B, N), p.device)
            rc = lib.umr_iou_forward_f64(_ptr(p), pbs, _ptr(t), _ptr(inter), _ptr(uni), _ptr(loss), B, N, _ptr(ws),
                                         _stream_ptr(p.device))
        _lib.check(rc, "umr_iou_forward_f64")
        ctx.save_for_backward(t, inter, uni)
        ctx.shape, ctx.dtype = tuple(predict.shape), predict.dtype
        return loss

    @staticmethod
    def _backward_f64(ctx, grad_loss):
        lib = _lib.load()
        t, inter, uni = ctx.saved_tensors
        B, N = t.shape
        g = grad_loss.contiguous().double()
        with torch.cuda.device(t.device):
            gp = torch.empty_like(t)
            rc = lib.umr_iou_backward_f64(_ptr(t), _ptr(inter), _ptr(uni), _ptr(g), _ptr(gp), B, N, _stream_ptr(t.device))
        _lib.check(rc, "umr_iou_backward_f64")
        return gp.view(ctx.shape).to(ctx.dtype), None


def neg_iou_per_image(predict, target):
    return NegIouFunction.apply(predict, target)


# -------------------------------------------------------------------------------------------------
# masked L1 texture loss
# -------------------------------------------------------------------------------------------------
class MaskedL1Function(torch.autograd.Function):
    """img_pred [B,C,H,W], img_gt [B,C,H,W], mask_gt [B,H,W], mask_pred [B,H,W] -> per-image
    mean |pred*mask_pred - gt*mask_gt| [B]  (loss_utils.py:103-116, avg=False form)."""

    @staticmethod
    def forward(ctx, img_pred, img_gt, mask_gt, mask_pred):
        _need_cuda(img_pred, img_gt, mask_gt, mask_pred)
        lib = _lib.load()
        B, C, H, W = img_pred.shape
        HW = H * W
        if tuple(img_gt.shape) != (B, C, H, W) or mask_gt.numel() != B * HW or mask_pred.numel() != B * HW:
            raise ValueError("texture_loss_masks: img_pred %s, img_gt %s, mask_gt %s, mask_pred %s do not match"
                             % (tuple(img_pred.shape), tuple(img_gt.shape), tuple(mask_gt.shape), tuple(mask_pred.shape)))
        ctx.f64 = _is_f64(img_pred, img_gt, mask_gt, mask_pred)
        if ctx.f64:
            return MaskedL1Function._forward_f64(ctx, img_pred, img_gt, mask_gt, mask_pred)
        p, pbs = _batch_view(img_pred.detach(), C * HW)
        mp, mbs = _batch_view(mask_pred.detach(), HW)
        g = img_gt.detach().contiguous().float()
        mg = mask_gt.detach().contiguous().float()
        det = torch.are_deterministic_algorithms_enabled()
        with torch.cuda.device(p.device):
            loss = torch.empty(B, device=p.device, dtype=torch.float32)
            if det:
                ws = _workspace(lib.umr_masked_l1_workspace_bytes_deterministic(B, HW), p.device)
                rc = lib.umr_masked_l1_forward_deterministic(_ptr(p), pbs, _ptr(mp), mbs, _ptr(g), _ptr(mg), _ptr(loss), B, C,
                                                             HW, _ptr(ws), _stream_ptr(p.device))
            else:
                rc = lib.umr_masked_l1_forward(_ptr(p), pbs, _ptr(mp), mbs, _ptr(g), _ptr(mg), _ptr(loss), B, C, HW,
                                               _stream_ptr(p.device))
        _lib.check(rc, "umr_masked_l1_forward_deterministic" if det else "umr_masked_l1_forward")
        ctx.save_for_backward(p, mp, g, mg)
        ctx.meta = (pbs, mbs, img_pred.requires_grad, mask_pred.requires_grad, tuple(img_pred.shape),
                    tuple(mask_pred.shape))
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        if ctx.f64:
            return MaskedL1Function._backward_f64(ctx, grad_loss)
        lib = _lib.load()
        p, mp, g, mg = ctx.saved_tensors
        pbs, mbs, need_p, need_m, pshape, mshape = ctx.meta
        B, C = pshape[0], pshape[1]
        HW = pshape[2] * pshape[3]
        gl = grad_loss.contiguous().float()
        with torch.cuda.device(p.device):
            gp = torch.empty(pshape, device=p.device, dtype=torch.float32) if need_p else None
            gm = torch.empty(mshape, device=p.device, dtype=torch.float32) if need_m else None
            rc = lib.umr_masked_l1_backward(_ptr(p), pbs, _ptr(mp), mbs, _ptr(g), _ptr(mg), _ptr(gl), _ptr(gp),
                                            _ptr(gm), B, C, HW, _stream_ptr(p.device))
        _lib.check(rc, "umr_masked_l1_backward")
        return gp, None, None, gm

    @staticmethod
    def _forward_f64(ctx, img_pred, img_gt, mask_gt, mask_pred):
        lib = _lib.load()
        B, C, H, W = img_pred.shape
        HW = H * W
        p, pbs = _batch_view(img_pred.detach(), C * HW, torch.float64)
        mp, mbs = _batch_view(mask_pred.detach(), HW, torch.float64)
        g, mg = _f64(img_gt), _f64(mask_gt)
        with torch.cuda.device(p.device):
            loss = torch.empty(B, device=p.device, dtype=torch.float64)
            ws = _workspace(lib.umr_masked_l1_workspace_bytes_f64(B, HW), p.device)
            rc = lib.umr_masked_l1_forward_f64(_ptr(p), pbs, _ptr(mp), mbs, _ptr(g), _ptr(mg), _ptr(loss), B, C, HW, _ptr(ws),
                                               _stream_ptr(p.device))
        _lib.check(rc, "umr_masked_l1_forward_f64")
        ctx.save_for_backward(p, mp, g, mg)
        ctx.meta = (pbs, mbs, img_pred.requires_grad, mask_pred.requires_grad, tuple(img_pred.shape), tuple(mask_pred.shape),
                    img_pred.dtype, mask_pred.dtype)
        return loss

    @staticmethod
    def _backward_f64(ctx, grad_loss):
        lib = _lib.load()
        p, mp, g, mg = ctx.saved_tensors
        pbs, mbs, need_p, need_m, pshape, mshape, pdtype, mdtype = ctx.meta
        B, C = pshape[0], pshape[1]
        HW = pshape[2] * pshape[3]
        gl = grad_loss.contiguous().double()
        with torch.cuda.device(p.device):
            gp = torch.empty(pshape, device=p.device, dtype=torch.float64) if need_p else None
            gm = torch.empty(mshape, device=p.device, dtype=torch.float64) if need_m else None
            rc = lib.umr_masked_l1_backward_f64(_ptr(p), pbs, _ptr(mp), mbs, _ptr(g), _ptr(mg), _ptr(gl), _ptr(gp), _ptr(gm),
                                                B, C, HW, _stream_ptr(p.device))
        _lib.check(rc, "umr_masked_l1_backward_f64")
        return (gp.to(pdtype) if gp is not None else None), None, None, (gm.to(mdtype) if gm is not None else None)


def masked_l1_per_image(img_pred, img_gt, mask_gt, mask_pred):
    return MaskedL1Function.apply(img_pred, img_gt, mask_gt, mask_pred)


# -------------------------------------------------------------------------------------------------
# fused loss head: w_iou * neg_iou_loss(alpha, mask) + w_tex * texture_loss_masks(rgb, gt, mask, alpha)
# -------------------------------------------------------------------------------------------------
class LossHeadFunction(torch.autograd.Function):
    """images [B,4,H,W] (one RGBA render), img_gt [B,3,H,W], mask_gt [B,H,W] -> (scalar loss, per_image [B,2]).
    One reduction + finalize forward, ONE backward kernel writing the whole [B,4,H,W] image gradient."""

    @staticmethod
    def forward(ctx, images, img_gt, mask_gt, w_iou, w_tex):
        _need_cuda(images, img_gt, mask_gt)
        lib = _lib.load()
        B, C, H, W = images.shape
        if C != 4 or tuple(img_gt.shape) != (B, 3, H, W) or mask_gt.numel() != B * H * W:
            raise ValueError("mask_texture_loss: images %s must be [B,4,H,W], img_gt %s [B,3,H,W], mask_gt %s [B,H,W]"
                             % (tuple(images.shape), tuple(img_gt.shape), tuple(mask_gt.shape)))
        ctx.f64 = _is_f64(images, img_gt, mask_gt)
        if ctx.f64:
            return LossHeadFunction._forward_f64(ctx, images, img_gt, mask_gt, w_iou, w_tex)
        x = images.detach().contiguous().float()
        g = img_gt.detach().contiguous().float()
        m = mask_gt.detach().contiguous().float()
        det = torch.are_deterministic_algorithms_enabled()
        with torch.cuda.device(x.device):
            stats = torch.empty(B, 3, device=x.device, dtype=torch.float32)
            per_image = torch.empty(B, 2, device=x.device, dtype=torch.float32)
            loss = torch.empty((), device=x.device, dtype=torch.float32)
            if det:
                ws = _workspace(lib.umr_loss_head_workspace_bytes_deterministic(B, H * W), x.device)
                rc = lib.umr_loss_head_forward_deterministic(_ptr(x), _ptr(g), _ptr(m), _ptr(stats), _ptr(per_image),
                                                             _ptr(loss), B, H * W, float(w_iou), float(w_tex), _ptr(ws),
                                                             _stream_ptr(x.device))
            else:
                rc = lib.umr_loss_head_forward(_ptr(x), _ptr(g), _ptr(m), _ptr(stats), _ptr(per_image), _ptr(loss), B,
                                               H * W, float(w_iou), float(w_tex), _stream_ptr(x.device))
        _lib.check(rc, "umr_loss_head_forward_deterministic" if det else "umr_loss_head_forward")
        ctx.save_for_backward(x, g, m, stats)
        ctx.w = (float(w_iou), float(w_tex))
        ctx.mark_non_differentiable(per_image)
        return loss, per_image

    @staticmethod
    def backward(ctx, grad_loss, _gp=None):
        if ctx.f64:
            return LossHeadFunction._backward_f64(ctx, grad_loss)
        lib = _lib.load()
        x, g, m, stats = ctx.saved_tensors
        B, _, H, W = x.shape
        gl = grad_loss.contiguous().float().reshape(1)
        with torch.cuda.device(x.device):
            gx = torch.empty_like(x)
            rc = lib.umr_loss_head_backward(_ptr(x), _ptr(g), _ptr(m), _ptr(stats), _ptr(gl), _ptr(gx), B, H * W,
                                            ctx.w[0], ctx.w[1], _stream_ptr(x.device))
        _lib.check(rc, "umr_loss_head_backward")
        return gx, None, None, None, None

    @staticmethod
    def _forward_f64(ctx, images, img_gt, mask_gt, w_iou, w_tex):
        lib = _lib.load()
        B, _, H, W = images.shape
        x, g, m = _f64(images), _f64(img_gt), _f64(mask_gt)
        with torch.cuda.device(x.device):
            stats = torch.empty(B, 3, device=x.device, dtype=torch.float64)
            per_image = torch.empty(B, 2, device=x.device, dtype=torch.float64)
            loss = torch.empty((), device=x.device, dtype=torch.float64)
            ws = _workspace(lib.umr_loss_head_workspace_bytes_f64(B, H * W), x.device)
            rc = lib.umr_loss_head_forward_f64(_ptr(x), _ptr(g), _ptr(m), _ptr(stats), _ptr(per_image), _ptr(loss), B, H * W,
                                               float(w_iou), float(w_tex), _ptr(ws), _stream_ptr(x.device))
        _lib.check(rc, "umr_loss_head_forward_f64")
        ctx.save_for_backward(x, g, m, stats)
        ctx.w = (float(w_iou), float(w_tex))
        ctx.dtype = images.dtype
        ctx.mark_non_differentiable(per_image)
        return loss, per_image

    @staticmethod
    def _backward_f64(ctx, grad_loss):
        lib = _lib.load()
        x, g, m, stats = ctx.saved_tensors
        B, _, H, W = x.shape
        gl = grad_loss.contiguous().double().reshape(1)
        with torch.cuda.device(x.device):
            gx = torch.empty_like(x)
            rc = lib.umr_loss_head_backward_f64(_ptr(x), _ptr(g), _ptr(m), _ptr(stats), _ptr(gl), _ptr(gx), B, H * W,
                                                ctx.w[0], ctx.w[1], _stream_ptr(x.device))
        _lib.check(rc, "umr_loss_head_backward_f64")
        return gx.to(ctx.dtype), None, None, None, None


def mask_texture_loss(images, img_gt, mask_gt, w_iou=1.0, w_tex=1.0):
    """-> (loss, per_image[B,2] = (1 - IoU, masked L1)) with loss == w_iou * neg_iou_loss(images[:,3], mask_gt) +
    w_tex * texture_loss_masks(images[:,:3], img_gt, mask_gt, images[:,3])."""
    return LossHeadFunction.apply(images, img_gt, mask_gt, w_iou, w_tex)


# -------------------------------------------------------------------------------------------------
# chamfer
# -------------------------------------------------------------------------------------------------
class ChamferFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        _need_cuda(a, b)
        ctx.f64 = _is_f64(a, b)
        if ctx.f64:
            return ChamferFunction._forward_f64(ctx, a, b)
        lib = _lib.load()
        x = a.detach().contiguous().float()
        y = b.detach().contiguous().float()
        B, N, D = x.shape
        M = y.shape[1]
        with torch.cuda.device(x.device):
            d_ab = torch.empty(B, N, device=x.device, dtype=torch.float32)
            d_ba = torch.empty(B, M, device=x.device, dtype=torch.float32)
            i_ab = torch.empty(B, N, device=x.device, dtype=torch.int32)
            i_ba = torch.empty(B, M, device=x.device, dtype=torch.int32)
            rc = lib.umr_chamfer_forward(_ptr(x), _ptr(y), _ptr(d_ab), _ptr(d_ba), _ptr(i_ab), _ptr(i_ba),
                                         B, N, M, D, _stream_ptr(x.device))
        _lib.check(rc, "umr_chamfer_forward")
        ctx.save_for_backward(x, y, i_ab, i_ba)
        ctx.mark_non_differentiable(i_ab, i_ba)
        ctx.det = torch.are_deterministic_algorithms_enabled()   # the forward has no atomics; the backward's mode
        return d_ab, d_ba, i_ab, i_ba

    @staticmethod
    def backward(ctx, g_ab, g_ba, _1=None, _2=None):
        if ctx.f64:
            return ChamferFunction._backward_f64(ctx, g_ab, g_ba)
        lib = _lib.load()
        x, y, i_ab, i_ba = ctx.saved_tensors
        B, N, D = x.shape
        M = y.shape[1]
        g1 = g_ab.contiguous().float() if g_ab is not None else None
        g2 = g_ba.contiguous().float() if g_ba is not None else None
        with torch.cuda.device(x.device):
            gx = torch.empty_like(x)
            gy = torch.empty_like(y)
            bwd = lib.umr_chamfer_backward_deterministic if ctx.det else lib.umr_chamfer_backward
            rc = bwd(_ptr(x), _ptr(y), _ptr(i_ab), _ptr(i_ba), _ptr(g1), _ptr(g2), _ptr(gx), _ptr(gy), B, N, M, D,
                     _stream_ptr(x.device))
        _lib.check(rc, "umr_chamfer_backward_deterministic" if ctx.det else "umr_chamfer_backward")
        return gx, gy

    @staticmethod
    def _forward_f64(ctx, a, b):
        lib = _lib.load()
        x, y = _f64(a), _f64(b)
        B, N, D = x.shape
        M = y.shape[1]
        with torch.cuda.device(x.device):
            d_ab = torch.empty(B, N, device=x.device, dtype=torch.float64)
            d_ba = torch.empty(B, M, device=x.device, dtype=torch.float64)
            i_ab = torch.empty(B, N, device=x.device, dtype=torch.int32)
            i_ba = torch.empty(B, M, device=x.device, dtype=torch.int32)
            rc = lib.umr_chamfer_forward_f64(_ptr(x), _ptr(y), _ptr(d_ab), _ptr(d_ba), _ptr(i_ab), _ptr(i_ba), B, N, M, D,
                                             _stream_ptr(x.device))
        _lib.check(rc, "umr_chamfer_forward_f64")
        ctx.save_for_backward(x, y, i_ab, i_ba)
        ctx.mark_non_differentiable(i_ab, i_ba)
        ctx.dtypes = (a.dtype, b.dtype)
        return d_ab, d_ba, i_ab, i_ba

    @staticmethod
    def _backward_f64(ctx, g_ab, g_ba):
        lib = _lib.load()
        x, y, i_ab, i_ba = ctx.saved_tensors
        B, N, D = x.shape
        M = y.shape[1]
        g1 = g_ab.contiguous().double() if g_ab is not None else None
        g2 = g_ba.contiguous().double() if g_ba is not None else None
        with torch.cuda.device(x.device):
            gx = torch.empty_like(x)
            gy = torch.empty_like(y)
            rc = lib.umr_chamfer_backward_f64(_ptr(x), _ptr(y), _ptr(i_ab), _ptr(i_ba), _ptr(g1), _ptr(g2), _ptr(gx), _ptr(gy),
                                              B, N, M, D, _stream_ptr(x.device))
        _lib.check(rc, "umr_chamfer_backward_f64")
        return gx.to(ctx.dtypes[0]), gy.to(ctx.dtypes[1])


def dist_chamfer(a, b):
    return ChamferFunction.apply(a, b)


# -------------------------------------------------------------------------------------------------
# texture cycle
# -------------------------------------------------------------------------------------------------
class TexCycleFunction(torch.autograd.Function):
    """flow [B,F,T2,2], prob [B,F,2], face_ids [B,P] (float plane, -1 = background) -> scalar loss.
    `visible` [B,F] uint8 (from raster.visibility(..., want_faces=True)) replaces the scan of the plane."""

    @staticmethod
    def forward(ctx, flow, prob, face_ids, visible=None):
        _need_cuda(flow, prob) if face_ids is None else _need_cuda(flow, prob, face_ids)
        ctx.f64 = _is_f64(flow, prob, face_ids)
        if ctx.f64:
            return TexCycleFunction._forward_f64(ctx, flow, prob, face_ids, visible)
        lib = _lib.load()
        fl = flow.detach().contiguous().float()
        pr = prob.detach().contiguous().float()
        B, F, T2 = fl.shape[0], fl.shape[1], fl.shape[2]
        if visible is not None:
            if visible.dtype != torch.uint8 or tuple(visible.shape) != (B, F) or not visible.is_cuda:
                raise ValueError("visible must be a CUDA uint8 tensor of shape [B,F]")
            ids, P = None, 0
        else:
            ids = face_ids.detach().contiguous().float()
            P = ids.shape[1]
        det = torch.are_deterministic_algorithms_enabled()
        with torch.cuda.device(fl.device):
            vis = visible.contiguous() if visible is not None else torch.empty(B, F, device=fl.device, dtype=torch.uint8)
            loss = torch.empty(1, device=fl.device, dtype=torch.float32)
            if det:
                ws = _workspace(lib.umr_texcycle_workspace_bytes_deterministic(B, F), fl.device)
                rc = lib.umr_texcycle_forward_deterministic(_ptr(fl), _ptr(pr), _ptr(ids), _ptr(vis), _ptr(loss), B, F, T2,
                                                            P, _ptr(ws), _stream_ptr(fl.device))
            else:
                rc = lib.umr_texcycle_forward(_ptr(fl), _ptr(pr), _ptr(ids), _ptr(vis), _ptr(loss), B, F, T2, P,
                                              _stream_ptr(fl.device))
        _lib.check(rc, "umr_texcycle_forward_deterministic" if det else "umr_texcycle_forward")
        ctx.save_for_backward(fl, pr, vis)
        return loss.view(())

    @staticmethod
    def backward(ctx, grad_loss):
        if ctx.f64:
            return TexCycleFunction._backward_f64(ctx, grad_loss)
        lib = _lib.load()
        fl, pr, vis = ctx.saved_tensors
        B, F, T2 = fl.shape[0], fl.shape[1], fl.shape[2]
        g = grad_loss.contiguous().float().view(1)
        with torch.cuda.device(fl.device):
            gflow = torch.empty_like(fl)
            rc = lib.umr_texcycle_backward(_ptr(fl), _ptr(pr), _ptr(vis), _ptr(g), _ptr(gflow), B, F, T2,
                                           _stream_ptr(fl.device))
        _lib.check(rc, "umr_texcycle_backward")
        return gflow, None, None, None

    @staticmethod
    def _forward_f64(ctx, flow, prob, face_ids, visible):
        lib = _lib.load()
        fl, pr = _f64(flow), _f64(prob)
        B, F, T2 = fl.shape[0], fl.shape[1], fl.shape[2]
        if visible is not None:
            if visible.dtype != torch.uint8 or tuple(visible.shape) != (B, F) or not visible.is_cuda:
                raise ValueError("visible must be a CUDA uint8 tensor of shape [B,F]")
            ids, P = None, 0
        else:
            # the visibility bitmap reads a float32 plane: face ids (and the background's -1) are integers below
            # UMR_RASTER_MAX_FACES = 2^24, which float32 holds exactly, so a float64 plane converts without rounding
            ids = face_ids.detach().contiguous().float()
            P = ids.shape[1]
        with torch.cuda.device(fl.device):
            vis = visible.contiguous() if visible is not None else torch.empty(B, F, device=fl.device, dtype=torch.uint8)
            loss = torch.empty(1, device=fl.device, dtype=torch.float64)
            ws = _workspace(lib.umr_texcycle_workspace_bytes_f64(B, F), fl.device)
            rc = lib.umr_texcycle_forward_f64(_ptr(fl), _ptr(pr), _ptr(ids), _ptr(vis), _ptr(loss), B, F, T2, P, _ptr(ws),
                                              _stream_ptr(fl.device))
        _lib.check(rc, "umr_texcycle_forward_f64")
        ctx.save_for_backward(fl, pr, vis)
        ctx.dtype = flow.dtype
        return loss.view(())

    @staticmethod
    def _backward_f64(ctx, grad_loss):
        lib = _lib.load()
        fl, pr, vis = ctx.saved_tensors
        B, F, T2 = fl.shape[0], fl.shape[1], fl.shape[2]
        g = grad_loss.contiguous().double().view(1)
        with torch.cuda.device(fl.device):
            gflow = torch.empty_like(fl)
            rc = lib.umr_texcycle_backward_f64(_ptr(fl), _ptr(pr), _ptr(vis), _ptr(g), _ptr(gflow), B, F, T2,
                                               _stream_ptr(fl.device))
        _lib.check(rc, "umr_texcycle_backward_f64")
        return gflow.to(ctx.dtype), None, None, None


def tex_cycle(flow, prob, face_ids=None, visible=None):
    return TexCycleFunction.apply(flow, prob, face_ids, visible)


# -------------------------------------------------------------------------------------------------
# mesh regularisers (SoftRas/losses.py) and the barrier distance transform (utils/image.py)
# -------------------------------------------------------------------------------------------------
class LaplacianFunction(torch.autograd.Function):
    """x [B,V,3] + CSR neighbour table -> per-sample |L x|^2 [B] (SoftRas/losses.py:31-37)."""

    @staticmethod
    def forward(ctx, x, rowptr, col, coef, tcoef):
        _need_cuda(x)
        ctx.f64 = _is_f64(x, coef, tcoef)
        if ctx.f64:
            return LaplacianFunction._forward_f64(ctx, x, rowptr, col, coef, tcoef)
        lib = _lib.load()
        xx = x.detach().contiguous().float()
        B, V = xx.shape[:2]
        det = torch.are_deterministic_algorithms_enabled()
        with torch.cuda.device(xx.device):
            y = torch.empty_like(xx)
            loss = torch.empty(B, device=xx.device, dtype=torch.float32)
            if det:
                ws = _workspace(lib.umr_laplacian_workspace_bytes_deterministic(B, V), xx.device)
                rc = lib.umr_laplacian_forward_deterministic(_ptr(xx), _ptr(rowptr), _ptr(col), _ptr(coef), _ptr(y),
                                                             _ptr(loss), B, V, _ptr(ws), _stream_ptr(xx.device))
            else:
                rc = lib.umr_laplacian_forward(_ptr(xx), _ptr(rowptr), _ptr(col), _ptr(coef), _ptr(y), _ptr(loss), B, V,
                                               _stream_ptr(xx.device))
        _lib.check(rc, "umr_laplacian_forward_deterministic" if det else "umr_laplacian_forward")
        ctx.save_for_backward(y, rowptr, col, tcoef)
        return loss

    @staticmethod
    def backward(ctx, g):
        if ctx.f64:
            return LaplacianFunction._backward_f64(ctx, g)
        lib = _lib.load()
        y, rowptr, col, tcoef = ctx.saved_tensors
        B, V = y.shape[:2]
        gl = g.contiguous().float()
        with torch.cuda.device(y.device):
            gx = torch.empty_like(y)
            rc = lib.umr_laplacian_backward(_ptr(y), _ptr(rowptr), _ptr(col), _ptr(tcoef), _ptr(gl), _ptr(gx), B, V,
                                            _stream_ptr(y.device))
        _lib.check(rc, "umr_laplacian_backward")
        return gx, None, None, None, None

    @staticmethod
    def _forward_f64(ctx, x, rowptr, col, coef, tcoef):
        lib = _lib.load()
        xx = _f64(x)
        B, V = xx.shape[:2]
        c, tc = _f64(coef), _f64(tcoef)   # the module's float32 -1/deg entries widen exactly
        with torch.cuda.device(xx.device):
            y = torch.empty_like(xx)
            loss = torch.empty(B, device=xx.device, dtype=torch.float64)
            ws = _workspace(lib.umr_laplacian_workspace_bytes_f64(B, V), xx.device)
            rc = lib.umr_laplacian_forward_f64(_ptr(xx), _ptr(rowptr), _ptr(col), _ptr(c), _ptr(y), _ptr(loss), B, V, _ptr(ws),
                                               _stream_ptr(xx.device))
        _lib.check(rc, "umr_laplacian_forward_f64")
        ctx.save_for_backward(y, rowptr, col, tc)
        ctx.dtype = x.dtype
        return loss

    @staticmethod
    def _backward_f64(ctx, g):
        lib = _lib.load()
        y, rowptr, col, tcoef = ctx.saved_tensors
        B, V = y.shape[:2]
        gl = g.contiguous().double()
        with torch.cuda.device(y.device):
            gx = torch.empty_like(y)
            rc = lib.umr_laplacian_backward_f64(_ptr(y), _ptr(rowptr), _ptr(col), _ptr(tcoef), _ptr(gl), _ptr(gx), B, V,
                                                _stream_ptr(y.device))
        _lib.check(rc, "umr_laplacian_backward_f64")
        return gx.to(ctx.dtype), None, None, None, None


class FlattenFunction(torch.autograd.Function):
    """vertices [B,V,3] + edge table [E,4] int32 -> per-sample sum_e (cos + 1)^2 [B] (SoftRas/losses.py:71-114).
    `vert_rowptr` / `vert_incidence`: the edge table's transposed incidence (`vertex_incidence(edges, V)` on the device),
    used by the deterministic backward; FlattenLoss builds it once.  Without it a deterministic call builds it here (a
    device-to-host copy of the edge table)."""

    @staticmethod
    def forward(ctx, vertices, edges, eps, vert_rowptr=None, vert_incidence=None):
        _need_cuda(vertices)
        ctx.f64 = _is_f64(vertices)
        lib = _lib.load()
        v = _f64(vertices) if ctx.f64 else vertices.detach().contiguous().float()
        B, V = v.shape[:2]
        E = edges.shape[0]
        det = torch.are_deterministic_algorithms_enabled()
        with torch.cuda.device(v.device):
            loss = torch.empty(B, device=v.device, dtype=v.dtype)
            if ctx.f64:
                ws = _workspace(lib.umr_flatten_forward_workspace_bytes_f64(B, E), v.device)
                rc = lib.umr_flatten_forward_f64(_ptr(v), _ptr(edges), _ptr(loss), B, V, E, float(eps), _ptr(ws),
                                                 _stream_ptr(v.device))
            elif det:
                ws = _workspace(lib.umr_flatten_forward_workspace_bytes_deterministic(B, E), v.device)
                rc = lib.umr_flatten_forward_deterministic(_ptr(v), _ptr(edges), _ptr(loss), B, V, E, float(eps), _ptr(ws),
                                                           _stream_ptr(v.device))
            else:
                rc = lib.umr_flatten_forward(_ptr(v), _ptr(edges), _ptr(loss), B, V, E, float(eps), _stream_ptr(v.device))
        _lib.check(rc, "umr_flatten_forward_f64" if ctx.f64 else
                   "umr_flatten_forward_deterministic" if det else "umr_flatten_forward")
        det = det or ctx.f64   # the float64 backward is a gather too: it needs the transposed table
        ctx.dtype = vertices.dtype
        if det:
            if vert_rowptr is None or vert_incidence is None:
                vert_rowptr, vert_incidence = _incidence_on(edges, V, v.device)
            elif vert_rowptr.numel() < V + 1:   # vertices beyond the table's are on no edge
                vert_rowptr = torch.cat((vert_rowptr, vert_rowptr[-1:].expand(V + 1 - vert_rowptr.numel())))
            elif vert_rowptr.numel() > V + 1:
                raise ValueError("flatten loss: the edge table indexes %d vertices, the mesh has %d"
                                 % (vert_rowptr.numel() - 1, V))
            ctx.save_for_backward(v, edges, vert_rowptr, vert_incidence)
        else:
            ctx.save_for_backward(v, edges)
        ctx.eps = float(eps)
        ctx.det = det
        return loss

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        v, edges = ctx.saved_tensors[:2]
        B, V = v.shape[:2]
        E = edges.shape[0]
        gl = g.contiguous().to(v.dtype)
        with torch.cuda.device(v.device):
            gv = torch.empty_like(v)
            if ctx.f64:
                rowptr, inc = ctx.saved_tensors[2:]
                ws = _workspace(lib.umr_flatten_backward_workspace_bytes_f64(B, E), v.device)
                rc = lib.umr_flatten_backward_f64(_ptr(v), _ptr(edges), _ptr(rowptr), _ptr(inc), _ptr(gl), _ptr(gv), B, V, E,
                                                  ctx.eps, _ptr(ws), _stream_ptr(v.device))
            elif ctx.det:
                rowptr, inc = ctx.saved_tensors[2:]
                ws = _workspace(lib.umr_flatten_backward_workspace_bytes_deterministic(B, E), v.device)
                rc = lib.umr_flatten_backward_deterministic(_ptr(v), _ptr(edges), _ptr(rowptr), _ptr(inc), _ptr(gl), _ptr(gv),
                                                            B, V, E, ctx.eps, _ptr(ws), _stream_ptr(v.device))
            else:
                rc = lib.umr_flatten_backward(_ptr(v), _ptr(edges), _ptr(gl), _ptr(gv), B, V, E, ctx.eps,
                                              _stream_ptr(v.device))
        _lib.check(rc, "umr_flatten_backward_f64" if ctx.f64 else
                   "umr_flatten_backward_deterministic" if ctx.det else "umr_flatten_backward")
        return gv.to(ctx.dtype), None, None, None, None


def dt_barrier(masks, k=50.0):
    """utils/image.py:130-141 `compute_dt_barrier` for a batch on the GPU: masks [B,H,W] or [H,W] -> same shape float32,
    exact Euclidean distances (the reference runs scipy on the host per image per step).  As in scipy, the outside
    distance is measured to the pixels equal to 1 and the inside distance to the pixels equal to 0; a value in between
    (the edge of a bilinearly resized mask) is neither."""
    _need_cuda(masks)
    lib = _lib.load()
    m = masks.detach().float()
    squeeze = m.dim() == 2
    if squeeze:
        m = m[None]
    m = m.contiguous()
    B, H, W = m.shape
    with torch.cuda.device(m.device):
        out = torch.empty_like(m)
        ws = torch.empty(lib.umr_dt_barrier_workspace_bytes(B, H, W), device=m.device, dtype=torch.uint8)
        rc = lib.umr_dt_barrier(_ptr(m), _ptr(out), _ptr(ws), B, H, W, float(k), _stream_ptr(m.device))
    _lib.check(rc, "umr_dt_barrier")
    return out[0] if squeeze else out


def create_texture_image(faces_uv, textures, image, eps=1e-5):
    """SoftRas cuda/create_texture_image (in place on `image` [H,W,3]); faces_uv [F,3,2], textures [F,R*R,3]."""
    _need_cuda(faces_uv, textures, image)
    lib = _lib.load()
    f = faces_uv.contiguous().float()
    t = textures.contiguous().float()
    if not image.is_contiguous() or image.dtype != torch.float32:
        raise ValueError("image must be a contiguous float32 [H,W,3] tensor")
    F_ = t.shape[0]
    R = int(round(t.shape[1] ** 0.5))
    rc = lib.umr_create_texture_image(_ptr(f), _ptr(t), _ptr(image), F_, R, image.shape[0], image.shape[1], float(eps),
                                      _stream_ptr(image.device))
    _lib.check(rc, "umr_create_texture_image")
    return image


def load_textures(image, faces_uv, textures, is_update):
    """SoftRas cuda/load_textures (in place on `textures` [F,R*R,3]); image [H,W,3], faces_uv [F,3,2], is_update [F] int32."""
    _need_cuda(image, faces_uv, textures, is_update)
    lib = _lib.load()
    img = image.contiguous().float()
    f = faces_uv.contiguous().float()
    u = is_update.contiguous().int()
    if not textures.is_contiguous() or textures.dtype != torch.float32:
        raise ValueError("textures must be a contiguous float32 [F,R*R,3] tensor")
    R = int(round(textures.shape[1] ** 0.5))
    rc = lib.umr_load_textures(_ptr(img), _ptr(f), _ptr(u), _ptr(textures), textures.shape[0], R, img.shape[0], img.shape[1],
                               _stream_ptr(textures.device))
    _lib.check(rc, "umr_load_textures")
    return textures


# -------------------------------------------------------------------------------------------------
# CorrLossChamfer fused (nnutils/loss_utils.py:218-248)
# -------------------------------------------------------------------------------------------------
class CorrChamferFunction(torch.autograd.Function):
    """verts [B,V,3] (or [1,V,3] / an expanded view: one mesh for all renders), cams [B,7], selection [NS] int32 (the four
    parts' vertex indices concatenated), targets = 4 tensors [B,m_g,2], part_ends (4 cumulative counts), weights (4 floats)
    -> (loss [B], vert2d [B,NS,2]).  One kernel per direction instead of ~250 torch launches.  `vert_rowptr` /
    `vert_selection`: the selection's transposed table (`vertex_incidence(selection, V)` on the device) for the
    deterministic backward; CorrLossChamfer caches it.  Without it a deterministic call builds it here (a device-to-host
    copy of the selection)."""

    @staticmethod
    def _cfg(targets, part_ends, weights, wtype=ctypes.c_float):
        tp = (ctypes.c_void_p * 4)(*[t.data_ptr() for t in targets])
        tc = (ctypes.c_int32 * 4)(*[int(t.shape[1]) for t in targets])
        pe = (ctypes.c_int32 * 4)(*[int(e) for e in part_ends])
        wt = (wtype * 4)(*[float(w) for w in weights])
        return tp, tc, pe, wt

    @staticmethod
    def forward(ctx, verts, cams, selection, t0, t1, t2, t3, part_ends, weights, vert_rowptr=None, vert_selection=None):
        _need_cuda(verts, cams, selection, t0, t1, t2, t3)
        lib = _lib.load()
        ctx.f64 = _is_f64(verts, cams, t0, t1, t2, t3)
        dtype = torch.float64 if ctx.f64 else torch.float32
        B = cams.shape[0]
        shared = verts.shape[0] == 1 or (verts.dim() == 3 and verts.stride(0) == 0)   # one mesh for every render
        vv = (verts[:1] if shared else verts).detach().contiguous().to(dtype)
        if not shared and vv.shape[0] != B:
            raise ValueError("verts batch %d does not match cams batch %d" % (vv.shape[0], B))
        V = vv.shape[1]
        cc = cams.detach().contiguous().to(dtype)
        targets = [t.detach().contiguous().to(dtype) for t in (t0, t1, t2, t3)]
        for t in targets:
            if t.dim() != 3 or t.shape[0] != B or t.shape[2] != 2:
                raise ValueError("part targets must be [B, m, 2]")
        sel = selection if selection.dtype == torch.int32 else selection.to(torch.int32)
        NS = int(sel.numel())
        ctx.dtypes = (verts.dtype, cams.dtype)
        if ctx.f64:
            return CorrChamferFunction._forward_f64(ctx, lib, vv, cc, sel, targets, part_ends, weights, vert_rowptr,
                                                    vert_selection, shared, tuple(verts.shape))
        with torch.cuda.device(vv.device):
            vert2d = torch.empty(B, NS, 2, device=vv.device, dtype=torch.float32)
            nn = torch.empty(B, NS, device=vv.device, dtype=torch.int32)
            loss = torch.empty(B, device=vv.device, dtype=torch.float32)
            tp, tc, pe, wt = CorrChamferFunction._cfg(targets, part_ends, weights)
            rc = lib.umr_corr_chamfer_forward(_ptr(vv), 0 if shared else V * 3, _ptr(cc), _ptr(sel), tp, tc, pe, wt, _ptr(vert2d),
                                              _ptr(nn), _ptr(loss), B, NS, _stream_ptr(vv.device))
        _lib.check(rc, "umr_corr_chamfer_forward")
        ctx.det = torch.are_deterministic_algorithms_enabled()   # the forward has no atomics; the backward's mode
        if ctx.det and (vert_rowptr is None or vert_selection is None):
            vert_rowptr, vert_selection = _incidence_on(sel, V, vv.device)
        ctx.save_for_backward(vv, cc, sel, vert2d, nn, *targets)
        ctx.vert_table = (vert_rowptr, vert_selection) if ctx.det else None   # constants of the loss module
        ctx.cfg = (tuple(int(e) for e in part_ends), tuple(float(w) for w in weights), shared, tuple(verts.shape))
        return loss, vert2d

    @staticmethod
    def backward(ctx, g_loss, g_v2d):
        if ctx.f64:
            return CorrChamferFunction._backward_f64(ctx, g_loss, g_v2d)
        lib = _lib.load()
        vv, cc, sel, vert2d, nn = ctx.saved_tensors[:5]
        targets = list(ctx.saved_tensors[5:])
        part_ends, weights, shared, vshape = ctx.cfg
        B, NS, V = cc.shape[0], vert2d.shape[1], vv.shape[1]
        gl = g_loss.contiguous().float() if g_loss is not None else torch.zeros(B, device=cc.device)
        gv2 = g_v2d.contiguous().float() if g_v2d is not None else None
        with torch.cuda.device(vv.device):
            gverts = torch.empty(B, V, 3, device=vv.device, dtype=torch.float32) if ctx.needs_input_grad[0] else None
            gcams = torch.empty(B, 7, device=vv.device, dtype=torch.float32) if ctx.needs_input_grad[1] else None
            tp, tc, pe, wt = CorrChamferFunction._cfg(targets, part_ends, weights)
            if ctx.det:
                rowptr, vsel = ctx.vert_table
                ws = _workspace(lib.umr_corr_chamfer_workspace_bytes_deterministic(B, NS), vv.device)
                rc = lib.umr_corr_chamfer_backward_deterministic(
                    _ptr(vv), 0 if shared else V * 3, _ptr(cc), _ptr(sel), tp, tc, pe, wt, _ptr(vert2d), _ptr(nn), _ptr(gl),
                    _ptr(gv2), _ptr(gverts), _ptr(gcams), B, NS, V, _ptr(rowptr), _ptr(vsel), _ptr(ws), _stream_ptr(vv.device))
            else:
                rc = lib.umr_corr_chamfer_backward(_ptr(vv), 0 if shared else V * 3, _ptr(cc), _ptr(sel), tp, tc, pe, wt,
                                                   _ptr(vert2d), _ptr(nn), _ptr(gl), _ptr(gv2), _ptr(gverts), _ptr(gcams), B,
                                                   NS, V, _stream_ptr(vv.device))
        _lib.check(rc, "umr_corr_chamfer_backward_deterministic" if ctx.det else "umr_corr_chamfer_backward")
        if gverts is not None and shared and vshape[0] == 1:
            gverts = gverts.sum(0, keepdim=True)   # a [1,V,3] input broadcast here; an expanded [B,V,3] view gets the per-render
        return (gverts, gcams) + (None,) * 9      # gradients and autograd's expand-backward sums them

    @staticmethod
    def _forward_f64(ctx, lib, vv, cc, sel, targets, part_ends, weights, vert_rowptr, vert_selection, shared, vshape):
        B, V, NS = cc.shape[0], vv.shape[1], int(sel.numel())
        with torch.cuda.device(vv.device):
            vert2d = torch.empty(B, NS, 2, device=vv.device, dtype=torch.float64)
            nn = torch.empty(B, NS, device=vv.device, dtype=torch.int32)
            loss = torch.empty(B, device=vv.device, dtype=torch.float64)
            tp, tc, pe, wt = CorrChamferFunction._cfg(targets, part_ends, weights, ctypes.c_double)
            rc = lib.umr_corr_chamfer_forward_f64(_ptr(vv), 0 if shared else V * 3, _ptr(cc), _ptr(sel), tp, tc, pe, wt,
                                                  _ptr(vert2d), _ptr(nn), _ptr(loss), B, NS, _stream_ptr(vv.device))
        _lib.check(rc, "umr_corr_chamfer_forward_f64")
        if vert_rowptr is None or vert_selection is None:   # the backward's per-vertex gather needs the transposed table
            vert_rowptr, vert_selection = _incidence_on(sel, V, vv.device)
        ctx.save_for_backward(vv, cc, sel, vert2d, nn, *targets)
        ctx.vert_table = (vert_rowptr, vert_selection)
        ctx.cfg = (tuple(int(e) for e in part_ends), tuple(float(w) for w in weights), shared, vshape)
        return loss, vert2d

    @staticmethod
    def _backward_f64(ctx, g_loss, g_v2d):
        lib = _lib.load()
        vv, cc, sel, vert2d, nn = ctx.saved_tensors[:5]
        targets = list(ctx.saved_tensors[5:])
        part_ends, weights, shared, vshape = ctx.cfg
        B, NS, V = cc.shape[0], vert2d.shape[1], vv.shape[1]
        gl = g_loss.contiguous().double() if g_loss is not None else torch.zeros(B, device=cc.device, dtype=torch.float64)
        gv2 = g_v2d.contiguous().double() if g_v2d is not None else None
        with torch.cuda.device(vv.device):
            gverts = torch.empty(B, V, 3, device=vv.device, dtype=torch.float64) if ctx.needs_input_grad[0] else None
            gcams = torch.empty(B, 7, device=vv.device, dtype=torch.float64) if ctx.needs_input_grad[1] else None
            tp, tc, pe, wt = CorrChamferFunction._cfg(targets, part_ends, weights, ctypes.c_double)
            rowptr, vsel = ctx.vert_table
            ws = _workspace(lib.umr_corr_chamfer_workspace_bytes_f64(B, NS), vv.device)
            rc = lib.umr_corr_chamfer_backward_f64(_ptr(vv), 0 if shared else V * 3, _ptr(cc), _ptr(sel), tp, tc, pe, wt,
                                                   _ptr(vert2d), _ptr(nn), _ptr(gl), _ptr(gv2), _ptr(gverts), _ptr(gcams), B,
                                                   NS, V, _ptr(rowptr), _ptr(vsel), _ptr(ws), _stream_ptr(vv.device))
        _lib.check(rc, "umr_corr_chamfer_backward_f64")
        if gverts is not None:
            if shared and vshape[0] == 1:
                gverts = gverts.sum(0, keepdim=True)   # as in the float32 backward
            gverts = gverts.to(ctx.dtypes[0])
        return (gverts, gcams.to(ctx.dtypes[1]) if gcams is not None else None) + (None,) * 9


def corr_chamfer(verts, cams, selection, targets, part_ends, weights, vert_table=(None, None)):
    return CorrChamferFunction.apply(verts, cams, selection, *targets, part_ends, weights, *vert_table)


_VOXEL_DTYPES = {torch.float32: 0, torch.float64: 1}  # UMR_DTYPE_FLOAT32 / UMR_DTYPE_FLOAT64
_voxel_status = {}  # device -> the status word of the last voxelize call on that device


def voxelize(faces, size, normalize=False):
    """SoftRas `functional.voxelization` (functional/voxelization.py:41-58): faces [B,F,3,3] float32 or float64 -> int32
    [B,size,size,size], 1 for surface voxels and enclosed empty voxels.  Coordinates are multiplied by `size` first
    unless `normalize` (the reference's `normalize` branch leaves them as they are).  `faces` is not modified; the result
    is on its device.  Contract: DESIGN.md §8."""
    size = int(size)
    if size < 1:
        raise ValueError("voxelize: size must be >= 1, got %d" % size)
    _need_cuda(faces)
    if faces.dtype not in _VOXEL_DTYPES:
        raise TypeError("voxelize: faces must be float32 or float64, got %s" % faces.dtype)
    if faces.dim() != 4 or faces.shape[2:] != (3, 3):
        raise ValueError("voxelize: faces must be [B, F, 3, 3], got %s" % (tuple(faces.shape),))
    lib = _lib.load()
    f = faces.detach().contiguous()
    B, F_ = f.shape[0], f.shape[1]
    dtype, scale = _VOXEL_DTYPES[f.dtype], 1.0 if normalize else float(size)
    nbytes = lib.umr_voxelize_workspace_bytes(B, size)
    if nbytes == 0:  # sizes the library refuses: it checks them before the buffers, so let it say which
        _lib.check(lib.umr_voxelize(_ptr(f), dtype, None, B, F_, size, scale, None, None), "umr_voxelize")
    with torch.cuda.device(f.device):
        out = torch.empty((B, size, size, size), dtype=torch.int32, device=f.device)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=f.device)
        rc = lib.umr_voxelize(_ptr(f), dtype, _ptr(out), B, F_, size, scale, _ptr(ws), _stream_ptr(f.device))
    _lib.check(rc, "umr_voxelize")
    _voxel_status[f.device] = ws[:4].view(torch.int32)
    return out


def voxelize_status(device=None):
    """The status word of the last `voxelize` call on `device` (synchronises): 0, or non-zero when the fill stopped at
    its sweep cap, which only a library bug can cause."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    st = _voxel_status.get(device)
    return 0 if st is None else int(st.item())
