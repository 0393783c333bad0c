"""torch.autograd bindings of the geometric-loss kernels (C ABI: include/umr_b200.h).

CUDA only: there is no CPU fallback (the CPU oracles live in oracle/ and are test infrastructure).

Each Function reads its kernel family once in `forward` into a `raster.KernelMode` kept in `ctx`, so a backward runs in
the mode of its forward.  Under torch.use_deterministic_algorithms(True) the Functions whose default kernels sum with
float atomics call the `*_deterministic` symbols instead (bitwise reproducible, DESIGN.md §2).

Dtype rule of the loss Functions (DESIGN.md §10): an op computes in float64, with the `*_f64` symbols, when any of its
floating-point tensor inputs is float64.  It then returns float64 values and each input's gradient in that input's dtype.
The float64 kernels are always bitwise reproducible, so the deterministic flag does not change them.  Every other dtype
(float32, half) computes in float32 as before.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .raster import KernelMode, _ptr, _stream_ptr


def _need_cuda(*ts):
    for t in ts:
        if not t.is_cuda:
            raise TypeError("umr_b200 ops support only cuda Tensors")


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


def _as(t, mode):
    """Detached, contiguous, in the compute dtype of `mode`."""
    return t.detach().contiguous().to(mode.dtype)


def _pairs(t):
    """`t` itself when its address is a multiple of 2 * itemsize, else an aligned copy: the kernels read the sampler's
    flow and TexCycle's flow / prob as (x, y) vector pairs, which a contiguous view at an odd element offset (e.g.
    `buf[1:].view(B, N, 2)`) would misalign.  The library refuses such a pointer."""
    return t if t.data_ptr() % (2 * t.element_size()) == 0 else t.clone()


# -------------------------------------------------------------------------------------------------
# bilinear texture-flow sampler
# -------------------------------------------------------------------------------------------------
SAMPLE_MAX_CHANNELS = 4   # channels one sampler kernel call takes; wider images are sampled in groups of this many


def _channel_groups(C):
    """[(first channel, count)] of the sampler calls for C channels: one call for C <= 4, else groups of at most 4."""
    return [(c, min(SAMPLE_MAX_CHANNELS, C - c)) for c in range(0, C, SAMPLE_MAX_CHANNELS)]


class BilinearSampleFunction(torch.autograd.Function):
    """images [B,C,H,W], flow [B,N,2] -> out [B,N,C]; bilinear, zeros padding, align_corners=True
    (the torch-1.1 semantics the reference was written for: geom_utils.py:55, loss_utils.py:64).

    The kernels take at most 4 channels.  A wider image (SCOPS's 5 part probabilities in avg_uv.py, K keypoint heat maps)
    runs them on channel groups of at most 4: the forward concatenates the groups' outputs, each group gets its own image
    gradient, and the flow gradient is the groups' flow gradients summed in ascending group order."""

    @staticmethod
    def forward(ctx, images, flow):
        _need_cuda(images, flow)
        m = KernelMode(_is_f64(images, flow))   # the forward has no atomics; the backward's mode
        img, fl = _as(images, m), _pairs(_as(flow, m))
        B, C, H, W = img.shape
        N = fl.shape[1]
        groups = _channel_groups(C)
        with torch.cuda.device(img.device):
            outs = []
            for c0, c in groups:
                part = img if len(groups) == 1 else img[:, c0:c0 + c].contiguous()
                out = torch.empty(B, N, c, device=img.device, dtype=m.dtype)
                m.call("umr_bilinear_sample_forward", False, _ptr(part), _ptr(fl), _ptr(out), B, c, H, W, N,
                       _stream_ptr(img.device))
                outs.append(out)
        ctx.save_for_backward(img, fl)
        ctx.img_grad = images.requires_grad
        ctx.mode = m
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=2)

    @staticmethod
    def backward(ctx, grad_out):
        m = ctx.mode
        img, fl = ctx.saved_tensors
        B, C, H, W = img.shape
        N = fl.shape[1]
        g = grad_out.contiguous().to(m.dtype)
        groups = _channel_groups(C)
        with torch.cuda.device(img.device):
            tables = ()
            if m.gather:   # the image gradient gathers over samples keyed by their top-left cell: the cell -> samples table
                rowptr = samples = None
                if ctx.img_grad:
                    cells = torch.empty(B, N, device=img.device, dtype=torch.int32)
                    m.call("umr_bilinear_sample_cells", False, _ptr(fl), _ptr(cells), B, H, W, N, _stream_ptr(img.device))
                    rowptr, samples = device_incidence(cells, B * (H + 1) * (W + 1))
                tables = (_ptr(rowptr), _ptr(samples))
            gflow, gimgs = None, []
            for c0, c in groups:
                part, gpart = (img, g) if len(groups) == 1 else (img[:, c0:c0 + c].contiguous(), g[:, :, c0:c0 + c].contiguous())
                gf = torch.empty_like(fl)
                gi = torch.empty_like(part) if ctx.img_grad else None
                m.call("umr_bilinear_sample_backward", True, _ptr(part), _ptr(fl), _ptr(gpart), _ptr(gf), _ptr(gi),
                       B, c, H, W, N, *tables, _stream_ptr(img.device))
                gflow = gf if gflow is None else gflow.add_(gf)
                if gi is not None:
                    gimgs.append(gi)
            gimg = (gimgs[0] if len(gimgs) == 1 else torch.cat(gimgs, dim=1)) if gimgs else None
        return gimg, gflow


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
        B = predict.shape[0]
        if target.shape[0] != B or target.numel() != predict.numel():
            raise ValueError("neg_iou_loss: predict %s and target %s must hold the same number of elements per image"
                             % (tuple(predict.shape), tuple(target.shape)))
        m = KernelMode(_is_f64(predict, target))
        t = _as(target, m).view(B, -1)
        N = t.shape[1]
        p, pbs = _batch_view(predict.detach(), N, m.dtype)  # e.g. the alpha plane of the RGBA render, read in place
        with torch.cuda.device(p.device):
            inter = torch.empty(B, device=p.device, dtype=m.dtype)
            uni = torch.empty_like(inter)
            loss = torch.empty_like(inter)
            ws = m.workspace("umr_iou_workspace_bytes", p.device, B, N)
            m.call("umr_iou_forward", True, _ptr(p), pbs, _ptr(t), _ptr(inter), _ptr(uni), _ptr(loss), B, N,
                   *((_ptr(ws),) if m.gather else ()), _stream_ptr(p.device))
        ctx.save_for_backward(t, inter, uni)
        ctx.shape = tuple(predict.shape)
        ctx.mode = m
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        t, inter, uni = ctx.saved_tensors
        B, N = t.shape
        g = grad_loss.contiguous().to(ctx.mode.dtype)
        with torch.cuda.device(t.device):
            gp = torch.empty_like(t)
            ctx.mode.call("umr_iou_backward", False, _ptr(t), _ptr(inter), _ptr(uni), _ptr(g), _ptr(gp), B, N,
                          _stream_ptr(t.device))
        return gp.view(ctx.shape), None


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
        B, C, H, W = img_pred.shape
        HW = H * W
        if tuple(img_gt.shape) != (B, C, H, W) or mask_gt.numel() != B * HW or mask_pred.numel() != B * HW:
            raise ValueError("texture_loss_masks: img_pred %s, img_gt %s, mask_gt %s, mask_pred %s do not match"
                             % (tuple(img_pred.shape), tuple(img_gt.shape), tuple(mask_gt.shape), tuple(mask_pred.shape)))
        m = KernelMode(_is_f64(img_pred, img_gt, mask_gt, mask_pred))
        p, pbs = _batch_view(img_pred.detach(), C * HW, m.dtype)
        mp, mbs = _batch_view(mask_pred.detach(), HW, m.dtype)
        g, mg = _as(img_gt, m), _as(mask_gt, m)
        with torch.cuda.device(p.device):
            loss = torch.empty(B, device=p.device, dtype=m.dtype)
            ws = m.workspace("umr_masked_l1_workspace_bytes", p.device, B, HW)
            m.call("umr_masked_l1_forward", True, _ptr(p), pbs, _ptr(mp), mbs, _ptr(g), _ptr(mg), _ptr(loss), B, C, HW,
                   *((_ptr(ws),) if m.gather else ()), _stream_ptr(p.device))
        ctx.save_for_backward(p, mp, g, mg)
        ctx.meta = (pbs, mbs, img_pred.requires_grad, mask_pred.requires_grad, tuple(img_pred.shape),
                    tuple(mask_pred.shape))
        ctx.mode = m
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        m = ctx.mode
        p, mp, g, mg = ctx.saved_tensors
        pbs, mbs, need_p, need_m, pshape, mshape = ctx.meta
        B, C = pshape[0], pshape[1]
        HW = pshape[2] * pshape[3]
        gl = grad_loss.contiguous().to(m.dtype)
        with torch.cuda.device(p.device):
            gp = torch.empty(pshape, device=p.device, dtype=m.dtype) if need_p else None
            gm = torch.empty(mshape, device=p.device, dtype=m.dtype) if need_m else None
            m.call("umr_masked_l1_backward", False, _ptr(p), pbs, _ptr(mp), mbs, _ptr(g), _ptr(mg), _ptr(gl), _ptr(gp),
                   _ptr(gm), B, C, HW, _stream_ptr(p.device))
        return gp, None, None, gm


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
        B, C, H, W = images.shape
        if C != 4 or tuple(img_gt.shape) != (B, 3, H, W) or mask_gt.numel() != B * H * W:
            raise ValueError("mask_texture_loss: images %s must be [B,4,H,W], img_gt %s [B,3,H,W], mask_gt %s [B,H,W]"
                             % (tuple(images.shape), tuple(img_gt.shape), tuple(mask_gt.shape)))
        m = KernelMode(_is_f64(images, img_gt, mask_gt))
        x, g, mk = _as(images, m), _as(img_gt, m), _as(mask_gt, m)
        with torch.cuda.device(x.device):
            stats = torch.empty(B, 3, device=x.device, dtype=m.dtype)
            per_image = torch.empty(B, 2, device=x.device, dtype=m.dtype)
            loss = torch.empty((), device=x.device, dtype=m.dtype)
            ws = m.workspace("umr_loss_head_workspace_bytes", x.device, B, H * W)
            m.call("umr_loss_head_forward", True, _ptr(x), _ptr(g), _ptr(mk), _ptr(stats), _ptr(per_image), _ptr(loss),
                   B, H * W, float(w_iou), float(w_tex), *((_ptr(ws),) if m.gather else ()), _stream_ptr(x.device))
        ctx.save_for_backward(x, g, mk, stats)
        ctx.w = (float(w_iou), float(w_tex))
        ctx.mode = m
        ctx.mark_non_differentiable(per_image)
        return loss, per_image

    @staticmethod
    def backward(ctx, grad_loss, _gp=None):
        x, g, mk, stats = ctx.saved_tensors
        B, _, H, W = x.shape
        gl = grad_loss.contiguous().to(ctx.mode.dtype).reshape(1)
        with torch.cuda.device(x.device):
            gx = torch.empty_like(x)
            ctx.mode.call("umr_loss_head_backward", False, _ptr(x), _ptr(g), _ptr(mk), _ptr(stats), _ptr(gl), _ptr(gx),
                          B, H * W, ctx.w[0], ctx.w[1], _stream_ptr(x.device))
        return gx, None, None, None, None


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
        m = KernelMode(_is_f64(a, b))   # the forward has no atomics; the backward's mode
        x, y = _as(a, m), _as(b, m)
        B, N, D = x.shape
        M = y.shape[1]
        with torch.cuda.device(x.device):
            d_ab = torch.empty(B, N, device=x.device, dtype=m.dtype)
            d_ba = torch.empty(B, M, device=x.device, dtype=m.dtype)
            i_ab = torch.empty(B, N, device=x.device, dtype=torch.int32)
            i_ba = torch.empty(B, M, device=x.device, dtype=torch.int32)
            m.call("umr_chamfer_forward", False, _ptr(x), _ptr(y), _ptr(d_ab), _ptr(d_ba), _ptr(i_ab), _ptr(i_ba),
                   B, N, M, D, _stream_ptr(x.device))
        ctx.save_for_backward(x, y, i_ab, i_ba)
        ctx.mark_non_differentiable(i_ab, i_ba)
        ctx.mode = m
        return d_ab, d_ba, i_ab, i_ba

    @staticmethod
    def backward(ctx, g_ab, g_ba, _1=None, _2=None):
        m = ctx.mode
        x, y, i_ab, i_ba = ctx.saved_tensors
        B, N, D = x.shape
        M = y.shape[1]
        g1 = g_ab.contiguous().to(m.dtype) if g_ab is not None else None
        g2 = g_ba.contiguous().to(m.dtype) if g_ba is not None else None
        with torch.cuda.device(x.device):
            gx = torch.empty_like(x)
            gy = torch.empty_like(y)
            m.call("umr_chamfer_backward", True, _ptr(x), _ptr(y), _ptr(i_ab), _ptr(i_ba), _ptr(g1), _ptr(g2), _ptr(gx),
                   _ptr(gy), B, N, M, D, _stream_ptr(x.device))
        return gx, gy


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
        m = KernelMode(_is_f64(flow, prob, face_ids))
        fl, pr = _pairs(_as(flow, m)), _pairs(_as(prob, m))
        B, F, T2 = fl.shape[0], fl.shape[1], fl.shape[2]
        if visible is not None:
            if visible.dtype != torch.uint8 or tuple(visible.shape) != (B, F) or not visible.is_cuda:
                raise ValueError("visible must be a CUDA uint8 tensor of shape [B,F]")
            ids, P = None, 0
        else:
            # the visibility bitmap reads a float32 plane in both precisions: face ids (and the background's -1) are
            # integers below UMR_RASTER_MAX_FACES = 2^24, which float32 holds exactly, so a float64 plane converts
            # without rounding
            ids = face_ids.detach().contiguous().float()
            P = ids.shape[1]
        with torch.cuda.device(fl.device):
            vis = visible.contiguous() if visible is not None else torch.empty(B, F, device=fl.device, dtype=torch.uint8)
            loss = torch.empty(1, device=fl.device, dtype=m.dtype)
            ws = m.workspace("umr_texcycle_workspace_bytes", fl.device, B, F)
            m.call("umr_texcycle_forward", True, _ptr(fl), _ptr(pr), _ptr(ids), _ptr(vis), _ptr(loss), B, F, T2, P,
                   *((_ptr(ws),) if m.gather else ()), _stream_ptr(fl.device))
        ctx.save_for_backward(fl, pr, vis)
        ctx.mode = m
        return loss.view(())

    @staticmethod
    def backward(ctx, grad_loss):
        fl, pr, vis = ctx.saved_tensors
        B, F, T2 = fl.shape[0], fl.shape[1], fl.shape[2]
        g = grad_loss.contiguous().to(ctx.mode.dtype).view(1)
        with torch.cuda.device(fl.device):
            gflow = torch.empty_like(fl)
            ctx.mode.call("umr_texcycle_backward", False, _ptr(fl), _ptr(pr), _ptr(vis), _ptr(g), _ptr(gflow), B, F, T2,
                          _stream_ptr(fl.device))
        return gflow, None, None, None


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
        m = KernelMode(_is_f64(x, coef, tcoef))
        xx = _as(x, m)
        B, V = xx.shape[:2]
        if m.f64:
            coef, tcoef = _as(coef, m), _as(tcoef, m)   # the module's float32 -1/deg entries widen exactly
        with torch.cuda.device(xx.device):
            y = torch.empty_like(xx)
            loss = torch.empty(B, device=xx.device, dtype=m.dtype)
            ws = m.workspace("umr_laplacian_workspace_bytes", xx.device, B, V)
            m.call("umr_laplacian_forward", True, _ptr(xx), _ptr(rowptr), _ptr(col), _ptr(coef), _ptr(y), _ptr(loss),
                   B, V, *((_ptr(ws),) if m.gather else ()), _stream_ptr(xx.device))
        ctx.save_for_backward(y, rowptr, col, tcoef)
        ctx.mode = m
        return loss

    @staticmethod
    def backward(ctx, g):
        y, rowptr, col, tcoef = ctx.saved_tensors
        B, V = y.shape[:2]
        gl = g.contiguous().to(ctx.mode.dtype)
        with torch.cuda.device(y.device):
            gx = torch.empty_like(y)
            ctx.mode.call("umr_laplacian_backward", False, _ptr(y), _ptr(rowptr), _ptr(col), _ptr(tcoef), _ptr(gl),
                          _ptr(gx), B, V, _stream_ptr(y.device))
        return gx, None, None, None, None


class FlattenFunction(torch.autograd.Function):
    """vertices [B,V,3] + edge table [E,4] int32 -> per-sample sum_e (cos + 1)^2 [B] (SoftRas/losses.py:71-114).
    `vert_rowptr` / `vert_incidence`: the edge table's transposed incidence (`vertex_incidence(edges, V)` on the device),
    used by the deterministic and float64 backwards; FlattenLoss builds it once.  Without it such a call builds it here
    (a device-to-host copy of the edge table)."""

    @staticmethod
    def forward(ctx, vertices, edges, eps, vert_rowptr=None, vert_incidence=None):
        _need_cuda(vertices)
        m = KernelMode(_is_f64(vertices))
        v = _as(vertices, m)
        B, V = v.shape[:2]
        E = edges.shape[0]
        with torch.cuda.device(v.device):
            loss = torch.empty(B, device=v.device, dtype=m.dtype)
            ws = m.workspace("umr_flatten_forward_workspace_bytes", v.device, B, E)
            m.call("umr_flatten_forward", True, _ptr(v), _ptr(edges), _ptr(loss), B, V, E, float(eps),
                   *((_ptr(ws),) if m.gather else ()), _stream_ptr(v.device))
        if m.gather:   # the deterministic and float64 backwards are per-vertex gathers over the transposed table
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
        ctx.mode = m
        return loss

    @staticmethod
    def backward(ctx, g):
        m = ctx.mode
        v, edges = ctx.saved_tensors[:2]
        B, V = v.shape[:2]
        E = edges.shape[0]
        gl = g.contiguous().to(m.dtype)
        with torch.cuda.device(v.device):
            gv = torch.empty_like(v)
            if m.gather:
                rowptr, inc = ctx.saved_tensors[2:]
                ws = m.workspace("umr_flatten_backward_workspace_bytes", v.device, B, E)
                m.call("umr_flatten_backward", True, _ptr(v), _ptr(edges), _ptr(rowptr), _ptr(inc), _ptr(gl), _ptr(gv),
                       B, V, E, ctx.eps, _ptr(ws), _stream_ptr(v.device))
            else:
                m.call("umr_flatten_backward", True, _ptr(v), _ptr(edges), _ptr(gl), _ptr(gv), B, V, E, ctx.eps,
                       _stream_ptr(v.device))
        return gv, None, None, None, None


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
    deterministic and float64 backwards; CorrLossChamfer caches it.  Without it such a call builds it here (a
    device-to-host copy of the selection)."""

    @staticmethod
    def _cfg(targets, part_ends, weights, mode):
        tp = (ctypes.c_void_p * 4)(*[t.data_ptr() for t in targets])
        tc = (ctypes.c_int32 * 4)(*[int(t.shape[1]) for t in targets])
        pe = (ctypes.c_int32 * 4)(*[int(e) for e in part_ends])
        wt = ((ctypes.c_double if mode.f64 else ctypes.c_float) * 4)(*[float(w) for w in weights])
        return tp, tc, pe, wt

    @staticmethod
    def forward(ctx, verts, cams, selection, t0, t1, t2, t3, part_ends, weights, vert_rowptr=None, vert_selection=None):
        _need_cuda(verts, cams, selection, t0, t1, t2, t3)
        m = KernelMode(_is_f64(verts, cams, t0, t1, t2, t3))   # the forward has no atomics; the backward's mode
        B = cams.shape[0]
        shared = verts.shape[0] == 1 or (verts.dim() == 3 and verts.stride(0) == 0)   # one mesh for every render
        vv = _as(verts[:1] if shared else verts, m)
        if not shared and vv.shape[0] != B:
            raise ValueError("verts batch %d does not match cams batch %d" % (vv.shape[0], B))
        V = vv.shape[1]
        cc = _as(cams, m)
        targets = [_as(t, m) for t in (t0, t1, t2, t3)]
        for t in targets:
            if t.dim() != 3 or t.shape[0] != B or t.shape[2] != 2:
                raise ValueError("part targets must be [B, m, 2]")
        sel = selection if selection.dtype == torch.int32 else selection.to(torch.int32)
        NS = int(sel.numel())
        with torch.cuda.device(vv.device):
            vert2d = torch.empty(B, NS, 2, device=vv.device, dtype=m.dtype)
            nn = torch.empty(B, NS, device=vv.device, dtype=torch.int32)
            loss = torch.empty(B, device=vv.device, dtype=m.dtype)
            tp, tc, pe, wt = CorrChamferFunction._cfg(targets, part_ends, weights, m)
            m.call("umr_corr_chamfer_forward", False, _ptr(vv), 0 if shared else V * 3, _ptr(cc), _ptr(sel), tp, tc, pe,
                   wt, _ptr(vert2d), _ptr(nn), _ptr(loss), B, NS, _stream_ptr(vv.device))
        if m.gather and (vert_rowptr is None or vert_selection is None):   # the backward's per-vertex gather
            vert_rowptr, vert_selection = _incidence_on(sel, V, vv.device)
        ctx.save_for_backward(vv, cc, sel, vert2d, nn, *targets)
        ctx.vert_table = (vert_rowptr, vert_selection) if m.gather else None   # constants of the loss module
        ctx.cfg = (tuple(int(e) for e in part_ends), tuple(float(w) for w in weights), shared, tuple(verts.shape))
        ctx.mode = m
        return loss, vert2d

    @staticmethod
    def backward(ctx, g_loss, g_v2d):
        m = ctx.mode
        vv, cc, sel, vert2d, nn = ctx.saved_tensors[:5]
        targets = list(ctx.saved_tensors[5:])
        part_ends, weights, shared, vshape = ctx.cfg
        B, NS, V = cc.shape[0], vert2d.shape[1], vv.shape[1]
        gl = g_loss.contiguous().to(m.dtype) if g_loss is not None else torch.zeros(B, device=cc.device, dtype=m.dtype)
        gv2 = g_v2d.contiguous().to(m.dtype) if g_v2d is not None else None
        with torch.cuda.device(vv.device):
            gverts = torch.empty(B, V, 3, device=vv.device, dtype=m.dtype) if ctx.needs_input_grad[0] else None
            gcams = torch.empty(B, 7, device=vv.device, dtype=m.dtype) if ctx.needs_input_grad[1] else None
            tp, tc, pe, wt = CorrChamferFunction._cfg(targets, part_ends, weights, m)
            gather = ()
            if m.gather:
                rowptr, vsel = ctx.vert_table
                ws = m.workspace("umr_corr_chamfer_workspace_bytes", vv.device, B, NS)
                gather = (_ptr(rowptr), _ptr(vsel), _ptr(ws))
            m.call("umr_corr_chamfer_backward", True, _ptr(vv), 0 if shared else V * 3, _ptr(cc), _ptr(sel), tp, tc, pe,
                   wt, _ptr(vert2d), _ptr(nn), _ptr(gl), _ptr(gv2), _ptr(gverts), _ptr(gcams), B, NS, V, *gather,
                   _stream_ptr(vv.device))
        if gverts is not None and shared and vshape[0] == 1:
            gverts = gverts.sum(0, keepdim=True)   # a [1,V,3] input broadcast here; an expanded [B,V,3] view gets the per-render
        return (gverts, gcams) + (None,) * 9      # gradients and autograd's expand-backward sums them


def corr_chamfer(verts, cams, selection, targets, part_ends, weights, vert_table=(None, None)):
    return CorrChamferFunction.apply(verts, cams, selection, *targets, part_ends, weights, *vert_table)


_DTYPE_IDS = {torch.float32: 0, torch.float64: 1}  # UMR_DTYPE_FLOAT32 / UMR_DTYPE_FLOAT64


# -------------------------------------------------------------------------------------------------
# part_matching_loss head (nnutils/loss_utils.py part_matching_loss after its render)
# -------------------------------------------------------------------------------------------------
def _planes(t, inner, dtype):
    """(tensor, batch stride) of `t` [B, ...] read in place when each image is dense, in `dtype` and aligned to its element
    size (the library refuses a misaligned pointer), else a contiguous copy."""
    v, bs = _batch_view(t.detach(), inner, dtype)
    if v.data_ptr() % v.element_size():
        v, bs = v.contiguous().clone(), inner
    return v, bs


class PartMatchingHeadFunction(torch.autograd.Function):
    """The head of part_matching_loss (DESIGN.md §13).  Part maps P_1..P_4 (each [B,H,H] dense per image: [B,1,H,H]
    tensors or channels of a render, read in place), c0 [B,H,H] (channel 0 of proj), part_segs [B,5,H,H], weights (5
    values), kld -> per-image terms [B,2]: (sum of the 8 squared centroid differences, the weighted squared-difference sum
    of the max-normalised maps, or for kld the KL sum).  Gradients reach the four maps; c0, part_segs and weights are
    data.  Forward: 4 launches (mse) or 2 (kld); backward: 1."""

    @staticmethod
    def forward(ctx, p1, p2, p3, p4, c0, part_segs, weights, kld):
        maps = (p1, p2, p3, p4)
        _need_cuda(*maps, c0, part_segs, weights)
        B, C, H, W = part_segs.shape
        if C != 5 or H != W:
            raise ValueError("part_matching_head: part_segs must be [B,5,H,H], got %s" % (tuple(part_segs.shape),))
        for t in maps + (c0,):
            if t.shape[0] != B or t[0].numel() != H * W:
                raise ValueError("part_matching_head: part maps and c0 must hold [B,%d,%d] values, got %s"
                                 % (H, W, tuple(t.shape)))
        if weights.numel() != 5:
            raise ValueError("part_matching_head: 5 weights expected, got %d" % weights.numel())
        m = KernelMode(_is_f64(*maps, c0, part_segs, weights))
        planes = [_planes(t, H * W, m.dtype) for t in maps]
        cz, cbs = _planes(c0, H * W, m.dtype)
        q, qbs = _planes(part_segs, 5 * H * W, m.dtype)
        w = _as(weights.reshape(-1), m)
        kld = 1 if kld else 0
        with torch.cuda.device(q.device):
            terms = torch.empty(B, 2, device=q.device, dtype=m.dtype)
            lib, dt = _lib.load(), _DTYPE_IDS[m.dtype]
            ws = torch.empty(lib.umr_part_head_workspace_bytes(B, H, dt), device=q.device, dtype=torch.uint8)
            mp = (ctypes.c_void_p * 4)(*[v.data_ptr() for v, _ in planes])
            mb = (ctypes.c_int64 * 4)(*[bs for _, bs in planes])
            _lib.check(lib.umr_part_head_forward(mp, mb, _ptr(cz), cbs, _ptr(q), qbs, _ptr(w), _ptr(terms), B, H, kld, dt,
                                                 _ptr(ws), _stream_ptr(q.device)), "umr_part_head_forward")
        ctx.inputs = (planes, cz, cbs, q, qbs, w, ws, kld, [(t.shape, t.dtype) for t in maps])
        ctx.mode = m
        return terms

    @staticmethod
    def backward(ctx, grad_terms):
        m = ctx.mode
        planes, cz, cbs, q, qbs, w, ws, kld, metas = ctx.inputs
        B, _, H, W = q.shape
        g = grad_terms.contiguous().to(m.dtype)
        with torch.cuda.device(q.device):
            gm = torch.empty(B, 4, H, W, device=q.device, dtype=m.dtype)
            mp = (ctypes.c_void_p * 4)(*[v.data_ptr() for v, _ in planes])
            mb = (ctypes.c_int64 * 4)(*[bs for _, bs in planes])
            _lib.check(_lib.load().umr_part_head_backward(mp, mb, _ptr(cz), cbs, _ptr(q), qbs, _ptr(w), _ptr(ws), _ptr(g),
                                                          _ptr(gm), B, H, kld, _DTYPE_IDS[m.dtype], _stream_ptr(q.device)),
                       "umr_part_head_backward")
        grads = tuple(gm[:, k].reshape(shape).to(dtype) if ctx.needs_input_grad[k] else None
                      for k, (shape, dtype) in enumerate(metas))
        return grads + (None,) * 4


def part_matching_head(maps, c0, part_segs, weights, kld):
    """-> terms [B,2] of the part_matching_loss head; see PartMatchingHeadFunction."""
    return PartMatchingHeadFunction.apply(*maps, c0, part_segs, weights, bool(kld))


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
    if faces.dtype not in _DTYPE_IDS:
        raise TypeError("voxelize: faces must be float32 or float64, got %s" % faces.dtype)
    if faces.dim() != 4 or faces.shape[2:] != (3, 3):
        raise ValueError("voxelize: faces must be [B, F, 3, 3], got %s" % (tuple(faces.shape),))
    lib = _lib.load()
    f = faces.detach().contiguous()
    B, F_ = f.shape[0], f.shape[1]
    dtype, scale = _DTYPE_IDS[f.dtype], 1.0 if normalize else float(size)
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
