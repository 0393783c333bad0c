"""neural_renderer's `lighting` on the sm_90a kernels (DESIGN.md §15).

lit = textures * light[:, :, None, None, None, :] with the light of DESIGN.md §7 step 2:
n = normalize(cross(v0 - v1, v2 - v1), eps=1e-5), light = Ia*ca + Id*(cd*relu(n.d)), a term whose intensity is 0 not
added.  The forward is one launch (`umr_nmr_lighting_forward`); the backward is one warp per (image, face) that writes
the texture gradient and chains sum(texel * g) through relu, normalize and cross into the face gradient, plus one small
launch that sums the light parameters' per-face partials in ascending face order when a colour or the direction
requires grad (`umr_nmr_lighting_backward`).  Nothing uses atomics, so every result is bitwise reproducible whatever
torch.use_deterministic_algorithms says.

Unlike upstream, which multiplies `textures` in place, this returns a new tensor: in-place multiplication breaks autograd
on leaf textures.
"""
import ctypes
import numbers

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from .. import _lib
from ..raster import _ptr, _stream_ptr

UMR_DTYPE_FLOAT32, UMR_DTYPE_FLOAT64 = 0, 1


def _vector(x, name, B, device):
    """A colour or direction as a tensor of shape [3] or [B,3] on `device`.  Sequences and ndarrays become float32, as
    upstream converts them; tensors keep their dtype (and their autograd graph)."""
    if torch.is_tensor(x):
        t = x.to(device)
    elif isinstance(x, np.ndarray):
        t = torch.from_numpy(np.ascontiguousarray(x)).float().to(device)
    elif isinstance(x, (list, tuple)):
        t = torch.tensor(x, dtype=torch.float32, device=device)
    else:
        raise TypeError("neural_renderer.lighting: %s must be a sequence, an ndarray or a tensor, got %s"
                        % (name, type(x).__name__))
    if not (t.is_floating_point() or t.dtype in (torch.int32, torch.int64)):
        raise ValueError("neural_renderer.lighting: %s must be real, got %s" % (name, t.dtype))
    if tuple(t.shape) not in ((3,), (B, 3)):
        raise ValueError("neural_renderer.lighting: %s must have shape [3] or [%d,3], got %s" % (name, B, tuple(t.shape)))
    return t


def _intensity(x, name):
    if torch.is_tensor(x):
        if x.requires_grad:
            raise NotImplementedError("neural_renderer.lighting: the gradient with respect to %s is not built "
                                      "(pass a number)" % name)
        if x.numel() != 1:
            raise ValueError("neural_renderer.lighting: %s must be a scalar, got shape %s" % (name, tuple(x.shape)))
        return float(x.item())
    if not isinstance(x, numbers.Real):
        raise TypeError("neural_renderer.lighting: %s must be a number, got %s" % (name, type(x).__name__))
    return float(x)


def _params(B, F, T, dtype, Ia, Id, ca, cd, direction):
    p = _lib.UmrNmrLightParams()
    p.batch_size, p.num_faces, p.texture_res = B, F, T
    p.dtype = UMR_DTYPE_FLOAT64 if dtype == torch.float64 else UMR_DTYPE_FLOAT32
    p.intensity_ambient, p.intensity_directional = Ia, Id
    p.color_ambient_bstride, p.color_directional_bstride, p.direction_bstride = (3 if t.dim() == 2 else 0
                                                                                 for t in (ca, cd, direction))
    p.reserved = 0
    return p


class _LightingFunction(torch.autograd.Function):
    """(faces [B,F,3,3], textures [B,F,T,T,T,3], ca, cd, direction [3] or [B,3]) -> lit textures, in `dtype`."""

    @staticmethod
    def forward(ctx, faces, textures, ca, cd, direction, params, dtype):
        lib = _lib.load()
        dev = faces.device
        args = [t.detach().to(dtype).contiguous() for t in (faces, textures, ca, cd, direction)]
        with torch.cuda.device(dev):
            out = torch.empty(textures.shape, device=dev, dtype=dtype)
            rc = lib.umr_nmr_lighting_forward(*[_ptr(t) for t in args], _ptr(out), ctypes.byref(params),
                                              _stream_ptr(dev))
        _lib.check(rc, "umr_nmr_lighting_forward")
        ctx.params, ctx.dtype = params, dtype
        ctx.in_dtypes = [t.dtype for t in (faces, textures, ca, cd, direction)]
        ctx.save_for_backward(*args)
        return out

    @staticmethod
    @once_differentiable   # the kernels' gradients are not themselves differentiable: double backward raises
    def backward(ctx, grad_out):
        lib = _lib.load()
        faces, textures, ca, cd, direction = ctx.saved_tensors
        p, dtype = ctx.params, ctx.dtype
        dev = faces.device
        B, F = p.batch_size, p.num_faces
        need = ctx.needs_input_grad
        g = grad_out.to(dtype).contiguous()
        grad_faces = grad_tex = grad_light = ws = None
        with torch.cuda.device(dev):
            if need[0]:
                grad_faces = torch.empty(faces.shape, device=dev, dtype=dtype)
            if need[1]:
                grad_tex = torch.empty(textures.shape, device=dev, dtype=dtype)
            if need[2] or need[3] or need[4]:
                grad_light = torch.empty(B, 9, device=dev, dtype=dtype)
                ws = torch.empty(lib.umr_nmr_lighting_workspace_bytes(B, F, p.dtype), device=dev, dtype=torch.uint8)
            if grad_faces is None and grad_tex is None and grad_light is None:
                return (None,) * 7
            rc = lib.umr_nmr_lighting_backward(_ptr(faces), _ptr(textures), _ptr(ca), _ptr(cd), _ptr(direction), _ptr(g),
                                               _ptr(grad_faces), _ptr(grad_tex), _ptr(grad_light), ctypes.byref(p),
                                               _ptr(ws), _stream_ptr(dev))
        _lib.check(rc, "umr_nmr_lighting_backward")
        grads = [grad_faces, grad_tex, None, None, None]
        for i, t in enumerate((ca, cd, direction)):
            if need[2 + i]:
                gi = grad_light[:, 3 * i:3 * i + 3]
                grads[2 + i] = gi if t.dim() == 2 else gi.sum(0)   # a [3] vector lights every image
        grads = [None if gr is None else gr.to(dt) for gr, dt in zip(grads, ctx.in_dtypes)]
        return (*grads, None, None)


def _prepare(faces, textures, intensity_ambient, intensity_directional, color_ambient, color_directional, direction):
    """Validated arguments -> (colour / direction tensors, UmrNmrLightParams, compute dtype), on faces' device."""
    if not torch.is_tensor(faces) or faces.dim() != 4 or tuple(faces.shape[2:]) != (3, 3) or faces.shape[0] < 1 \
            or faces.shape[1] < 1:
        raise ValueError("neural_renderer.lighting: faces [B,F,3,3] expected, got %s"
                         % (tuple(faces.shape) if torch.is_tensor(faces) else type(faces).__name__,))
    B, F = faces.shape[:2]
    if not torch.is_tensor(textures) or textures.dim() != 6 or tuple(textures.shape[:2]) != (B, F) \
            or textures.shape[3] != textures.shape[2] or textures.shape[4] != textures.shape[2] \
            or textures.shape[5] != 3 or textures.shape[2] < 1:
        raise ValueError("neural_renderer.lighting: textures [B,F,T,T,T,3] with B = %d, F = %d expected, got %s"
                         % (B, F, tuple(textures.shape) if torch.is_tensor(textures) else type(textures).__name__))
    for name, t in (("faces", faces), ("textures", textures)):
        if not t.is_floating_point():
            raise ValueError("neural_renderer.lighting: %s must be floating point, got %s" % (name, t.dtype))
    Ia = _intensity(intensity_ambient, "intensity_ambient")
    Id = _intensity(intensity_directional, "intensity_directional")
    dev = faces.device
    ca = _vector(color_ambient, "color_ambient", B, dev)
    cd = _vector(color_directional, "color_directional", B, dev)
    d = _vector(direction, "direction", B, dev)
    dtype = torch.float64 if any(t.dtype == torch.float64 for t in (faces, textures, ca, cd, d)) else torch.float32
    T = textures.shape[2]
    if B * F * 3 * T ** 3 >= 2 ** 31 or B * F * 9 >= 2 ** 31:
        raise ValueError("neural_renderer.lighting: B*F*3*T^3 = %d elements do not fit int32 indexing"
                         % (B * F * 3 * T ** 3))
    return ca, cd, d, _params(B, F, T, dtype, Ia, Id, ca, cd, d), dtype


def lighting(faces, textures, intensity_ambient=0.5, intensity_directional=0.5, color_ambient=(1, 1, 1),
             color_directional=(1, 1, 1), direction=(0, 1, 0)):
    """faces [B,F,3,3], textures [B,F,T,T,T,3] -> lit textures [B,F,T,T,T,3] (a new tensor).  Colours and the direction
    are sequences, ndarrays or tensors of shape [3] or [B,3]; the intensities are numbers.  Computes in float64 when any
    tensor argument is float64, else in float32 (half inputs included); the result has that dtype, and each gradient
    comes back in its input's dtype."""
    ca, cd, d, params, dtype = _prepare(faces, textures, intensity_ambient, intensity_directional, color_ambient,
                                        color_directional, direction)
    if not faces.is_cuda or not textures.is_cuda or textures.device != faces.device:
        raise TypeError("neural_renderer.lighting supports only cuda tensors (faces and textures on one device)")
    return _LightingFunction.apply(faces, textures, ca, cd, d, params, dtype)
