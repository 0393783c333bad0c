"""neural_renderer's functional rasterisers: `rasterize_rgbad`, `rasterize`, `rasterize_silhouettes`, `rasterize_depth`.

Face coordinates [B,F,3,3] are already in NDC: the caller applies its camera, and bakes lighting into the textures,
as upstream's `Renderer` does before it calls these.  There is no fill-back, light or camera inside.  The forward is
`umr_nmr_forward` (DESIGN.md §7) with one copy per face, eye_z = 0 and light exactly 1; the faces are handed to it as
a [B,3F,3] vertex array with an index table.  Gradients flow to `faces`, from every requested output, through NMR's
approximate edge gradient and the analytic depth gradient (umr_nmr_backward_faces, DESIGN.md §14), and to `textures`
through the exact texture gradient of `Renderer`.  Both are bitwise reproducible: the geometry gradient has no atomics,
and the texture gradient takes its deterministic gather under torch.use_deterministic_algorithms(True).
"""
import ctypes

import torch

from .. import _lib
from ..raster import _ptr, _stream_ptr

DEFAULT_IMAGE_SIZE = 256
DEFAULT_ANTI_ALIASING = True
DEFAULT_NEAR = 0.1
DEFAULT_FAR = 100
DEFAULT_EPS = 1e-4
DEFAULT_BACKGROUND_COLOR = (0, 0, 0)

_MAX_FACES = (2 ** 31 - 1) // 3   # the vertex array [B,3F,3] is indexed with int32


def _params(B, F, T, image_size, anti_aliasing, near, far, background_color):
    p = _lib.UmrNmrParams()
    p.batch_size, p.num_vertices, p.num_faces, p.texture_res = B, 3 * F, F, T
    p.image_size, p.anti_aliasing, p.fill_back, p.shared_textures = image_size, int(bool(anti_aliasing)), 0, 1
    p.eye_z = 0.0                                   # look_at is then the identity on z
    p.near_plane, p.far_plane = float(near), float(far)
    p.light_intensity_ambient, p.light_intensity_directional = 1.0, 0.0   # light = 0 + 1 * 1: exactly 1
    p.light_color_ambient[:] = [1.0, 1.0, 1.0]
    p.light_color_directional[:] = [1.0, 1.0, 1.0]
    p.light_direction[:] = [0.0, 1.0, 0.0]
    p.background_color[:] = background_color
    return p


class _RasterizeFunction(torch.autograd.Function):
    """(faces [B,F,3,3], textures [B,F,T,T,T,3] | None) -> (rgb | None, alpha | None, depth | None)."""

    @staticmethod
    def forward(ctx, faces, textures, params, eps, want_rgb, want_alpha, want_depth):
        lib = _lib.load()
        dev = faces.device
        B, F, IS = params.batch_size, params.num_faces, params.image_size
        S = IS * (2 if params.anti_aliasing else 1)
        verts = faces.detach().contiguous().float().reshape(B, 3 * F, 3)
        tex = None if textures is None else textures.detach().contiguous().float()
        with torch.cuda.device(dev):
            index = torch.arange(3 * F, device=dev, dtype=torch.int32).reshape(1, F, 3).expand(B, F, 3).contiguous()
            ws = torch.empty(lib.umr_nmr_workspace_bytes(B, F, 0), device=dev, dtype=torch.uint8)
            fidx = torch.empty(B, S, S, device=dev, dtype=torch.int32)
            rdepth = torch.empty(B, S, S, device=dev, dtype=torch.float32)
            rgb = torch.empty(B, 3, IS, IS, device=dev, dtype=torch.float32) if want_rgb else None
            alpha = torch.empty(B, IS, IS, device=dev, dtype=torch.float32) if want_alpha else None
            depth = torch.empty(B, IS, IS, device=dev, dtype=torch.float32) if want_depth else None
            rc = lib.umr_nmr_forward(_ptr(verts), _ptr(index), _ptr(tex), _ptr(fidx), _ptr(rdepth), _ptr(rgb),
                                     _ptr(alpha), _ptr(depth), ctypes.byref(params), _ptr(ws), _stream_ptr(dev))
        _lib.check(rc, "umr_nmr_forward")
        ctx.params, ctx.eps = params, eps
        ctx.det = torch.are_deterministic_algorithms_enabled()
        ctx.dtypes = (faces.dtype, None if textures is None else textures.dtype)
        ctx.save_for_backward(verts, index, fidx, tex)
        return rgb, alpha, depth

    @staticmethod
    def backward(ctx, grad_rgb, grad_alpha, grad_depth):
        lib = _lib.load()
        verts, index, fidx, tex = ctx.saved_tensors
        p = ctx.params
        dev = verts.device
        B, F, IS = p.batch_size, p.num_faces, p.image_size
        g = [None if t is None else t.contiguous().float() for t in (grad_rgb, grad_alpha, grad_depth)]
        if tex is None:
            g[0] = None
        grad_faces = grad_tex = None
        with torch.cuda.device(dev):
            if ctx.needs_input_grad[0]:
                grad_faces = torch.empty(B, F, 3, 3, device=dev, dtype=torch.float32)
                ws = torch.empty(lib.umr_nmr_backward_faces_workspace_bytes(B, F, IS, p.anti_aliasing), device=dev,
                                 dtype=torch.uint8)
                rc = lib.umr_nmr_backward_faces(_ptr(verts), _ptr(index), _ptr(fidx), _ptr(tex), _ptr(g[0]), _ptr(g[1]),
                                                _ptr(g[2]), _ptr(grad_faces), ctypes.byref(p), ctx.eps, _ptr(ws),
                                                _stream_ptr(dev))
                _lib.check(rc, "umr_nmr_backward_faces")
                grad_faces = grad_faces.to(ctx.dtypes[0])
            if ctx.needs_input_grad[1]:
                if g[0] is None:
                    grad_tex = torch.zeros(tex.shape, device=dev, dtype=ctx.dtypes[1])
                else:
                    ws = torch.empty(lib.umr_nmr_workspace_bytes(B, F, 0), device=dev, dtype=torch.uint8)
                    grad_tex = torch.empty(tex.shape, device=dev, dtype=torch.float32)
                    name = "umr_nmr_backward_textures_deterministic" if ctx.det else "umr_nmr_backward_textures"
                    rc = getattr(lib, name)(_ptr(verts), _ptr(index), _ptr(fidx), _ptr(g[0]), _ptr(grad_tex),
                                            ctypes.byref(p), _ptr(ws), _stream_ptr(dev))
                    _lib.check(rc, name)
                    grad_tex = grad_tex.to(ctx.dtypes[1])
        return grad_faces, grad_tex, None, None, None, None, None


def rasterize_rgbad(faces, textures=None, image_size=DEFAULT_IMAGE_SIZE, anti_aliasing=DEFAULT_ANTI_ALIASING,
                    near=DEFAULT_NEAR, far=DEFAULT_FAR, eps=DEFAULT_EPS, background_color=DEFAULT_BACKGROUND_COLOR,
                    return_rgb=True, return_alpha=True, return_depth=True):
    """faces [B,F,3,3] in NDC, textures [B,F,T,T,T,3] (needed for rgb) -> {'rgb': [B,3,is,is] | None,
    'alpha': [B,is,is] | None, 'depth': [B,is,is] | None}.  Float64 inputs are rendered in float32; their gradients
    come back in float64."""
    if not torch.is_tensor(faces) or faces.dim() != 4 or tuple(faces.shape[2:]) != (3, 3) or faces.shape[0] < 1 \
            or faces.shape[1] < 1:
        raise ValueError("neural_renderer: faces [B,F,3,3] expected, got %s"
                         % (tuple(faces.shape) if torch.is_tensor(faces) else type(faces).__name__,))
    if not faces.is_floating_point():
        raise ValueError("neural_renderer: faces must be floating point, got %s" % (faces.dtype,))
    B, F = faces.shape[:2]
    if F > _MAX_FACES:
        raise ValueError("neural_renderer: at most %d faces, got %d" % (_MAX_FACES, F))
    if not (return_rgb or return_alpha or return_depth):
        raise ValueError("neural_renderer: nothing to return (return_rgb, return_alpha and return_depth are all False)")
    image_size = int(image_size)
    if image_size < 1:
        raise ValueError("neural_renderer: image_size must be positive, got %d" % image_size)
    eps = float(eps)
    if not 0.0 <= eps < float("inf"):
        raise ValueError("neural_renderer: eps must be finite and >= 0, got %r" % eps)
    bg = [float(a) for a in (background_color.tolist() if torch.is_tensor(background_color) else background_color)]
    if len(bg) != 3:
        raise ValueError("neural_renderer: background_color must have 3 components, got %r" % (background_color,))
    T = 0
    if textures is not None:
        if not torch.is_tensor(textures) or textures.dim() != 6 or tuple(textures.shape[:2]) != (B, F) \
                or textures.shape[3] != textures.shape[2] or textures.shape[4] != textures.shape[2] \
                or textures.shape[5] != 3:
            raise ValueError("neural_renderer: textures [B,F,T,T,T,3] with B = %d, F = %d expected, got %s"
                             % (B, F, tuple(textures.shape) if torch.is_tensor(textures) else type(textures).__name__))
        T = textures.shape[2]
        if T < 2:
            raise NotImplementedError("neural_renderer: texture size T=%d is not built (T >= 2)" % T)
    elif return_rgb:
        raise ValueError("neural_renderer: return_rgb needs textures")
    if not faces.is_cuda or (textures is not None and (not textures.is_cuda or textures.device != faces.device)):
        raise TypeError("neural_renderer supports only cuda tensors (faces and textures on one device)")
    params = _params(B, F, T, image_size, anti_aliasing, near, far, bg)
    rgb, alpha, depth = _RasterizeFunction.apply(faces, textures if return_rgb else None, params, eps, bool(return_rgb),
                                                 bool(return_alpha), bool(return_depth))
    return {"rgb": rgb, "alpha": alpha, "depth": depth}


def rasterize(faces, textures, image_size=DEFAULT_IMAGE_SIZE, anti_aliasing=DEFAULT_ANTI_ALIASING, near=DEFAULT_NEAR,
              far=DEFAULT_FAR, eps=DEFAULT_EPS, background_color=DEFAULT_BACKGROUND_COLOR):
    """[B,3,is,is] rgb."""
    return rasterize_rgbad(faces, textures, image_size, anti_aliasing, near, far, eps, background_color, True, False,
                           False)["rgb"]


def rasterize_silhouettes(faces, image_size=DEFAULT_IMAGE_SIZE, anti_aliasing=DEFAULT_ANTI_ALIASING, near=DEFAULT_NEAR,
                          far=DEFAULT_FAR, eps=DEFAULT_EPS):
    """[B,is,is] alpha."""
    return rasterize_rgbad(faces, None, image_size, anti_aliasing, near, far, eps, DEFAULT_BACKGROUND_COLOR, False,
                           True, False)["alpha"]


def rasterize_depth(faces, image_size=DEFAULT_IMAGE_SIZE, anti_aliasing=DEFAULT_ANTI_ALIASING, near=DEFAULT_NEAR,
                    far=DEFAULT_FAR, eps=DEFAULT_EPS):
    """[B,is,is] depth (far where no face is drawn)."""
    return rasterize_rgbad(faces, None, image_size, anti_aliasing, near, far, eps, DEFAULT_BACKGROUND_COLOR, False,
                           False, True)["depth"]


def vertices_to_faces(vertices, faces):
    """vertices [B,V,3], faces [B,F,3] integer -> face coordinates [B,F,3,3] (a differentiable gather)."""
    if vertices.dim() != 3 or vertices.shape[2] != 3 or faces.dim() != 3 or faces.shape[2] != 3 \
            or faces.shape[0] != vertices.shape[0]:
        raise ValueError("neural_renderer: vertices [B,V,3] and faces [B,F,3] expected, got %s and %s"
                         % (tuple(vertices.shape), tuple(faces.shape)))
    if faces.is_floating_point() or faces.is_complex():
        raise ValueError("neural_renderer: faces must be an integer tensor, got %s" % (faces.dtype,))
    B, V = vertices.shape[:2]
    idx = faces.to(device=vertices.device, dtype=torch.long)
    if idx.numel() and (idx.min() < 0 or idx.max() >= V):
        raise ValueError("neural_renderer: face indices must lie in [0, %d)" % V)
    return torch.gather(vertices, 1, idx.reshape(B, -1, 1).expand(-1, -1, 3)).reshape(B, faces.shape[1], 3, 3)
