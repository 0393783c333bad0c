"""`Renderer`: NMR's keyword names and defaults, UMR's configuration, kernels of csrc/nmr.cu (C ABI umr_nmr_*)."""
import ctypes
import math

import torch

from .. import _lib
from ..raster import _ptr, _stream_ptr

_NO_VERTEX_GRAD = (
    "neural_renderer: NMR's approximate vertex / camera gradient is not built -- only the textures get a gradient.  "
    "Every UMR call site renders detached geometry (experiments/train_s2.py:246,248,322-324; demo.py:110 under "
    "torch.no_grad; nnutils/loss_utils.py:311 pred_vs.detach()): detach the vertices and cameras, or render under "
    "torch.no_grad()")


class _NmrFunction(torch.autograd.Function):
    """(textures | None, vertices, faces) -> (rgb | None, alpha | None, depth | None); gradient for textures only.
    Under torch.use_deterministic_algorithms(True), read once in `forward`, the texture gradient is the bitwise
    reproducible face-parallel gather (umr_nmr_backward_textures_deterministic)."""

    @staticmethod
    def forward(ctx, textures, vertices, faces, params, want_rgb, want_alpha, want_depth):
        lib = _lib.load()
        dev = vertices.device
        B, IS = params.batch_size, params.image_size
        S = IS * (2 if params.anti_aliasing else 1)
        with torch.cuda.device(dev):
            ws = torch.empty(lib.umr_nmr_workspace_bytes(B, params.num_faces, params.fill_back), device=dev,
                             dtype=torch.uint8)
            fidx = torch.empty(B, S, S, device=dev, dtype=torch.int32)
            rdepth = torch.empty(B, S, S, device=dev, dtype=torch.float32)
            rgb = torch.empty(B, 3, IS, IS, device=dev, dtype=torch.float32) if want_rgb else None
            alpha = torch.empty(B, IS, IS, device=dev, dtype=torch.float32) if want_alpha else None
            depth = torch.empty(B, IS, IS, device=dev, dtype=torch.float32) if want_depth else None
            rc = lib.umr_nmr_forward(_ptr(vertices), _ptr(faces), _ptr(textures), _ptr(fidx), _ptr(rdepth), _ptr(rgb),
                                     _ptr(alpha), _ptr(depth), ctypes.byref(params), _ptr(ws), _stream_ptr(dev))
        _lib.check(rc, "umr_nmr_forward")
        ctx.params = params
        ctx.det = torch.are_deterministic_algorithms_enabled()   # the forward has no atomics; the backward's mode
        ctx.tex_shape = None if textures is None else textures.shape
        ctx.save_for_backward(vertices, faces, fidx)
        for t in (alpha, depth):
            if t is not None:
                ctx.mark_non_differentiable(t)
        return rgb, alpha, depth

    @staticmethod
    def backward(ctx, grad_rgb, grad_alpha, grad_depth):
        if grad_rgb is None or ctx.tex_shape is None or not ctx.needs_input_grad[0]:
            return (None,) * 7
        lib = _lib.load()
        vertices, faces, fidx = ctx.saved_tensors
        p = ctx.params
        dev = vertices.device
        g = grad_rgb.contiguous().float()
        with torch.cuda.device(dev):
            ws = torch.empty(lib.umr_nmr_workspace_bytes(p.batch_size, p.num_faces, p.fill_back), device=dev,
                             dtype=torch.uint8)
            grad_tex = torch.empty(ctx.tex_shape, device=dev, dtype=torch.float32)
            bwd = lib.umr_nmr_backward_textures_deterministic if ctx.det else lib.umr_nmr_backward_textures
            rc = bwd(_ptr(vertices), _ptr(faces), _ptr(fidx), _ptr(g), _ptr(grad_tex), ctypes.byref(p), _ptr(ws),
                     _stream_ptr(dev))
        _lib.check(rc, "umr_nmr_backward_textures_deterministic" if ctx.det else "umr_nmr_backward_textures")
        return (grad_tex,) + (None,) * 6


class Renderer(torch.nn.Module):
    """neural_renderer.Renderer for UMR's configuration.  `eye`, the `light_*` attributes and `background_color` are
    plain attributes read at every call (nmr_pytorch.py:95,98,105-115 assign them)."""

    def __init__(self, image_size=256, anti_aliasing=True, background_color=[0, 0, 0], fill_back=True,
                 camera_mode="projection", perspective=True, viewing_angle=30, near=0.1, far=100,
                 light_intensity_ambient=0.5, light_intensity_directional=0.5, light_color_ambient=[1, 1, 1],
                 light_color_directional=[1, 1, 1], light_direction=[0, 1, 0]):
        super().__init__()
        self.image_size = image_size
        self.anti_aliasing = anti_aliasing
        self.background_color = background_color
        self.fill_back = fill_back
        self.camera_mode = camera_mode
        self.perspective = perspective
        self.viewing_angle = viewing_angle
        self.eye = [0, 0, -(1. / math.tan(math.radians(viewing_angle)) + 1)]
        self.near = near
        self.far = far
        self.light_intensity_ambient = light_intensity_ambient
        self.light_intensity_directional = light_intensity_directional
        self.light_color_ambient = light_color_ambient
        self.light_color_directional = light_color_directional
        self.light_direction = light_direction
        self._check_camera()

    def _check_camera(self):
        if self.camera_mode != "look_at":
            raise NotImplementedError("neural_renderer: camera_mode=%r is not built (only 'look_at', UMR's "
                                      "configuration)" % (self.camera_mode,))
        if self.perspective:
            raise NotImplementedError("neural_renderer: perspective=True is not built (only the orthographic "
                                      "look_at camera UMR uses)")
        eye = [float(e) for e in self.eye]
        if len(eye) != 3 or eye[0] != 0.0 or eye[1] != 0.0 or not eye[2] < 0.0:
            raise NotImplementedError("neural_renderer: eye=%r is not built (only an eye (0, 0, e) with e < 0, where "
                                      "look_at is a translation along z)" % (self.eye,))

    @staticmethod
    def _vec3(x, name):
        v = [float(a) for a in (x.tolist() if torch.is_tensor(x) else x)]
        if len(v) != 3:
            raise ValueError("neural_renderer: %s must have 3 components, got %r" % (name, x))
        return v

    def _params(self, B, V, F, T, G):
        p = _lib.UmrNmrParams()
        p.batch_size, p.num_vertices, p.num_faces, p.texture_res = B, V, F, T
        p.image_size, p.anti_aliasing, p.fill_back = int(self.image_size), int(bool(self.anti_aliasing)), int(bool(self.fill_back))
        p.shared_textures = G
        p.eye_z = float(self.eye[2])
        p.near_plane, p.far_plane = float(self.near), float(self.far)
        p.light_intensity_ambient = float(self.light_intensity_ambient)
        p.light_intensity_directional = float(self.light_intensity_directional)
        p.light_color_ambient[:] = self._vec3(self.light_color_ambient, "light_color_ambient")
        p.light_color_directional[:] = self._vec3(self.light_color_directional, "light_color_directional")
        p.light_direction[:] = self._vec3(self.light_direction, "light_direction")
        p.background_color[:] = self._vec3(self.background_color, "background_color")
        return p

    def _render(self, vertices, faces, textures, want_rgb, want_alpha, want_depth):
        self._check_camera()
        if torch.is_grad_enabled() and vertices.requires_grad:
            raise NotImplementedError(_NO_VERTEX_GRAD)
        if vertices.dim() != 3 or vertices.shape[2] != 3 or faces.dim() != 3 or faces.shape[2] != 3 \
                or faces.shape[0] != vertices.shape[0]:
            raise ValueError("neural_renderer: vertices [B,V,3] and faces [B,F,3] expected, got %s and %s"
                             % (tuple(vertices.shape), tuple(faces.shape)))
        B, V, F = vertices.shape[0], vertices.shape[1], faces.shape[1]
        T, G, tex = 0, 1, None
        if textures is not None:
            T = textures.shape[2] if textures.dim() == 6 else 0
            if textures.dim() != 6 or textures.shape[1] != F or tuple(textures.shape[3:]) != (T, T, 3) \
                    or textures.shape[0] < 1 or B % textures.shape[0] != 0:
                raise ValueError("neural_renderer: textures [B,F,T,T,T,3] expected, got %s" % (tuple(textures.shape),))
            if T < 2:
                raise NotImplementedError("neural_renderer: texture size T=%d is not built (T >= 2; NMR indexes past "
                                          "the texture cube for T = 1)" % T)
            G = B // textures.shape[0]   # G consecutive renders sharing one texture (camera hypotheses)
        if not vertices.is_cuda or (textures is not None and not textures.is_cuda):
            raise TypeError("neural_renderer supports only cuda tensors")
        if textures is not None:
            tex = textures.contiguous().float()
        verts = vertices.detach().contiguous().float()
        fcs = faces.detach().to(device=vertices.device, dtype=torch.int32).contiguous()
        params = self._params(B, V, F, T, G)
        return _NmrFunction.apply(tex, verts, fcs, params, want_rgb, want_alpha, want_depth)

    def render_silhouettes(self, vertices, faces):
        """[B, is, is] coverage."""
        return self._render(vertices, faces, None, False, True, False)[1]

    def render_depth(self, vertices, faces):
        """[B, is, is] depth (far where no face is drawn)."""
        return self._render(vertices, faces, None, False, False, True)[2]

    def render_rgb(self, vertices, faces, textures):
        """textures [B,F,T,T,T,3] -> [B, 3, is, is]."""
        return self._render(vertices, faces, textures, True, False, False)[0]

    def render(self, vertices, faces, textures):
        """(rgb [B,3,is,is], depth [B,is,is], alpha [B,is,is])."""
        rgb, alpha, depth = self._render(vertices, faces, textures, True, True, True)
        return rgb, depth, alpha

    def forward(self, vertices, faces, textures=None, mode=None):
        if mode is None:
            return self.render(vertices, faces, textures)
        if mode == "rgb":
            return self.render_rgb(vertices, faces, textures)
        if mode == "silhouettes":
            return self.render_silhouettes(vertices, faces)
        if mode == "depth":
            return self.render_depth(vertices, faces)
        raise ValueError("mode should be one of None, 'silhouettes' or 'depth'")
