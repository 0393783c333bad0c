"""torch.autograd binding of the fused vertex pipeline (csrc/vertex.cu, include/umr_b200.h).

project_faces(vertices, cams, faces, ...) = orthographic_proj_withz -> y flip -> look_at(eye on z)
-> orthogonal -> face gather [-> per-face surface light], one kernel forward and two backward,
replacing ~70 tiny torch launches per render of the reference host path (SURVEY.md §8f-1).

Under torch.use_deterministic_algorithms(True) (read once in `forward`, kept in `ctx`) the backward takes
umr_project_faces_backward_deterministic: a gather over the faces' vertex -> corner table instead of float atomics."""
import ctypes

import torch

from . import _lib
from .ops import device_incidence
from .raster import _ptr, _stream_ptr


def make_project_params(B, V, F, faces_bstride, offset_z, eye_z, viewing_scale, flip_y, light, hypotheses=1):
    p = _lib.UmrProjectParams()
    p.batch_size, p.num_vertices, p.num_faces = B, V, F
    p.flip_y = 1 if flip_y else 0
    p.faces_batch_stride = faces_bstride
    p.offset_z, p.eye_z, p.viewing_scale = float(offset_z), float(eye_z), float(viewing_scale)
    p.num_hypotheses = int(hypotheses)
    if light is None:
        p.light_enabled = 0
    else:
        ia, ca, idir, cd, d = light
        p.light_enabled = 1
        p.light_intensity_ambient, p.light_intensity_directional = float(ia), float(idir)
        for k in range(3):
            p.light_color_ambient[k] = float(ca[k])
            p.light_color_directional[k] = float(cd[k])
            p.light_direction[k] = float(d[k])
    return p


def _corner_incidence(faces, V, batched):
    """vertex -> (face * 3 + corner) table of the deterministic backward (include/umr_b200.h): rows v over V vertices for
    one shared face list, rows vb * V + v over the meshes of batched faces [Bv,F,3].  A face index outside [0, V) has no
    row: the kernel stores zeros for such a face, and in a batched list it must not land in another mesh's rows."""
    if not batched:
        return device_incidence(faces, V)
    Bv = faces.shape[0]
    idx = faces.long()
    keys = (idx + torch.arange(Bv, device=faces.device, dtype=torch.int64).view(Bv, 1, 1) * V).masked_fill(
        (idx < 0) | (idx >= V), -1)
    return device_incidence(keys, Bv * V)


class ProjectFacesFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, vertices, cams, faces, offset_z, eye_z, viewing_scale, flip_y, light):
        if not vertices.is_cuda:
            raise TypeError("umr_b200 vertex pipeline supports only cuda Tensors")
        lib = _lib.load()
        dev = vertices.device
        v = vertices.detach().contiguous().float()
        c = cams.detach().contiguous().float()
        f = faces if (faces.dtype == torch.int32 and faces.is_contiguous()) else faces.int().contiguous()
        Bv, V = v.shape[:2]
        B = c.shape[0]                       # renders = cameras; Bv meshes, B / Bv camera hypotheses each
        if B % Bv != 0:
            raise ValueError("cams batch %d is not a multiple of the vertices batch %d" % (B, Bv))
        H = B // Bv
        if f.dim() == 2:
            F, fstride = f.shape[0], 0
        else:
            if f.shape[0] not in (1, Bv):
                raise ValueError("faces batch %d does not match the vertices batch %d" % (f.shape[0], Bv))
            F, fstride = f.shape[1], (f.shape[1] * 3 if f.shape[0] > 1 else 0)
        params = make_project_params(B, V, F, fstride, offset_z, eye_z, viewing_scale, flip_y, light, H)
        with torch.cuda.device(dev):
            fv = torch.empty(B, F, 3, 3, device=dev, dtype=torch.float32)
            lt = torch.empty(B, F, 3, device=dev, dtype=torch.float32) if light is not None else None
            rc = lib.umr_project_faces_forward(_ptr(v), _ptr(c), _ptr(f), _ptr(fv), _ptr(lt), ctypes.byref(params),
                                               _stream_ptr(dev))
        _lib.check(rc, "umr_project_faces_forward")
        ctx.params = params
        ctx.save_for_backward(v, c, f)
        ctx.needs = (vertices.requires_grad, cams.requires_grad)
        ctx.has_light = light is not None
        ctx.det = torch.are_deterministic_algorithms_enabled()   # the forward has no atomics; the backward's mode
        if lt is None:
            lt = fv.new_empty(0)
            ctx.mark_non_differentiable(lt)
        return fv, lt

    @staticmethod
    def backward(ctx, g_fv, g_light):
        lib = _lib.load()
        v, c, f = ctx.saved_tensors
        dev = v.device
        V = v.shape[1]
        B = c.shape[0]
        with torch.cuda.device(dev):
            if g_fv is None:
                g_fv = torch.zeros(B, ctx.params.num_faces, 9, device=dev, dtype=torch.float32)
            g = g_fv.contiguous().float()
            gl = g_light.contiguous().float() if (ctx.has_light and g_light is not None) else None
            gproj = torch.empty(B, V, 3, device=dev, dtype=torch.float32)
            gv = torch.empty_like(v) if ctx.needs[0] else None
            gc = torch.empty_like(c) if ctx.needs[1] else None
            if ctx.det:
                rowptr, inc = _corner_incidence(f, V, ctx.params.faces_batch_stride != 0)
                ws = torch.empty(lib.umr_project_faces_workspace_bytes_deterministic(B, V, ctx.params.num_faces), device=dev,
                                 dtype=torch.uint8)
                rc = lib.umr_project_faces_backward_deterministic(_ptr(v), _ptr(c), _ptr(f), _ptr(g), _ptr(gl), _ptr(gproj),
                                                                  _ptr(gv), _ptr(gc), ctypes.byref(ctx.params), _ptr(rowptr),
                                                                  _ptr(inc), _ptr(ws), _stream_ptr(dev))
            else:
                rc = lib.umr_project_faces_backward(_ptr(v), _ptr(c), _ptr(f), _ptr(g), _ptr(gl), _ptr(gproj), _ptr(gv),
                                                    _ptr(gc), ctypes.byref(ctx.params), _stream_ptr(dev))
        _lib.check(rc, "umr_project_faces_backward_deterministic" if ctx.det else "umr_project_faces_backward")
        return gv, gc, None, None, None, None, None, None


def project_faces(vertices, cams, faces, offset_z=5.0, eye_z=-2.732, viewing_scale=1.0, flip_y=True, light=None):
    """vertices [B,V,3], cams [B,7], faces [B,F,3] or [F,3] (int) ->
    (face_vertices [B,F,3,3] in raster space, light [B,F,3] or None).
    light = (Ia, colour_a, Id, colour_d, direction) or None."""
    fv, lt = ProjectFacesFunction.apply(vertices, cams, faces, offset_z, eye_z, viewing_scale, flip_y, light)
    return fv, (lt if light is not None else None)
