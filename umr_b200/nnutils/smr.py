"""`SoftRenderer` -- THE drop-in boundary (reference: nnutils/smr.py:49-87).

Same constructor, same methods (`forward`, `project_points`, `ambient_light_only`, `set_bgcolor`)
and the same attribute paths the reference pokes (`renderer.transform.transformer._eye`,
`renderer.lighting.ambient.light_intensity`, ...).  forward() returns
(images [B,4,is,is], p2f_info [B,F,2], aggrs_info [B,2,S,S]) with S = 2*is (anti_aliasing).
"""
import torch

from .. import soft_renderer as sr
from ..vertex import project_faces
from . import geom_utils


class Render(torch.nn.Module):
    """smr.py:29-44: y-flip, wrap into a Mesh, render."""

    def __init__(self, renderer):
        super().__init__()
        self.renderer = renderer

    def forward(self, vertices, faces, textures=None):
        vs = vertices
        vs[:, :, 1] *= -1  # in place, like the reference (smr.py:36)
        mesh_ = sr.Mesh(vs, faces) if textures is None else sr.Mesh(vs, faces, textures)
        return self.renderer.render_mesh(mesh_)


class SoftRenderer(torch.nn.Module):
    def __init__(self, img_size=256, render_type="softmax", background_color=[0, 0, 0], sigma_val=1e-5,
                 gamma_val=1e-4, dist_eps=1e-10, anti_aliasing=True):
        super().__init__()
        self.renderer = sr.SoftRenderer(image_size=img_size, aggr_func_rgb=render_type, camera_mode="look_at",
                                        sigma_val=sigma_val, dist_eps=dist_eps, gamma_val=gamma_val,
                                        background_color=background_color, anti_aliasing=anti_aliasing,
                                        perspective=False)
        self.renderer.transform.transformer._eye = [0, 0, -2.732]  # smr.py:60
        self.renderer.lighting.ambient.light_intensity = 0.8       # smr.py:63
        self.proj_fn = geom_utils.orthographic_proj_withz
        self.offset_z = 5.

    def ambient_light_only(self):
        self.renderer.lighting.ambient.light_intensity = 1
        self.renderer.lighting.directionals[0].light_intensity = 0

    def set_bgcolor(self, color):
        self.renderer.rasterizer.background_color = color

    def project_points(self, verts, cams):
        return self.proj_fn(verts, cams)[:, :, :2]

    # -- fused path ---------------------------------------------------------------------------------
    fuse_vertex_pipeline = True  # class-level switch (tests compare both paths)

    def _fusable(self, vertices):
        """True when forward() takes the fused vertex kernel.  Under torch.use_deterministic_algorithms(True) too: its
        backward then takes the deterministic gather (vertex.ProjectFacesFunction)."""
        return self._projectable(vertices)

    def _projectable(self, vertices):
        """The fused vertex kernel covers exactly the configuration this wrapper sets up (smr.py:56-66):
        look_at camera with the eye on the z axis, orthographic, surface lighting with at most the one
        default directional light, in float32.  Anything else takes the generic torch path below; float64 vertices then
        reach the float64 rasteriser."""
        r = self.renderer
        tr = r.transform.transformer
        eye = getattr(tr, "_eye", None)
        if not (self.fuse_vertex_pipeline and vertices.is_cuda and vertices.dtype != torch.float64 and r.transform.camera_mode == "look_at"
                and not tr.perspective and isinstance(eye, (list, tuple)) and len(eye) == 3):
            return False
        if float(eye[0]) != 0.0 or float(eye[1]) != 0.0 or not float(eye[2]) < 0.0:
            return False
        if self.proj_fn is not geom_utils.orthographic_proj_withz or len(r.lighting.directionals) != 1:
            return False
        return r.rasterizer.texture_type == "surface"

    def _forward_fused(self, vertices, faces, cams, textures):
        r = self.renderer
        tr = r.transform.transformer
        amb, dl = r.lighting.ambient, r.lighting.directionals[0]
        light_cfg = None
        if float(dl.light_intensity) != 0.0:
            light_cfg = (amb.light_intensity, amb.light_color, dl.light_intensity, dl.light_color, dl.light_direction)
        fv, light = project_faces(vertices, cams, faces, offset_z=self.offset_z, eye_z=float(tr._eye[2]),
                                  viewing_scale=tr.viewing_scale, flip_y=True, light=light_cfg)
        B, F = fv.shape[:2]
        if light is not None:
            # ones * light == light; textures * light[:, :, None, :] as in lighting.py:57
            if textures is not None and textures.shape[0] not in (1, B):   # hypothesis-shared textures meet a per-render light
                textures = textures.repeat_interleave(B // textures.shape[0], dim=0)
            tex = light[:, :, None, :] if textures is None else textures * light[:, :, None, :]
        else:
            c = [float(amb.light_intensity) * float(k) for k in amb.light_color]
            if textures is None:
                tex = torch.tensor(c, dtype=torch.float32, device=fv.device).view(1, 1, 1, 3).expand(1, F, 1, 3)  # one texture shared by the batch
            elif c == [1.0, 1.0, 1.0]:
                tex = textures  # x * 1 == x
            else:
                tex = textures * torch.tensor(c, dtype=torch.float32, device=fv.device)
        return r.rasterizer.rasterize(fv, tex)

    def visibility(self, vertices, faces, cams):
        """(p2f_info, aggrs_info) of this renderer WITHOUT the image: what `MultiTextureLoss` keeps of its hard render
        (loss_utils.py:327-329, `_, p2f_info, aggr_info = self.hard_renderer(...)`).  For the hard renderer on CUDA this
        runs the visibility-only kernel (z-buffer winner per pixel; p2f_info is zero in hard mode, kernel.cu:417-431);
        every other configuration renders normally and drops the image."""
        r = self.renderer
        if self._projectable(vertices) and r.rasterizer.supports_visibility():
            tr = r.transform.transformer
            fv, _ = project_faces(vertices.detach(), cams.detach(), faces, offset_z=self.offset_z, eye_z=float(tr._eye[2]),
                                  viewing_scale=tr.viewing_scale, flip_y=True, light=None)
            aggrs = r.rasterizer.visibility(fv)
            return torch.zeros(fv.shape[0], fv.shape[1], 2, device=fv.device, dtype=torch.float32), aggrs
        _, p2f, aggrs = self.forward(vertices, faces, cams)
        return p2f, aggrs

    def visible_faces(self, vertices, faces, cams):
        """(p2f_info, visible [B,F] uint8) -- the set of faces TexCycle extracts from the hard render's face-index plane
        (loss_utils.py:161-166), computed by the visibility kernel itself so that no plane is written or re-read.
        None when this renderer / device has no visibility kernel (callers then use `visibility` / `forward`)."""
        r = self.renderer
        if not (self._projectable(vertices) and r.rasterizer.supports_visibility()):
            return None
        tr = r.transform.transformer
        fv, _ = project_faces(vertices.detach(), cams.detach(), faces, offset_z=self.offset_z, eye_z=float(tr._eye[2]),
                              viewing_scale=tr.viewing_scale, flip_y=True, light=None)
        mask = r.rasterizer.visibility(fv, want_faces=True)
        return torch.zeros(fv.shape[0], fv.shape[1], 2, device=fv.device, dtype=torch.float32), mask

    def forward(self, vertices, faces, cams, textures=None):
        """vertices [B,V,3], faces [B,F,3], cams [B,7], textures [B,F,T2,3] | None, as the reference (smr.py:80-87).
        Extension (SURVEY.md §8f-1): `cams` may hold H camera hypotheses per mesh -- cams [B*H,7] with vertices / faces
        [B,...] and textures [B,...] (or [1,...]) NOT repeated; the kernels broadcast instead of the reference's
        repeat(1, 8, ...) copies (loss_utils.py:260-261, 303-305).  Returns B*H renders."""
        if self._fusable(vertices):
            return self._forward_fused(vertices, faces, cams, textures)
        H = cams.shape[0] // vertices.shape[0]
        if H > 1:  # generic torch path: materialise the copies like the reference
            vertices = vertices.repeat_interleave(H, dim=0)
            faces = faces.repeat_interleave(H, dim=0) if faces.dim() == 3 and faces.shape[0] > 1 else faces
            if textures is not None and textures.shape[0] > 1:
                textures = textures.repeat_interleave(cams.shape[0] // textures.shape[0], dim=0)
        faces = faces.int()
        if faces.dim() == 2:
            faces = faces[None]
        if faces.shape[0] == 1 and cams.shape[0] > 1:  # one face list for every render, as the fused path accepts it
            faces = faces.expand(cams.shape[0], -1, -1)
        verts = self.proj_fn(vertices, cams, offset_z=self.offset_z)
        if textures is not None:
            return Render(self.renderer)(verts, faces, textures)
        return Render(self.renderer)(verts, faces)
