"""Lighting of the drop-in package.  Reference: SoftRas/lighting.py (module / attribute names: UMR pokes
`renderer.lighting.ambient.light_intensity` and `renderer.lighting.directionals[0].light_intensity`,
nnutils/smr.py:63,70-71), functional/{ambient,directional}_lighting.py (the formulas)."""
import torch
import torch.nn as nn

from . import functional as srf
from ._args import bind


class _Light(nn.Module):
    FIELDS = ()

    def __init__(self, *args, **kwargs):
        super().__init__()
        for key, value in bind(type(self).__name__, self.FIELDS, args, kwargs).items():
            setattr(self, key, value)


class AmbientLighting(_Light):
    FIELDS = (("light_intensity", 0.5), ("light_color", (1, 1, 1)))

    def forward(self, light):
        return srf.ambient_lighting(light, self.light_intensity, self.light_color)


class DirectionalLighting(_Light):
    FIELDS = (("light_intensity", 0.5), ("light_color", (1, 1, 1)), ("light_direction", (0, 1, 0)))

    def forward(self, light, normals):
        return srf.directional_lighting(light, normals, self.light_intensity, self.light_color, self.light_direction)


class Lighting(nn.Module):
    """textures *= ambient + sum_d directional_d(normals); per face ('surface') or per vertex ('vertex')."""
    FIELDS = (("light_mode", "surface"), ("intensity_ambient", 0.5), ("color_ambient", (1, 1, 1)),
              ("intensity_directionals", 0.5), ("color_directionals", (1, 1, 1)), ("directions", (0, 1, 0)))

    def __init__(self, *args, **kwargs):
        super().__init__()
        cfg = bind("Lighting", self.FIELDS, args, kwargs)
        if cfg["light_mode"] not in ("surface", "vertex"):
            raise ValueError("Lighting mode only support surface and vertex")
        self.light_mode = cfg["light_mode"]
        self.ambient = AmbientLighting(cfg["intensity_ambient"], cfg["color_ambient"])
        self.directionals = nn.ModuleList([DirectionalLighting(cfg["intensity_directionals"], cfg["color_directionals"],
                                                               cfg["directions"])])

    def _needs_normals(self):
        return any(float(d.light_intensity) != 0.0 for d in self.directionals)

    def forward(self, mesh):
        per_face = self.light_mode == "surface"
        count = mesh.num_faces if per_face else mesh.num_vertices
        dtype = torch.float64 if mesh.vertices.dtype == torch.float64 else torch.float32
        light = self.ambient(torch.zeros(mesh.batch_size, count, 3, dtype=dtype, device=mesh.device))
        if self._needs_normals():  # zero-intensity lights add exactly 0: skip the normal computation
            normals = mesh.surface_normals if per_face else mesh.vertex_normals
            for directional in self.directionals:
                light = directional(light, normals)
        # [B,F,T2,3] * [B,F,1,3]   or   [B,V,3] * [B,V,3]
        mesh.textures = mesh.textures * (light[:, :, None, :] if per_face else light)
        return mesh
