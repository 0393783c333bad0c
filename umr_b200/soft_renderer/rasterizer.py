"""`sr.SoftRasterizer` on the sm_90a kernels.  Reference: SoftRas/rasterizer.py:8-55 (argument names, defaults
and error messages); the 2x supersampling + `avg_pool2d` of rasterizer.py:43,52-53 is fused into the kernels."""
import torch.nn as nn

from ..raster import raster_calls_wrapped, soft_rasterize, soft_rasterize_silhouettes, soft_rasterize_split, visibility
from ._args import bind

# (name, default) in the reference's positional order
FIELDS = (("image_size", 256), ("background_color", (0, 0, 0)), ("near", 1), ("far", 100), ("anti_aliasing", False),
          ("fill_back", False), ("eps", 1e-3), ("sigma_val", 1e-5), ("dist_func", "euclidean"), ("dist_eps", 1e-4),
          ("gamma_val", 1e-4), ("aggr_func_rgb", "softmax"), ("aggr_func_alpha", "prod"), ("texture_type", "surface"))
CHOICES = {
    "dist_func": (("hard", "euclidean", "barycentric"), "Distance function only support hard, euclidean and barycentric"),
    "aggr_func_rgb": (("hard", "softmax"), "Aggregate function(rgb) only support hard and softmax"),
    "aggr_func_alpha": (("hard", "prod", "sum"), "Aggregate function(a) only support hard, prod and sum"),
    "texture_type": (("surface", "vertex"), "Texture type only support surface and vertex"),
}
# positional order of functional.soft_rasterize after (face_vertices, textures)
KERNEL_ARGS = ("image_size", "background_color", "near", "far", "fill_back", "eps", "sigma_val", "dist_func",
               "dist_eps", "gamma_val", "aggr_func_rgb", "aggr_func_alpha", "texture_type", "anti_aliasing")


class SoftRasterizer(nn.Module):
    """Every field of FIELDS is a plain attribute (UMR overwrites e.g. `background_color`, nnutils/smr.py:74)."""

    def __init__(self, *args, **kwargs):
        super().__init__()
        cfg = bind("SoftRasterizer", FIELDS, args, kwargs)
        for key, (allowed, message) in CHOICES.items():
            if cfg[key] not in allowed:
                raise ValueError(message)
        for key, value in cfg.items():
            setattr(self, key, value)

    def rasterize(self, face_vertices, face_textures):
        """Rasterise raster-space face vertices [B,F,3,3] with face textures [B,F,T2,3]."""
        return soft_rasterize(face_vertices, face_textures, *[getattr(self, k) for k in KERNEL_ARGS])

    def rasterize_split(self, face_vertices, face_textures):
        """`rasterize` whose backward sends the alpha plane's gradient to the geometry and the RGB planes' gradient to the
        textures only (raster.soft_rasterize_split); see supports_split."""
        return soft_rasterize_split(face_vertices, face_textures, *[getattr(self, k) for k in KERNEL_ARGS])

    def supports_split(self):
        """The split backward exists for UMR's configuration (euclidean / prod / surface), softmax or hard colours."""
        return self.dist_func == "euclidean" and self.aggr_func_alpha == "prod" and self.texture_type == "surface"

    def rasterize_silhouettes(self, face_vertices):
        """The alpha plane [B,is,is] of `rasterize` (whatever the textures and colour mode), rendered without colour
        (raster.soft_rasterize_silhouettes); see supports_silhouettes."""
        return soft_rasterize_silhouettes(face_vertices, self.image_size, self.near, self.far, self.fill_back, self.eps,
                                          self.sigma_val, self.dist_eps, self.gamma_val, self.anti_aliasing)

    def supports_silhouettes(self):
        """The silhouette kernels exist for UMR's configuration (euclidean distance, prod alpha, surface textures).  While a
        wrapper is installed on SoftRasterizeFunction.apply (raster.raster_calls_wrapped) callers render in full, through
        it."""
        return (self.dist_func == "euclidean" and self.aggr_func_alpha == "prod" and self.texture_type == "surface"
                and not raster_calls_wrapped())

    def supports_visibility(self):
        """The visibility-only kernel exists for UMR's configuration of the hard renderer (nnutils/smr.py:52-58)."""
        return (self.dist_func == "euclidean" and self.aggr_func_alpha == "prod" and self.texture_type == "surface"
                and self.aggr_func_rgb == "hard")

    def visibility(self, face_vertices, want_faces=False):
        """aggrs_info [B,2,S,S] of the hard z-buffer (depth_min, face_index_min) without rendering the image; or, with
        want_faces, only the [B,F] uint8 "face is visible" bytes."""
        return visibility(face_vertices, self.image_size, self.near, self.far, self.fill_back, self.eps, self.sigma_val,
                          self.dist_eps, self.gamma_val, self.anti_aliasing, want_faces)

    def forward(self, mesh, mode=None):
        return self.rasterize(mesh.face_vertices, mesh.face_textures)
