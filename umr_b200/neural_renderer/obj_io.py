"""neural_renderer's `load_obj` / `save_obj`, geometry only (DESIGN.md §15), on soft_renderer's OBJ parser and writer.

Textures are not built: `load_obj(..., load_texture=True)` and `save_obj(..., textures=...)` raise NotImplementedError.
"""
from ..soft_renderer.functional import obj_io


def load_obj(filename_obj, normalization=True, texture_size=4, load_texture=False, texture_wrapping="REPEAT",
             use_bilinear=True):
    """Vertices [V,3] float32 and faces [F,3] int32 on the GPU.  Polygons are fan-triangulated from their first vertex;
    `v`, `v/vt`, `v//vn` and `v/vt/vn` face entries are accepted.  `normalization`: shift by the per-axis minimum,
    divide by the largest |coordinate|, multiply by 2 and subtract half the per-axis maximum, so the longest side spans
    [-1, 1] and the mesh is centred."""
    if load_texture:
        raise NotImplementedError("neural_renderer.load_obj: load_texture=True is not built (geometry only)")
    return obj_io.load_obj(filename_obj, normalization=normalization)


def save_obj(filename, vertices, faces, textures=None, texture_size_out=16):
    """Write vertices [V,3] and faces [F,3] (0-based) as `v` and `f` lines."""
    if textures is not None:
        raise NotImplementedError("neural_renderer.save_obj: textures=... is not built (geometry only)")
    obj_io.save_obj(filename, vertices, faces)
