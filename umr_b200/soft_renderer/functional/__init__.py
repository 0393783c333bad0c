"""Functional layer of the drop-in package (reference: SoftRas/functional/__init__.py)."""
from .geometry import (face_vertices, get_points_from_angles, look, look_at, orthogonal, perspective, projection,
                       vertex_normals)
from .lights import ambient_lighting, directional_lighting
from .soft_rasterize import soft_rasterize
from .obj_io import create_texture_image, load_mtl, load_obj, load_textures, save_obj, save_voxel
from .voxelization import voxelization
