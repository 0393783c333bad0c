"""`sr.Mesh`: a batched triangle-mesh container (reference: SoftRas/mesh.py -- attribute and property names).

Holds vertices [B,V,3], faces [B,F,3] (int) and textures (surface: [B,F,T2,3]; vertex: [B,V,3]).  Derived
quantities (`face_vertices`, `surface_normals`, `vertex_normals`) are cached until vertices or faces are
reassigned.  OBJ loading / saving (incl. the texture atlas kernels) live in functional/obj_io.py.
"""
import numpy as np

import torch
import torch.nn.functional as F

from . import functional as srf


def _tensor(x, dtype):
    """numpy arrays are moved to the GPU like the reference does (mesh.py:19-22); tensors pass through."""
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(x).to(dtype).cuda()
    return x


def _batched(x, unbatched_dims):
    return x[None] if x.dim() == unbatched_dims else x


class Mesh(object):
    def __init__(self, vertices, faces, textures=None, texture_res=1, texture_type="surface"):
        if texture_type not in ("surface", "vertex"):
            raise ValueError("texture type not applicable")
        self._vertices = _batched(_tensor(vertices, torch.float32), 2)
        self._faces = _batched(_tensor(faces, torch.int32), 2)
        self.device = self._vertices.device
        self.texture_type = texture_type
        self._cache = {}
        self._fill_back = False
        if textures is None:
            self._textures, self.texture_res = self._white(texture_res)
        else:
            textures = _tensor(textures, torch.float32)
            self._textures = _batched(textures, 3 if texture_type == "surface" else 2)
            self.texture_res = int(np.sqrt(self._textures.shape[2]))  # mesh.py:63
        self._origin = (self._vertices, self._faces, self._textures)

    def _white(self, texture_res):
        """All-ones texture (mesh.py:44-54): [B,F,res^2,3] per face or [B,V,3] per vertex."""
        if self.texture_type == "surface":
            shape, res = (self.batch_size, self.num_faces, texture_res ** 2, 3), texture_res
        else:
            shape, res = (self.batch_size, self.num_vertices, 3), 1
        # float64 vertices render in double precision: their default texture follows them
        dtype = torch.float64 if self._vertices.dtype == torch.float64 else torch.float32
        return torch.ones(shape, dtype=dtype, device=self.device), res

    # --- sizes ------------------------------------------------------------------------------
    @property
    def batch_size(self):
        return self._vertices.shape[0]

    @property
    def num_vertices(self):
        return self._vertices.shape[1]

    @property
    def num_faces(self):
        return self._faces.shape[1]

    # --- geometry (setting either invalidates the cached derived quantities) -----------------
    @property
    def vertices(self):
        return self._vertices

    @vertices.setter
    def vertices(self, value):
        self._vertices = value
        self._cache.clear()

    @property
    def faces(self):
        return self._faces

    @faces.setter
    def faces(self, value):
        self._faces = value
        self._cache.clear()

    @property
    def textures(self):
        return self._textures

    @textures.setter
    def textures(self, value):
        self._textures = value

    def _cached(self, key, compute):
        if key not in self._cache:
            self._cache[key] = compute()
        return self._cache[key]

    @property
    def face_vertices(self):
        return self._cached("fv", lambda: srf.face_vertices(self._vertices, self._faces))

    @property
    def surface_normals(self):
        def compute():  # mesh.py:112-118
            fv = self.face_vertices
            return F.normalize(torch.cross(fv[:, :, 2] - fv[:, :, 1], fv[:, :, 0] - fv[:, :, 1], dim=-1), p=2, dim=2,
                               eps=1e-6)
        return self._cached("sn", compute)

    @property
    def vertex_normals(self):
        return self._cached("vn", lambda: srf.vertex_normals(self._vertices, self._faces))

    @property
    def face_textures(self):
        if self.texture_type == "surface":
            return self._textures
        return srf.face_vertices(self._textures, self._faces)

    def fill_back_(self):
        if not self._fill_back:
            self.faces = torch.cat((self._faces, self._faces[:, :, [2, 1, 0]]), dim=1)
            self.textures = torch.cat((self._textures, self._textures), dim=1)
            self._fill_back = True

    def reset_(self):
        self.vertices, self.faces, self.textures = self._origin
        self._fill_back = False

    # --- host I/O (outside the hot path) ----------------------------------------------------
    def save_obj(self, filename_obj, save_texture=False, texture_res_out=16):
        """SoftRas/mesh.py:141-148: geometry, plus (save_texture) the texture atlas PNG / .mtl written from the
        `create_texture_image` kernel (csrc/mesh_ops.cu)."""
        if self.batch_size != 1:
            raise ValueError("Could not save when batch size >= 1")
        from .functional.obj_io import save_obj
        if save_texture:
            save_obj(filename_obj, self._vertices[0], self._faces[0], textures=self._textures[0],
                     texture_res=texture_res_out, texture_type=self.texture_type)
        else:
            save_obj(filename_obj, self._vertices[0], self._faces[0], textures=None)

    @classmethod
    def from_obj(cls, filename_obj, normalization=False, load_texture=False, texture_res=1, texture_type="surface"):
        from .functional.obj_io import load_obj
        loaded = load_obj(filename_obj, normalization, load_texture, texture_res, texture_type)
        textures = loaded[2] if load_texture else None
        return cls(loaded[0], loaded[1], textures, texture_res, texture_type)

    def voxelize(self, voxel_size=32):
        """SoftRas/mesh.py:177-179: the face vertices mapped by x * vs / (vs - 1) + 0.5, voxelised at vs^3 through the
        `voxelization` kernels -> int32 [B, vs, vs, vs]."""
        if voxel_size < 2:
            raise ValueError("voxel_size must be >= 2 (the reference divides by voxel_size - 1), got %r" % (voxel_size,))
        face_vertices_norm = self.face_vertices * voxel_size / (voxel_size - 1) + 0.5
        return srf.voxelization(face_vertices_norm, voxel_size, False)
