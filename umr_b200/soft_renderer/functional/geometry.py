"""Vertex-side helpers of the drop-in package (pure torch, a handful of tiny ops).

References: functional/face_vertices.py:4-22, look_at.py:6-62, look.py, orthogonal.py:4-17,
perspective.py, projection.py, vertex_normals.py, get_points_from_angles.py.  UMR itself only uses
look_at + orthogonal (`smr.py:56`), which the fused CUDA vertex pipeline covers; everything here is the
generic torch path of the drop-in package (SURVEY.md §8f-3).
"""
import math

import torch
import torch.nn.functional as F


def face_vertices(vertices, faces):
    """vertices [B,V,3], faces [B,F,3] (int) -> [B,F,3,3]: per-face corner coordinates."""
    if vertices.dim() != 3 or faces.dim() != 3 or vertices.shape[0] != faces.shape[0]:
        raise ValueError("face_vertices expects vertices [B,V,3] and faces [B,F,3]")
    B, V = vertices.shape[:2]
    idx = faces.long() + (torch.arange(B, device=vertices.device, dtype=torch.long) * V)[:, None, None]
    return vertices.reshape(B * V, vertices.shape[2])[idx]


def _as_batch(x, B, vertices):
    """A camera constant (eye, at, up, direction) as [B,3]: float64 beside float64 vertices, float32 otherwise."""
    dtype = torch.float64 if vertices.dtype == torch.float64 else torch.float32
    t = torch.as_tensor(x, dtype=dtype, device=vertices.device)
    if t.dim() == 1:
        t = t[None, :].expand(B, -1)
    return t


def look_at(vertices, eye, at=(0, 0, 0), up=(0, 1, 0)):
    """Camera frame with origin `eye` looking at `at` (look_at.py:48-60; normalise eps 1e-5)."""
    if vertices.dim() != 3:
        raise ValueError("vertices Tensor should have 3 dimensions")
    B = vertices.shape[0]
    eye, at, up = _as_batch(eye, B, vertices), _as_batch(at, B, vertices), _as_batch(up, B, vertices)
    z_axis = F.normalize(at - eye, eps=1e-5)
    x_axis = F.normalize(torch.cross(up, z_axis, dim=-1), eps=1e-5)
    y_axis = F.normalize(torch.cross(z_axis, x_axis, dim=-1), eps=1e-5)
    rot = torch.stack((x_axis, y_axis, z_axis), dim=1)  # [B,3,3], rows = axes
    return torch.matmul(vertices - eye[:, None, :], rot.transpose(1, 2))


def orthogonal(vertices, scale):
    """x, y scaled; z kept (orthogonal.py:13-16)."""
    if vertices.dim() != 3:
        raise ValueError("vertices Tensor should have 3 dimensions")
    return torch.stack((vertices[:, :, 0] * scale, vertices[:, :, 1] * scale, vertices[:, :, 2]), dim=2)


def perspective(vertices, angle=30.0):
    """Pinhole projection with half field-of-view `angle` degrees (functional/perspective.py)."""
    if vertices.dim() != 3:
        raise ValueError("vertices Tensor should have 3 dimensions")
    width = math.tan(math.radians(float(angle)))
    z = vertices[:, :, 2]
    return torch.stack((vertices[:, :, 0] / z / width, vertices[:, :, 1] / z / width, z), dim=2)


def _camera_frame(z_dir, up):
    """Right-handed camera axes (rows of the rotation) from a viewing direction and an up vector."""
    z_axis = F.normalize(z_dir, eps=1e-5)
    x_axis = F.normalize(torch.cross(up, z_axis, dim=-1), eps=1e-5)
    y_axis = F.normalize(torch.cross(z_axis, x_axis, dim=-1), eps=1e-5)
    return torch.stack((x_axis, y_axis, z_axis), dim=1)


def look(vertices, eye, direction=(0, 1, 0), up=(0, 1, 0)):
    """Camera at `eye` looking along `direction` (functional/look.py)."""
    if vertices.dim() != 3:
        raise ValueError("vertices Tensor should have 3 dimensions")
    B = vertices.shape[0]
    eye, direction, up = _as_batch(eye, B, vertices), _as_batch(direction, B, vertices), _as_batch(up, B, vertices)
    rot = _camera_frame(direction, up)
    return torch.matmul(vertices - eye[:, None, :], rot.transpose(1, 2))


def projection(vertices, P, dist_coeffs, orig_size):
    """Pinhole projection with a [B,3,4] matrix and 5 OpenCV-style distortion coefficients, mapped to
    [-1,1] image coordinates (functional/projection.py)."""
    hom = torch.cat([vertices, torch.ones_like(vertices[:, :, :1])], dim=-1)
    cam = torch.bmm(hom, P.transpose(2, 1))
    x, y, z = cam[:, :, 0], cam[:, :, 1], cam[:, :, 2]
    xn, yn = x / (z + 1e-5), y / (z + 1e-5)
    k1, k2, p1, p2, k3 = (dist_coeffs[:, None, i] for i in range(5))
    r2 = xn ** 2 + yn ** 2
    radial = 1 + k1 * r2 + k2 * r2 ** 2 + k3 * r2 ** 3
    xd = xn * radial + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn ** 2)
    yd = yn * radial + p1 * (r2 + 2 * yn ** 2) + 2 * p2 * xn * yn
    xs = 2 * (xd - orig_size / 2.) / orig_size
    ys = 2 * (yd - orig_size / 2.) / orig_size
    return torch.stack([xs, ys, z], dim=-1)


def vertex_normals(vertices, faces):
    """Area-weighted vertex normals: every face adds its (unnormalised) corner cross product to its three
    vertices, then normalise (functional/vertex_normals.py)."""
    if vertices.dim() != 3 or faces.dim() != 3 or vertices.shape[0] != faces.shape[0]:
        raise ValueError("vertex_normals expects vertices [B,V,3] and faces [B,F,3]")
    B, V = vertices.shape[:2]
    idx = (faces.long() + (torch.arange(B, device=vertices.device, dtype=torch.long) * V)[:, None, None]).view(-1, 3)
    flat = vertices.reshape(B * V, 3)
    c = flat[idx]  # [B*F, 3 corners, 3]
    normals = torch.zeros(B * V, 3, device=vertices.device, dtype=vertices.dtype)
    normals.index_add_(0, idx[:, 1], torch.cross(c[:, 2] - c[:, 1], c[:, 0] - c[:, 1], dim=-1))
    normals.index_add_(0, idx[:, 2], torch.cross(c[:, 0] - c[:, 2], c[:, 1] - c[:, 2], dim=-1))
    normals.index_add_(0, idx[:, 0], torch.cross(c[:, 1] - c[:, 0], c[:, 2] - c[:, 0], dim=-1))
    return F.normalize(normals, eps=1e-6, dim=1).reshape(B, V, 3)


def get_points_from_angles(distance, elevation, azimuth, degrees=True):
    """Eye position on a sphere around the origin (functional/get_points_from_angles.py)."""
    if isinstance(distance, (float, int)):
        if degrees:
            elevation, azimuth = math.radians(elevation), math.radians(azimuth)
        return (distance * math.cos(elevation) * math.sin(azimuth), distance * math.sin(elevation),
                -distance * math.cos(elevation) * math.cos(azimuth))
    if degrees:
        elevation, azimuth = math.pi / 180. * elevation, math.pi / 180. * azimuth
    return torch.stack([distance * torch.cos(elevation) * torch.sin(azimuth), distance * torch.sin(elevation),
                        -distance * torch.cos(elevation) * torch.cos(azimuth)]).transpose(1, 0)
