"""neural_renderer's camera functions (DESIGN.md §15): a few torch ops on [B,V,3], gradients through autograd.

SoftRas copied NMR's camera code, so `look_at` and `get_points_from_angles` are soft_renderer's own definitions, and
`look` is soft_renderer's with NMR's `up=None` default.  `perspective` and `projection` are NMR's, which differ:
`perspective` takes the tangent of a float32 angle tensor, and `projection` takes K, R and t and flips v.
"""
import math

import torch

from ..soft_renderer.functional import geometry
from ..soft_renderer.functional.geometry import get_points_from_angles, look_at

__all__ = ["look_at", "look", "perspective", "projection", "get_points_from_angles"]


def look(vertices, eye, direction=(0, 1, 0), up=None):
    """Camera at `eye` looking along `direction`; `up` defaults to (0, 1, 0)."""
    return geometry.look(vertices, eye, direction, (0, 1, 0) if up is None else up)


def perspective(vertices, angle=30.):
    """Pinhole projection with half field-of-view `angle` degrees: (x / z) / w, (y / z) / w and z, where w is the
    tangent of the angle in radians held as a float32 tensor (soft_renderer's `perspective` takes a double tangent)."""
    if vertices.dim() != 3:
        raise ValueError("vertices Tensor should have 3 dimensions")
    radians = angle / 180 * math.pi            # in double for a number, then rounded to float32
    w = torch.tan(torch.as_tensor(radians, dtype=torch.float32, device=vertices.device).reshape(-1, 1))
    depth = vertices[:, :, 2]
    return torch.stack((vertices[:, :, 0] / depth / w, vertices[:, :, 1] / depth / w, depth), dim=2)


def projection(vertices, K, R, t, dist_coeffs, orig_size, eps=1e-9):
    """Calibrated pinhole projection: world vertices [B,V,3] -> (u, v, z) with u, v in [-1, 1] and z the camera depth.

    R [B,3,3] and t [B,1,3] take world to camera coordinates; the image-plane point (x/(z+eps), y/(z+eps)) is distorted
    by dist_coeffs [B,5] = (k1, k2, p1, p2, k3) in OpenCV's model, with the radial factor a polynomial in the radius
    itself (rho^2, rho^4, rho^6 of rho = sqrt(x^2 + y^2)); K [B,3,3] maps it to pixels of an orig_size-wide image, v is
    flipped (orig_size - v) so that the first image row is at the top, and both are scaled to [-1, 1]."""
    cam = torch.matmul(vertices, R.transpose(1, 2)) + t
    depth = cam[:, :, 2]
    xn = cam[:, :, 0] / (depth + eps)
    yn = cam[:, :, 1] / (depth + eps)
    k1, k2, p1, p2, k3 = (dist_coeffs[:, i, None] for i in range(5))
    rho = torch.sqrt(xn ** 2 + yn ** 2)
    radial = 1 + k1 * rho ** 2 + k2 * rho ** 4 + k3 * rho ** 6
    xd = xn * radial + 2 * p1 * xn * yn + p2 * (rho ** 2 + 2 * xn ** 2)
    yd = yn * radial + p1 * (rho ** 2 + 2 * yn ** 2) + 2 * p2 * xn * yn
    pix = torch.matmul(torch.stack((xd, yd, torch.ones_like(depth)), dim=-1), K.transpose(1, 2))
    half = orig_size / 2.
    ndc = [(c - half) * 2 / orig_size for c in (pix[:, :, 0], orig_size - pix[:, :, 1])]
    return torch.stack((ndc[0], ndc[1], depth), dim=-1)
