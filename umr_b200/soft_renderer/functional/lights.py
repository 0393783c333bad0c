"""Lighting helpers (references: functional/ambient_lighting.py:7-18, directional_lighting.py:7-28)."""
import torch
import torch.nn.functional as F


def _color(c, light):
    """A colour / direction constant as a [1|B,3] tensor: float64 beside a float64 light buffer, float32 otherwise."""
    dtype = torch.float64 if light.dtype == torch.float64 else torch.float32
    t = torch.as_tensor(c, dtype=dtype, device=light.device)
    return t[None, :] if t.dim() == 1 else t


def ambient_lighting(light, light_intensity=0.5, light_color=(1, 1, 1)):
    """light [B,N,3] += intensity * colour (in place, like the reference)."""
    light += light_intensity * _color(light_color, light)[:, None, :]
    return light


def directional_lighting(light, normals, light_intensity=0.5, light_color=(1, 1, 1), light_direction=(0, 1, 0)):
    """light [B,N,3] += intensity * colour * relu(n . d)."""
    color = _color(light_color, light)
    direction = _color(light_direction, light)
    cosine = F.relu(torch.sum(normals * direction[:, None, :], dim=2))
    light += light_intensity * (color[:, None, :] * cosine[:, :, None])
    return light
