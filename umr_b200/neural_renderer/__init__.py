"""`neural_renderer.Renderer` (NMR) for UMR's visuals and its `MultiTextureLoss(renderer="nmr")`, on the H100 kernels.

`umr_b200.compat.install()` registers this package under the import name `neural_renderer`, so the reference's own
`nnutils/nmr_pytorch.py` drives it unmodified (`NeuralRenderer`, :89-128, built at train_s2.py:111-113,
train_s1.py:112-115 and demo.py:64-67).

Supported configuration -- UMR's: `camera_mode='look_at'`, `perspective=False`, eye (0, 0, e) with e < 0 (there look_at
is the exact translation z - e).  Anything else raises NotImplementedError naming the setting.  Only the textures get a
gradient: NMR's approximate vertex gradient is not built, and every UMR call site renders detached geometry.

Render contract (DESIGN.md §7; oracle/nmr.py restates it).  fp32, one rounding per operation; S = 2*is with
anti-aliasing, else is.
1. Face set: with fill_back, faces F..2F-1 are faces 0..F-1 with the vertex order reversed; their texture is
   textures.permute(0,1,4,3,2,5), i.e. a back copy reads texel (t2,t1,t0) of the original cube.
2. Light, per face copy, from the input vertices before look_at: n = normalize(cross(v0-v1, v2-v1), eps=1e-5),
   light = Ia*ca + Id*(cd*relu(n.d)) (d not normalised; a term with zero intensity is not added).  A reversed copy's
   normal is exactly -n.  The texel is multiplied by the light before blending.
3. Z-buffer: pixel centres xp = (2*xi+1-S)/S; face vertices in pixel units 0.5*(x*S+S-1).  A face copy is skipped when
   it is back-facing, (y2-y0)(x1-x0) < (y1-y0)(x2-x0) in NDC; when the pixel centre fails one of the three edge tests
   (strict '<'); or when zp <= near, zp >= far or zp is NaN.  w = face_inv . (xi, yi, 1) in pixel units, each
   component clamped to [0, 1], renormalised by its sum; zp = 1/(w0/z0 + w1/z1 + w2/z2).  The winner is the
   lexicographic minimum of (zp, face copy index).
4. Texture: tif_k = clamp(w_k*(T-1)*(zp/z_k), 0, T-1-1e-3); the 8 corners pn = 0..7, bit k of pn choosing floor or
   floor+1 on axis k, weight = product of (1-frac) or frac, texel ((i0*T)+i1)*T+i2; z_k is the winner's own depth.
5. Output: background pixels take background_color, alpha = (face >= 0), depth = far where no face wins; the planes
   are flipped vertically, then 2x2 average-pooled (window summed row-major in the flipped image, divided by 4).
6. Texture gradient: light * w_pn * grad_rgb at the 8 texels of every covered raster pixel (back copies on the
   transposed texel), through the adjoint of the pool and the flip.
Equivalence of this contract to the upstream package is not verified (its source is not available offline).
"""
from .renderer import Renderer

__all__ = ["Renderer"]
