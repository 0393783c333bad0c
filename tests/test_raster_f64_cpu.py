"""What the float64 rasteriser rests on, without a GPU:

* oracle B's double instantiation -- the yardstick of tests/test_raster_f64_gpu.py -- is bit-exact with oracle A's (the
  reference's own device code compiled for the host with scalar_t = double) in every mode combination
  (test_raster_modes_cpu.py pins the float instantiation only);
* the host logic of the dtype rule: CPU tensors still raise, `Mesh` and the generic vertex chain keep float64;
* the arithmetic of the fixed-point p2f accumulator of csrc/raster_f64.cu (rounding to 2^-128, 26-bit limbs in wrapping
  64-bit words, carry propagation, one rounding on read-back), restated in Python integers, against exact rational sums."""
import re
import struct
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest
import torch

import softras
from umr_b200 import raster, synth
from umr_b200 import soft_renderer as sr
from umr_b200.nnutils import geom_utils
from util import scene

SOFT = dict(sigma_val=1e-4, dist_eps=1e-4, gamma_val=1e-3)
COMBOS = [(d, a, t, r, fb) for d in ("hard", "barycentric", "euclidean") for a in ("hard", "sum", "prod")
          for t in ("surface", "vertex") for r in ("softmax", "hard") for fb in (True, False)]
assert len(COMBOS) == 72


@pytest.mark.skipif(not softras.have_oracle_a(), reason="oracle A (reference on host) not built")
@pytest.mark.parametrize("dist,alpha,textype,rgb,fill_back", COMBOS)
def test_oracle_b_f64_bit_exact_with_reference_on_host(dist, alpha, textype, rgb, fill_back):
    S = 33
    fv, tex = scene(2, 2, 1, seed=70)    # 320 faces; T2 = 1: the reference's texel gradient is defined there only
    rng = np.random.default_rng(71)
    if textype == "vertex":
        tex = rng.uniform(0, 1, size=(2, fv.shape[1], 3, 3))
    fv = fv.astype(np.float64) + rng.normal(size=fv.shape) * 1e-9   # genuine doubles
    kw = dict(SOFT, dist_func=dist, aggr_func_alpha=alpha, texture_type=textype, aggr_func_rgb=rgb, fill_back=fill_back,
              background_color=(0.25, 0.5, 0.75))
    res = {}
    for impl in "AB":
        cfg = softras.RasterCfg(S, **kw)
        fwd = softras.forward(fv, tex, cfg, impl=impl, nthreads=1, dtype=np.float64)
        g = np.random.default_rng(S).normal(size=fwd["soft_colors"].shape)
        gf, gt = softras.backward(fwd, g, cfg, impl=impl, nthreads=1)
        res[impl] = dict(soft_colors=fwd["soft_colors"], aggrs_info=fwd["aggrs_info"], p2f_info=fwd["p2f_info"],
                         grad_faces=gf, grad_textures=gt)
    for k in res["A"]:
        assert res["B"][k].dtype == np.float64 and np.array_equal(res["A"][k], res["B"][k]), k
    assert (res["B"]["aggrs_info"][:, 1] != res["B"]["aggrs_info"][:, 1, :1, :1]).any()
    assert np.abs(res["B"]["grad_faces"]).max() > 0 or (rgb == "hard" and dist == "hard")


# ---------------------------------------------------------------------------------------------------------------------
# host logic
# ---------------------------------------------------------------------------------------------------------------------
def test_cpu_float64_tensors_still_raise():
    with pytest.raises(TypeError, match="Rasterize module supports only cuda Tensors"):
        raster.soft_rasterize(torch.zeros(1, 2, 3, 3, dtype=torch.float64), torch.zeros(1, 2, 1, 3, dtype=torch.float64), 8)


def _mesh(dtype, texture_type="surface", textures=False):
    v, f = synth.icosphere(1)
    verts = torch.from_numpy(synth.bird_like(v, np.random.default_rng(0), 2)).to(dtype)
    faces = torch.from_numpy(np.repeat(f.astype(np.int32)[None], 2, 0))
    tex = torch.rand(2, f.shape[0], 4, 3, generator=torch.Generator().manual_seed(3)).to(dtype) if textures else None
    return sr.Mesh(verts, faces, tex, texture_res=2, texture_type=texture_type)


@pytest.mark.parametrize("texture_type", ["surface", "vertex"])
def test_mesh_keeps_float64(texture_type):
    m = _mesh(torch.float64, texture_type)
    assert m.vertices.dtype == m.textures.dtype == m.face_vertices.dtype == m.face_textures.dtype == torch.float64
    assert m.vertex_normals.dtype == m.surface_normals.dtype == torch.float64
    m32 = _mesh(torch.float32, texture_type)
    assert m32.textures.dtype == m32.face_vertices.dtype == torch.float32
    assert _mesh(torch.float16, texture_type).textures.dtype == torch.float32   # as before: only float64 is followed


@pytest.mark.parametrize("camera", [dict(camera_mode="look_at", perspective=False, viewing_scale=0.9, eye=[0.2, 0.1, -2.7]),
                                    dict(camera_mode="look_at", perspective=True),
                                    dict(camera_mode="look", perspective=True, eye=[0.0, 0.0, -3.0])])
@pytest.mark.parametrize("light_mode", ["surface", "vertex"])
def test_generic_vertex_chain_carries_the_dtype(camera, light_mode):
    """Lighting and Transform on CPU tensors: float64 in, float64 out, and equal to the float32 chain to float32 accuracy
    (so the float64 constants are the same constants)."""
    out = {}
    for dt in (torch.float64, torch.float32):
        mesh = _mesh(dt, light_mode, textures=light_mode == "surface")
        mesh = sr.Transform(**camera)(sr.Lighting(light_mode=light_mode, color_ambient=(0.3, 0.6, 0.9),
                                                  directions=(0.3, 0.8, -0.5))(mesh))
        assert mesh.face_vertices.dtype == mesh.face_textures.dtype == dt
        out[dt] = (mesh.face_vertices, mesh.face_textures)
    for a, b in zip(out[torch.float64], out[torch.float32]):
        assert torch.allclose(a, b.double(), rtol=1e-4, atol=1e-5)
        assert not torch.equal(a, b.double())   # computed in double, not widened afterwards
    cams = torch.from_numpy(synth.cameras(np.random.default_rng(1), 2)).double()
    assert geom_utils.orthographic_proj_withz(_mesh(torch.float64).vertices, cams, offset_z=5.).dtype == torch.float64


# ---------------------------------------------------------------------------------------------------------------------
# fixed-point p2f accumulator
# ---------------------------------------------------------------------------------------------------------------------
def _constants():
    src = (Path(raster.__file__).parent / "csrc" / "raster_f64.cu").read_text()
    return {k: int(re.search(r"constexpr int %s = (\d+);" % k, src).group(1)) for k in ("P2F_LIMBS", "P2F_LIMB_BITS", "P2F_FRAC_BITS")}


C = _constants()
LIMBS, BITS, FRAC = C["P2F_LIMBS"], C["P2F_LIMB_BITS"], C["P2F_FRAC_BITS"]
M64 = (1 << 64) - 1


def red_fixed(words, v):
    """red_fixed of raster_f64.cu: round(|v| * 2^FRAC) half away from zero, limbs added into wrapping uint64 words."""
    u = struct.unpack("<Q", struct.pack("<d", v))[0]
    e = (u >> 52) & 0x7ff
    s = (e if e else 1) - (1075 - FRAC)
    assert e != 0x7ff and s <= LIMBS * BITS - 53
    m = (u & ((1 << 52) - 1)) | ((1 << 52) if e else 0)
    up = s
    if s < 0:
        if s <= -54:
            return
        m, up = (m + (1 << (-s - 1))) >> (-s), 0
    for k in range(LIMBS):
        d = k * BITS - up                      # limb k = bits [d, d + BITS) of the 64-bit m
        if d >= 0:
            limb = (m >> d) if d < 64 else 0
        else:
            limb = ((m << -d) & M64) if -d < BITS else 0
        limb &= (1 << BITS) - 1
        words[k] = (words[k] + (-limb if u >> 63 else limb)) & M64


def fixed_value(words):
    """fixed_value of raster_f64.cu, step for step: signed words, upward carries, magnitude, the leading four limbs with a
    sticky bit, 64 leading bits rounded to nearest even."""
    limbs, carry = [], 0
    for k in range(LIMBS):
        t = (words[k] - (1 << 64) if words[k] >> 63 else words[k]) + carry
        if k < LIMBS - 1:
            carry = t >> BITS
            limbs.append(t - (carry << BITS))
        else:
            limbs.append(t)
    neg = limbs[-1] < 0
    if neg:
        borrow = 0
        for k in range(LIMBS):
            t = -limbs[k] - borrow
            if k < LIMBS - 1:
                borrow = 1 if t < 0 else 0
                t += borrow << BITS
            limbs[k] = t
    h = LIMBS - 1
    while h > 0 and limbs[h] == 0:
        h -= 1
    m, sticky = 0, False
    for k in range(LIMBS - 1, -1, -1):
        if h - 4 < k <= h:
            m = (m << BITS) | limbs[k]
        elif k <= h - 4 and limbs[k]:
            sticky = True
    assert m < 1 << 127
    expo = (h - 3 if h > 3 else 0) * BITS - FRAC
    if m >> 64:
        sh = (m >> 64).bit_length()
        sticky |= (m & ((1 << sh) - 1)) != 0
        m >>= sh
        expo += sh
    if sticky:
        m |= 1
    # __ull2double_rn: 64 bits to 53, nearest even
    if m.bit_length() > 53:
        drop = m.bit_length() - 53
        half, rest = 1 << (drop - 1), m & ((1 << drop) - 1)
        m >>= drop
        if rest > half or (rest == half and (m & 1)):
            m += 1
        expo += drop
    v = float(np.ldexp(float(m), expo))
    return -v if neg else v


@pytest.mark.parametrize("seed", range(6))
def test_fixed_point_accumulator_against_exact_sums(seed):
    """Random bounded partials (|v| <= 32, magnitudes from 2^-140 to 32, both signs) in a random order: the words do not
    depend on the order, and the read-back is the exact sum of the rounded partials rounded once, which lies within
    n * 2^-(FRAC + 1) of the exact sum of the partials themselves."""
    rng = np.random.default_rng(seed)
    n = 4000
    vals = rng.uniform(-32, 32, size=n) * np.exp2(-rng.integers(0, 140, size=n).astype(np.float64) * (rng.random(n) < 0.7))
    if seed % 2:
        vals = np.abs(vals)      # the weight sum: all terms non-negative
    if seed == 4:
        vals *= 2.0 ** -60       # a sum near the clamp_min(1e-12) of the finalize
    vals[:4] = [32.0, -32.0 if seed % 2 == 0 else 32.0, 5e-324, 2.0 ** -129]
    words, words_perm = [0] * LIMBS, [0] * LIMBS
    for v in vals:
        red_fixed(words, float(v))
    for v in rng.permutation(vals):
        red_fixed(words_perm, float(v))
    assert words == words_perm
    exact_rounded = sum(int(round_half_away(Fraction(float(v)) * (1 << FRAC))) for v in vals)
    got = fixed_value(words)
    want = Fraction(exact_rounded, 1 << FRAC)
    assert got == nearest_double(want)
    exact = sum(Fraction(float(v)) for v in vals)
    assert abs(Fraction(got) - exact) <= n * Fraction(1, 1 << (FRAC + 1)) + abs(exact) * Fraction(1, 1 << 53)


def round_half_away(x):
    f = abs(x)
    r = int(f) + (1 if f - int(f) >= Fraction(1, 2) else 0)
    return r if x >= 0 else -r


def nearest_double(x):
    """Fraction -> the nearest double, ties to even (float(Fraction) is correctly rounded)."""
    return float(x)


def test_accumulator_bound_stated_in_the_source():
    """>= 100 fractional bits; limbs cover a partial of magnitude 32; a word cannot overflow within 2^36 partials."""
    assert FRAC >= 100 and LIMBS * BITS >= FRAC + 6 and BITS + 36 <= 62
