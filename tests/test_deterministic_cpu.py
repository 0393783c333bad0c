"""Host-side contract of the rasteriser's deterministic mode (no GPU): the three entry points are exported, the default
workspace size is unchanged, the deterministic workspace follows its formula, and the fixed-point p2f accumulators cannot
overflow for any raster the kernels can launch (DESIGN.md §3)."""
import math
import os
import re

import pytest

from umr_b200 import _lib

_SRC = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "umr_b200", "csrc", "raster.cu")).read()


def _const(name):   # the constants as raster.cu defines them, so this bound follows any change there
    return int(re.search(r"constexpr int %s = (\d+);" % name, _SRC).group(1))


P2F_LIMBS, P2F_LIMB_BITS, P2F_FRAC_BITS = _const("P2F_LIMBS"), _const("P2F_LIMB_BITS"), _const("P2F_FRAC_BITS")
P2F_DET_WORDS = 3 * P2F_LIMBS + 1
MAX_RASTER = 65535 * 16                                # DET_MAX_RASTER: gridDim.y limit of the 16x16-tile forward


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _a(x):
    return (x + 255) // 256 * 256


def test_symbols_exported(lib):
    for name in ("umr_raster_workspace_bytes_deterministic", "umr_raster_forward_deterministic",
                 "umr_raster_backward_deterministic"):
        assert getattr(lib, name) is not None


@pytest.mark.parametrize("B,F,isz,aa", [(1, 1, 64, 1), (16, 1280, 256, 1), (3, 20480, 37, 0), (2, 65537, 64, 1),
                                        (1, 1 << 24, 256, 1)])
def test_workspace_formula(lib, B, F, isz, aa):
    base = lib.umr_raster_workspace_bytes(B, F, isz, aa)
    assert lib.umr_raster_workspace_bytes_deterministic(B, F, isz, aa) == base + _a(B * F * P2F_DET_WORDS * 8)
    assert lib.umr_raster_workspace_bytes_deterministic(0, F, isz, aa) == 0


def test_default_workspace_unchanged(lib):
    assert lib.umr_raster_workspace_bytes(16, 1280, 256, 1) == 5902592   # test_raster_large_faces_cpu.NARROW_WORKSPACE


@pytest.mark.parametrize("S", [2, 64, 512, 4096, 1 << 16, 1 << 18, MAX_RASTER])
def test_p2f_limbs_cannot_overflow(S):
    """A (warp, face) partial |v| <= 32 (32 pixel terms of magnitude <= 1) becomes round(|v| * 2^96) < 2^102, which the
    limbs cover; every limb of a contribution is < 2^26, and a face gets at most one contribution per 8x4 pixel block of the
    raster (one per warp of every 16x16 tile), so each int64 limb word stays below 2^63 in magnitude."""
    assert 32 * 2 ** P2F_FRAC_BITS < 2 ** (P2F_LIMBS * P2F_LIMB_BITS)
    assert P2F_LIMB_BITS >= 24   # a 24-bit mantissa touches at most two limbs
    # red_fixed: |v| = m * 2^s with m < 2^24.  s is capped at LIMBS * LIMB_BITS - 24 (so m << s fits the limbs); every finite
    # |v| <= 32 (exponent field <= 132) stays below that cap, and s <= -32 rounds to 0 (|v| < 2^-(FRAC_BITS + 8))
    s_max_finite = 132 - (150 - P2F_FRAC_BITS)
    assert s_max_finite <= P2F_LIMBS * P2F_LIMB_BITS - 24
    assert 2 ** 24 * 2.0 ** (-32) < 0.5
    tiles = math.ceil(S / 16) ** 2
    contributions = tiles * 8
    assert contributions * (2 ** P2F_LIMB_BITS - 1) < 2 ** 63
