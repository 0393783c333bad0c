"""Host-side contract of meshes above 65535 faces (no GPU): workspace sizes below the limit are unchanged, the wide
workspace follows its documented formula, and the face limit is enforced before any device work."""
import ctypes

import pytest

from umr_b200 import _lib

MAX_FACES = 1 << 24   # UMR_RASTER_MAX_FACES

# umr_raster_workspace_bytes / umr_raster_pair_buffer_bytes of the build before meshes above 65535 faces were accepted
NARROW_WORKSPACE = [((1, 1, 64, 1), 1536), ((16, 1280, 256, 1), 5902592), ((16, 5120, 256, 1), 23597312),
                    ((4, 65535, 32, 1), 42467328), ((2, 65535, 1024, 1), 289411072), ((3, 20480, 37, 0), 9953792),
                    ((7, 2049, 500, 1), 9646336), ((1, 65535, 2048, 1), 547365120)]
PAIR_BUFFER = [((16, 256, 1, 1000), 1672448), ((1, 37, 0, 7), 12800), ((4, 1024, 1, 123456), 190647808)]


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


@pytest.mark.parametrize("args,want", NARROW_WORKSPACE)
def test_narrow_workspace_unchanged(lib, args, want):
    assert lib.umr_raster_workspace_bytes(*args) == want


@pytest.mark.parametrize("args,want", PAIR_BUFFER)
def test_pair_buffer_unchanged(lib, args, want):
    assert lib.umr_raster_pair_buffer_bytes(*args) == want


def _a(x):
    return (x + 255) // 256 * 256


@pytest.mark.parametrize("B,F,isz,aa", [(1, 65536, 32, 1), (16, 327680, 256, 1), (2, 327680, 1024, 1),
                                        (1, MAX_FACES, 256, 1)])
def test_wide_workspace_formula(lib, B, F, isz, aa):
    """DESIGN.md §3: face records, cull boxes and p2f accumulators as below the limit, the union boxes, a {count, offset}
    pair per 64-pixel bin plus the pool cursor, and a pool of 8 u32 entries per face -- 192 bytes per face, no term in
    bins x F."""
    S = isz * (2 if aa else 1)
    n, nbin = B * F, B * ((S + 63) // 64) ** 2
    want = _a(n * 128) + _a(n * 16) + _a(n * 16) + _a(B * 16) + _a(nbin * 8 + 8) + _a(min(8 * n, 0xfffffff0) * 4)
    assert lib.umr_raster_workspace_bytes(B, F, isz, aa) == want


def _forward_rc(lib, F):
    p = _lib.UmrRasterParams()
    p.batch_size, p.num_faces, p.texture_size, p.image_size = 1, F, 1, 32
    p.func_id_dist, p.func_id_rgb, p.func_id_alpha = 2, 1, 2
    null = ctypes.c_void_p(0)
    return lib.umr_raster_forward(null, null, null, null, null, null, ctypes.byref(p), null, null)


def test_face_limit(lib):
    """F = 2^24 passes the size checks (and fails on the null buffers); one more face is refused as too large, and the
    Python layer raises on that code."""
    assert _forward_rc(lib, MAX_FACES) == -2          # UMR_ERR_BAD_ARG: past the limit check
    assert _forward_rc(lib, 65536) == -2
    assert _forward_rc(lib, MAX_FACES + 1) == -3      # UMR_ERR_TOO_LARGE
    with pytest.raises(RuntimeError):
        _lib.check(_forward_rc(lib, MAX_FACES + 1), "umr_raster_forward")
