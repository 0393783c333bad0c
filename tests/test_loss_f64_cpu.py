"""Host side of the float64 loss kernels (DESIGN.md §10), without a GPU: the `umr_*_f64` symbols are exported, their
workspace queries follow the documented formulas, bad arguments are refused before anything reaches the device, and the
dtype rule of ops.py picks float64 exactly when a floating-point input is float64."""
import ctypes

import pytest
import torch

from umr_b200 import _lib, ops

UMR_ERR_BAD_ARG, UMR_ERR_TOO_LARGE = -2, -3
F64_SYMBOLS = [n for n in _lib.EXPORTS if n.endswith("_f64") and not n.startswith("umr_raster")]
FAKE = ctypes.c_void_p(256)   # a non-null pointer that is never dereferenced: validation fails before any launch


def test_symbols_exported():
    assert len(F64_SYMBOLS) == 27
    lib = _lib.load()
    for name in F64_SYMBOLS:
        assert getattr(lib, name) is not None
    assert lib.umr_version() == 204


def _cdiv(a, b):
    return (a + b - 1) // b


@pytest.mark.parametrize("B,N", [(1, 1), (3, 2048), (3, 2049), (7, 600 * 600)])
def test_workspace_formulas(B, N):
    lib = _lib.load()
    assert lib.umr_iou_workspace_bytes_f64(B, N) == 16 * B * _cdiv(N, 2048)
    assert lib.umr_masked_l1_workspace_bytes_f64(B, N) == 8 * B * _cdiv(N, 2048)
    assert lib.umr_loss_head_workspace_bytes_f64(B, N) == 24 * B * _cdiv(N, 2048)
    assert lib.umr_texcycle_workspace_bytes_f64(B, N) == 8 * _cdiv(B * N, 256)
    assert lib.umr_laplacian_workspace_bytes_f64(B, N) == 8 * B * _cdiv(N, 256)
    assert lib.umr_flatten_forward_workspace_bytes_f64(B, N) == 8 * B * _cdiv(N, 128)
    assert lib.umr_flatten_backward_workspace_bytes_f64(B, N) == 96 * B * N
    assert lib.umr_corr_chamfer_workspace_bytes_f64(B, N) == 24 * B * N
    for q in ("iou", "masked_l1", "loss_head"):
        assert getattr(lib, "umr_%s_workspace_bytes_f64" % q)(0, N) == 0
        assert getattr(lib, "umr_%s_workspace_bytes_f64" % q)(B, 0) == 0


def test_bad_arguments_refused():
    lib = _lib.load()
    launches = lib.umr_launch_count()
    N0 = ctypes.c_void_p(0)
    assert lib.umr_bilinear_sample_forward_f64(N0, FAKE, FAKE, 1, 3, 4, 4, 10, None) == UMR_ERR_BAD_ARG
    assert lib.umr_bilinear_sample_forward_f64(FAKE, FAKE, FAKE, 0, 3, 4, 4, 10, None) == UMR_ERR_BAD_ARG
    assert lib.umr_bilinear_sample_forward_f64(FAKE, FAKE, FAKE, 65536, 3, 4, 4, 10, None) == UMR_ERR_TOO_LARGE
    assert lib.umr_bilinear_sample_cells_f64(FAKE, FAKE, 2, 65536, 65536, 10, None) == UMR_ERR_TOO_LARGE
    # an image gradient without its cell table
    assert lib.umr_bilinear_sample_backward_f64(FAKE, FAKE, FAKE, FAKE, FAKE, 1, 3, 4, 4, 10, N0, N0, None) == UMR_ERR_BAD_ARG
    assert lib.umr_iou_forward_f64(FAKE, 16, FAKE, FAKE, FAKE, FAKE, 1, 16, N0, None) == UMR_ERR_BAD_ARG   # no workspace
    assert lib.umr_iou_forward_f64(FAKE, 16, FAKE, FAKE, FAKE, FAKE, 65536, 16, FAKE, None) == UMR_ERR_TOO_LARGE
    assert lib.umr_iou_backward_f64(FAKE, FAKE, FAKE, FAKE, FAKE, 1, 0, None) == UMR_ERR_BAD_ARG
    assert lib.umr_masked_l1_forward_f64(FAKE, 0, FAKE, 0, FAKE, FAKE, FAKE, 1, 3, 0, FAKE, None) == UMR_ERR_BAD_ARG
    assert lib.umr_masked_l1_backward_f64(FAKE, 0, FAKE, 0, FAKE, FAKE, N0, FAKE, FAKE, 1, 3, 5, None) == UMR_ERR_BAD_ARG
    assert lib.umr_loss_head_forward_f64(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, 65536, 4, 1.0, 1.0, FAKE, None) == UMR_ERR_TOO_LARGE
    assert lib.umr_loss_head_backward_f64(FAKE, FAKE, FAKE, N0, FAKE, FAKE, 1, 4, 1.0, 1.0, None) == UMR_ERR_BAD_ARG
    assert lib.umr_chamfer_forward_f64(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, 1, 0, 3, 3, None) == UMR_ERR_BAD_ARG
    # a distance gradient without its nearest indices
    assert lib.umr_chamfer_backward_f64(FAKE, FAKE, N0, FAKE, FAKE, N0, FAKE, FAKE, 1, 4, 3, 3, None) == UMR_ERR_BAD_ARG
    assert lib.umr_texcycle_forward_f64(FAKE, FAKE, FAKE, FAKE, FAKE, 1, 4, 9, 0, FAKE, None) == UMR_ERR_BAD_ARG   # P = 0
    assert lib.umr_texcycle_backward_f64(FAKE, FAKE, FAKE, FAKE, FAKE, 65536, 4, 9, None) == UMR_ERR_TOO_LARGE
    assert lib.umr_laplacian_forward_f64(FAKE, FAKE, FAKE, N0, FAKE, FAKE, 1, 5, FAKE, None) == UMR_ERR_BAD_ARG
    assert lib.umr_laplacian_backward_f64(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, 65536, 5, None) == UMR_ERR_TOO_LARGE
    assert lib.umr_flatten_forward_f64(FAKE, FAKE, FAKE, 1, 5, 0, 1e-6, FAKE, None) == UMR_ERR_BAD_ARG
    assert lib.umr_flatten_backward_f64(FAKE, FAKE, N0, FAKE, FAKE, FAKE, 1, 5, 3, 1e-6, FAKE, None) == UMR_ERR_BAD_ARG
    tp = (ctypes.c_void_p * 4)(256, 256, 256, 256)
    tc = (ctypes.c_int32 * 4)(3, 3, 3, 3)
    wt = (ctypes.c_double * 4)(1, 1, 0, 0)
    bad_ends = (ctypes.c_int32 * 4)(2, 1, 3, 4)   # not ascending
    ends = (ctypes.c_int32 * 4)(1, 2, 3, 4)
    assert lib.umr_corr_chamfer_forward_f64(FAKE, 0, FAKE, FAKE, tp, tc, bad_ends, wt, FAKE, FAKE, FAKE, 2, 4,
                                            None) == UMR_ERR_BAD_ARG
    assert lib.umr_corr_chamfer_forward_f64(FAKE, 0, FAKE, FAKE, tp, tc, ends, wt, FAKE, FAKE, FAKE, 2, 5,
                                            None) == UMR_ERR_BAD_ARG   # the parts do not cover NS
    # a vertex gradient without its transposed selection table
    assert lib.umr_corr_chamfer_backward_f64(FAKE, 0, FAKE, FAKE, tp, tc, ends, wt, FAKE, FAKE, FAKE, N0, FAKE, N0, 2, 4, 9,
                                             N0, N0, FAKE, None) == UMR_ERR_BAD_ARG
    assert lib.umr_corr_chamfer_backward_f64(FAKE, 0, FAKE, FAKE, tp, tc, ends, wt, FAKE, FAKE, FAKE, N0, N0, FAKE, 65536, 4,
                                             9, N0, N0, N0, None) == UMR_ERR_TOO_LARGE
    assert lib.umr_launch_count() == launches   # a refused call launches nothing


def test_misaligned_vector_pointers_refused():
    """The sampler's flow / grad_flow and TexCycle's flow / prob / grad_flow are read as (x, y) vector pairs: a pointer
    that is not a multiple of 2 * sizeof(element) is refused with UMR_ERR_BAD_ARG in every precision, before any launch
    (ops.py copies such an input to aligned storage first: test_dispatch_cpu.py::test_odd_offset_pairs_reach_the_library_aligned)."""
    lib = _lib.load()
    launches = lib.umr_launch_count()
    N0 = ctypes.c_void_p(0)
    for suffix, step in (("", 4), ("_deterministic", 4), ("_f64", 8)):
        odd = ctypes.c_void_p(FAKE.value + step)   # aligned to the element, not to the pair
        fwd = getattr(lib, "umr_bilinear_sample_forward" + ("_f64" if suffix == "_f64" else ""))
        assert fwd(FAKE, odd, FAKE, 1, 3, 4, 4, 10, None) == UMR_ERR_BAD_ARG, suffix
        cells = getattr(lib, "umr_bilinear_sample_cells" + ("_f64" if suffix == "_f64" else ""))
        assert cells(odd, FAKE, 1, 4, 4, 10, None) == UMR_ERR_BAD_ARG, suffix
        bwd = getattr(lib, "umr_bilinear_sample_backward" + suffix)
        table = () if suffix == "" else (N0, N0)
        for flow, gflow in ((odd, FAKE), (FAKE, odd)):
            assert bwd(FAKE, flow, FAKE, gflow, N0, 1, 3, 4, 4, 10, *table, None) == UMR_ERR_BAD_ARG, suffix
        tfwd = getattr(lib, "umr_texcycle_forward" + suffix)
        ws = () if suffix == "" else (FAKE,)
        for flow, prob in ((odd, FAKE), (FAKE, odd)):
            assert tfwd(flow, prob, N0, FAKE, FAKE, 2, 4, 9, 0, *ws, None) == UMR_ERR_BAD_ARG, suffix
        if suffix != "_deterministic":   # the deterministic mode uses the default TexCycle backward
            tbwd = getattr(lib, "umr_texcycle_backward" + suffix)
            for flow, prob, gflow in ((odd, FAKE, FAKE), (FAKE, odd, FAKE), (FAKE, FAKE, odd)):
                assert tbwd(flow, prob, FAKE, FAKE, gflow, 2, 4, 9, None) == UMR_ERR_BAD_ARG, suffix
    assert lib.umr_launch_count() == launches


def test_texcycle_size_limit_in_every_precision():
    """B * F is the kernels' int32 (image, face) index: every TexCycle entry point refuses B * F > INT32_MAX."""
    lib = _lib.load()
    N0 = ctypes.c_void_p(0)
    B, F = 65535, 32769   # B * F = 2^31 + 32767
    for suffix in ("", "_deterministic", "_f64"):
        ws = () if suffix == "" else (FAKE,)
        assert getattr(lib, "umr_texcycle_forward" + suffix)(FAKE, FAKE, N0, FAKE, FAKE, B, F, 9, 0, *ws,
                                                             None) == UMR_ERR_TOO_LARGE, suffix
    for suffix in ("", "_f64"):
        assert getattr(lib, "umr_texcycle_backward" + suffix)(FAKE, FAKE, FAKE, FAKE, FAKE, B, F, 9,
                                                              None) == UMR_ERR_TOO_LARGE, suffix


def test_dtype_rule():
    f32, f64, f16 = torch.zeros(1), torch.zeros(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float16)
    assert ops._is_f64(f32, f64) and ops._is_f64(f64) and ops._is_f64(None, f64)
    assert not ops._is_f64(f32, f16) and not ops._is_f64(f32, None) and not ops._is_f64()
