"""Return codes of the float32 loss, mesh-op, vertex, CorrLossChamfer and all-reduce C entry points for inputs they refuse
(no GPU).

Every refusal comes before any device work: the call returns its code, launches no kernel (umr_launch_count() does not
move) and runs no memset.  Without a GPU a memset or launch that ran first would come back as a CUDA error instead of the
refusal.  The fake buffer addresses are never touched."""
import ctypes

import pytest

from umr_b200 import _lib

UNSUPPORTED, BAD_ARG, TOO_LARGE = -1, -2, -3

F = 256          # non-NULL, 256-byte aligned
N0 = None        # NULL
ODD = 256 + 4    # float-aligned, not float2-aligned

_TP = (ctypes.c_void_p * 4)(F, F, F, F)
_TC = (ctypes.c_int32 * 4)(3, 3, 3, 3)
_WT = (ctypes.c_float * 4)(1, 1, 0, 0)
_ENDS = (ctypes.c_int32 * 4)(1, 2, 3, 4)
_BAD_ENDS = (ctypes.c_int32 * 4)(2, 1, 3, 4)   # not ascending
_MAPS = (ctypes.c_void_p * 4)(F, F, F, F)
_MAP_BS = (ctypes.c_int64 * 4)(16, 16, 16, 16)


def _proj(B=2, V=5, F_=4, H=1):
    p = _lib.UmrProjectParams()
    p.batch_size, p.num_vertices, p.num_faces, p.num_hypotheses = B, V, F_, H
    return ctypes.byref(p)


def _corr(ends=_ENDS):
    return (F, 0, F, F, _TP, _TC, ends, _WT)


# (entry point, arguments without the trailing stream, expected code)
CASES = [
    # sampler; C past 4 is refused before the launch (forward) and before zeroing grad_image (backward)
    ("umr_bilinear_sample_forward", (F, F, F, 1, 5, 4, 4, 10), UNSUPPORTED),
    ("umr_bilinear_sample_forward", (N0, F, F, 1, 3, 4, 4, 10), BAD_ARG),
    ("umr_bilinear_sample_forward", (F, F, F, 1, 0, 4, 4, 10), BAD_ARG),
    ("umr_bilinear_sample_forward", (F, ODD, F, 1, 3, 4, 4, 10), BAD_ARG),
    ("umr_bilinear_sample_forward", (F, F, F, 65536, 5, 4, 4, 10), TOO_LARGE),
    ("umr_bilinear_sample_backward", (F, F, F, F, F, 1, 5, 4, 4, 10), UNSUPPORTED),
    ("umr_bilinear_sample_backward", (F, F, F, F, N0, 1, 5, 4, 4, 10), UNSUPPORTED),
    ("umr_bilinear_sample_backward", (F, F, F, N0, F, 1, 3, 4, 4, 10), BAD_ARG),
    ("umr_bilinear_sample_backward", (F, F, F, ODD, F, 1, 3, 4, 4, 10), BAD_ARG),
    ("umr_bilinear_sample_backward", (F, F, F, F, F, 65536, 3, 4, 4, 10), TOO_LARGE),
    ("umr_bilinear_sample_cells", (F, N0, 1, 4, 4, 10), BAD_ARG),
    ("umr_bilinear_sample_cells", (F, F, 2, 65536, 65536, 10), TOO_LARGE),
    ("umr_bilinear_sample_backward_deterministic", (F, F, F, F, F, 1, 3, 4, 4, 10, N0, F), BAD_ARG),
    ("umr_bilinear_sample_backward_deterministic", (F, F, F, F, F, 1, 5, 4, 4, 10, F, F), UNSUPPORTED),
    ("umr_bilinear_sample_backward_deterministic", (F, F, F, F, F, 2, 3, 65536, 65536, 10, F, F), TOO_LARGE),
    # IoU
    ("umr_iou_forward", (F, 16, F, F, F, N0, 1, 16), BAD_ARG),
    ("umr_iou_forward", (F, 16, F, F, F, F, 1, 0), BAD_ARG),
    ("umr_iou_forward", (F, 16, F, F, F, F, 65536, 16), TOO_LARGE),
    ("umr_iou_forward_deterministic", (F, 16, F, F, F, F, 1, 16, N0), BAD_ARG),
    ("umr_iou_forward_deterministic", (F, 16, F, F, F, F, 65536, 16, F), TOO_LARGE),
    ("umr_iou_backward", (F, F, F, F, N0, 1, 16), BAD_ARG),
    ("umr_iou_backward", (F, F, F, F, F, 65536, 16), TOO_LARGE),
    # chamfer; a distance gradient without its indices is refused before grad_a / grad_b are zeroed
    ("umr_chamfer_forward", (F, F, F, F, F, F, 1, 4, 3, 4), UNSUPPORTED),
    ("umr_chamfer_forward", (F, F, F, F, N0, F, 1, 4, 3, 3), BAD_ARG),
    ("umr_chamfer_forward", (F, F, F, F, F, F, 65536, 4, 3, 3), TOO_LARGE),
    ("umr_chamfer_backward", (F, F, N0, F, F, F, F, F, 1, 4, 3, 3), BAD_ARG),
    ("umr_chamfer_backward", (F, F, F, N0, F, F, F, F, 1, 4, 3, 3), BAD_ARG),
    ("umr_chamfer_backward", (F, F, F, N0, N0, F, F, F, 1, 4, 3, 2), BAD_ARG),
    ("umr_chamfer_backward", (F, F, N0, F, F, F, F, F, 1, 4, 3, 4), UNSUPPORTED),
    ("umr_chamfer_backward", (F, F, F, F, F, F, N0, F, 1, 4, 3, 3), BAD_ARG),
    ("umr_chamfer_backward", (F, F, F, F, F, F, F, F, 65536, 4, 3, 3), TOO_LARGE),
    ("umr_chamfer_backward_deterministic", (F, F, F, N0, F, F, F, F, 1, 4, 3, 3), BAD_ARG),
    ("umr_chamfer_backward_deterministic", (F, F, F, F, F, F, F, F, 1, 4, 3, 4), UNSUPPORTED),
    # TexCycle
    ("umr_texcycle_forward", (F, F, F, F, F, 1, 4, 9, 0), BAD_ARG),
    ("umr_texcycle_forward", (F, ODD, N0, F, F, 1, 4, 9, 0), BAD_ARG),
    ("umr_texcycle_forward", (F, F, N0, F, F, 65536, 4, 9, 0), TOO_LARGE),
    ("umr_texcycle_forward", (F, F, N0, F, F, 2, 2 ** 30, 9, 0), TOO_LARGE),
    ("umr_texcycle_forward_deterministic", (F, F, N0, F, F, 1, 4, 9, 0, N0), BAD_ARG),
    ("umr_texcycle_forward_deterministic", (F, F, N0, F, F, 65536, 4, 9, 0, F), TOO_LARGE),
    ("umr_texcycle_backward", (F, F, F, F, ODD, 2, 4, 9), BAD_ARG),
    ("umr_texcycle_backward", (F, F, F, F, F, 2, 2 ** 30, 9), TOO_LARGE),
    # masked L1
    ("umr_masked_l1_forward", (F, 0, F, 0, F, F, F, 1, 2, 16), UNSUPPORTED),
    ("umr_masked_l1_forward", (F, 0, F, 0, F, F, N0, 1, 3, 16), BAD_ARG),
    ("umr_masked_l1_forward", (F, 0, F, 0, F, F, F, 65536, 3, 16), TOO_LARGE),
    ("umr_masked_l1_forward_deterministic", (F, 0, F, 0, F, F, F, 1, 3, 16, N0), BAD_ARG),
    ("umr_masked_l1_forward_deterministic", (F, 0, F, 0, F, F, F, 1, 2, 16, F), UNSUPPORTED),
    ("umr_masked_l1_backward", (F, 0, F, 0, F, F, N0, F, F, 1, 3, 16), BAD_ARG),
    ("umr_masked_l1_backward", (F, 0, F, 0, F, F, F, F, F, 1, 2, 16), UNSUPPORTED),
    # loss head
    ("umr_loss_head_forward", (F, F, F, N0, F, F, 1, 16, 1.0, 1.0), BAD_ARG),
    ("umr_loss_head_forward", (F, F, F, F, F, F, 65536, 16, 1.0, 1.0), TOO_LARGE),
    ("umr_loss_head_forward_deterministic", (F, F, F, F, F, F, 1, 16, 1.0, 1.0, N0), BAD_ARG),
    ("umr_loss_head_backward", (F, F, F, F, F, F, 1, 0, 1.0, 1.0), BAD_ARG),
    ("umr_loss_head_backward", (F, F, F, F, F, F, 65536, 16, 1.0, 1.0), TOO_LARGE),
    # part head (float32 through the dtype argument)
    ("umr_part_head_forward", (_MAPS, _MAP_BS, F, 0, F, 0, F, F, 1, 4, 2, 0, F), BAD_ARG),
    ("umr_part_head_forward", (_MAPS, _MAP_BS, F, 0, F, 0, F, F, 1, 4, 0, 7, F), BAD_ARG),
    ("umr_part_head_forward", (_MAPS, _MAP_BS, F, 0, F, 0, F, F, 65536, 4, 0, 0, F), TOO_LARGE),
    ("umr_part_head_backward", (_MAPS, _MAP_BS, F, 0, F, 0, F, F, F, N0, 1, 4, 0, 0), BAD_ARG),
    # mesh ops
    ("umr_create_texture_image", (F, F, F, 0, 4, 16, 16, 1e-5), BAD_ARG),
    ("umr_create_texture_image", (F, F, F, 100, 4, 16, 5, 1e-5), BAD_ARG),
    ("umr_load_textures", (F, F, F, F, 4, 4, 1, 16), BAD_ARG),
    ("umr_laplacian_forward", (F, F, F, F, F, N0, 1, 5), BAD_ARG),
    ("umr_laplacian_forward", (F, F, F, F, F, F, 65536, 5), TOO_LARGE),
    ("umr_laplacian_forward_deterministic", (F, F, F, F, F, F, 1, 5, N0), BAD_ARG),
    ("umr_laplacian_backward", (F, F, F, F, F, N0, 1, 5), BAD_ARG),
    ("umr_laplacian_backward", (F, F, F, F, F, F, 65536, 5), TOO_LARGE),
    ("umr_flatten_forward", (F, F, F, 1, 5, 0, 1e-6), BAD_ARG),
    ("umr_flatten_forward", (F, F, F, 65536, 5, 3, 1e-6), TOO_LARGE),
    ("umr_flatten_forward_deterministic", (F, F, F, 1, 5, 3, 1e-6, N0), BAD_ARG),
    ("umr_flatten_backward", (F, F, F, N0, 1, 5, 3, 1e-6), BAD_ARG),
    ("umr_flatten_backward", (F, F, F, F, 65536, 5, 3, 1e-6), TOO_LARGE),
    ("umr_flatten_backward_deterministic", (F, F, F, N0, F, F, 1, 5, 3, 1e-6, F), BAD_ARG),
    ("umr_dt_barrier", (F, F, N0, 1, 8, 8, 1.0), BAD_ARG),
    ("umr_dt_barrier", (F, F, F, 1, 8, 4097, 1.0), TOO_LARGE),
    # vertex / projection; a batch that is not a multiple of the hypotheses is refused before the launch
    ("umr_project_faces_forward", (F, F, F, F, F, _proj(B=3, H=2)), BAD_ARG),
    ("umr_project_faces_forward", (F, F, F, F, F, None), BAD_ARG),
    ("umr_project_faces_forward", (F, F, F, N0, F, _proj()), BAD_ARG),
    ("umr_project_faces_forward", (F, F, F, F, F, _proj(B=65536)), TOO_LARGE),
    ("umr_project_faces_backward", (F, F, F, F, F, F, F, F, _proj(B=3, H=2)), BAD_ARG),
    ("umr_project_faces_backward", (F, F, F, F, F, N0, F, F, _proj()), BAD_ARG),
    ("umr_project_faces_backward", (F, F, F, F, F, F, F, F, _proj(B=65536)), TOO_LARGE),
    ("umr_project_faces_backward_deterministic", (F, F, F, F, F, F, F, F, _proj(), F, F, N0), BAD_ARG),
    ("umr_project_faces_backward_deterministic", (F, F, F, F, F, F, F, F, _proj(B=3, H=2), F, F, F), BAD_ARG),
    # CorrLossChamfer
    ("umr_corr_chamfer_forward", _corr(_BAD_ENDS) + (F, F, F, 2, 4), BAD_ARG),
    ("umr_corr_chamfer_forward", _corr() + (F, F, F, 2, 5), BAD_ARG),   # the parts do not cover NS
    ("umr_corr_chamfer_forward", _corr() + (F, N0, F, 2, 4), BAD_ARG),
    ("umr_corr_chamfer_backward", _corr() + (F, F, N0, F, F, F, 2, 4, 9), BAD_ARG),
    ("umr_corr_chamfer_backward", _corr(_BAD_ENDS) + (F, F, F, F, F, F, 2, 4, 9), BAD_ARG),
    ("umr_corr_chamfer_backward_deterministic", _corr() + (F, F, F, N0, F, N0, 2, 4, 9, N0, N0, F), BAD_ARG),
    ("umr_corr_chamfer_backward_deterministic", _corr() + (F, F, F, N0, N0, F, 65536, 4, 9, N0, N0, N0), TOO_LARGE),
    # peer all-reduce
    ("umr_p2p_allreduce", (F, F, 3, 256, F, 0, 2, 1.0), BAD_ARG),
    ("umr_p2p_allreduce", (F, F, 4, 256, F, 2, 2, 1.0), BAD_ARG),
    ("umr_p2p_allreduce", (F, F, 4, 8, F, 0, 2, 1.0), BAD_ARG),
    ("umr_p2p_allreduce", (N0, F, 4, 256, F, 0, 2, 1.0), BAD_ARG),
]


def _id(case):
    name, args, code = case
    return "%s-%d" % (name[4:], CASES.index(case))


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def test_every_entry_point_is_covered():
    names = {c[0] for c in CASES}
    float32 = {n for n in _lib.EXPORTS if not n.endswith("_f64") and not n.startswith(("umr_raster", "umr_nmr", "umr_voxel"))
               and "workspace" not in n and "sizeof" not in n and "flag_bytes" not in n and "event" not in n}
    float32 -= {"umr_error_string", "umr_version", "umr_launch_count"}
    assert float32 <= names, sorted(float32 - names)


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_refused_before_device_work(lib, case):
    name, args, code = case
    before = lib.umr_launch_count()
    assert getattr(lib, name)(*args, None) == code
    assert lib.umr_launch_count() == before
