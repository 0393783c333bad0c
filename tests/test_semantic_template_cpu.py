"""The SCOPS semantic template (DESIGN.md §18) without a GPU: the numpy restatement pinned against the reference's own
`compute_uv` (tests/golden/semantic_template/reference.npz, made by tests/golden/make_semantic_template_golden.py), its
tie, NaN and incidence rules on hand-built cases, and every refusal of the C ABI and of the Python arguments, which
come before any device work."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import semantic_template_oracle as sto
from umr_b200 import _lib
from umr_b200.utils import semantic_template as st

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "semantic_template", "reference.npz")
PARTS = ("head", "neck", "back", "belly")


# ---------------------------------------------------------------------------------------------------------------------
# the restatement against the reference's own compute_uv
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_average_matches_the_reference(golden):
    batches = [(golden["part_segs"][i], golden["uvimage_pred"][i]) for i in range(len(golden["part_segs"]))]
    avg, _ = sto.average(batches, golden["best_uv"], int(golden["k"]))
    # the reference's grid_sample and torch.sum round differently: float32 summation tolerance on values <= 1
    np.testing.assert_allclose(avg, golden["semantic_prob"], rtol=0, atol=4 * 2.0 ** -24 * (2 * int(golden["k"]) + 8))
    np.testing.assert_array_equal(sto.argmax(avg, 2).astype(np.uint8), golden["semantic_seg"])


def test_labels_and_parts_match_the_reference(golden):
    lab = sto.label(golden["semantic_prob"], golden["uv_sampler"], golden["faces"], int(golden["num_sym_faces"]))
    np.testing.assert_array_equal(lab["label_image"], golden["semantic_seg"])
    for p, name in enumerate(PARTS):
        np.testing.assert_array_equal(lab["part_vertices"][p], golden[name])
    assert all(len(golden[n]) > 0 for n in PARTS)


# ---------------------------------------------------------------------------------------------------------------------
# the contract's rules on hand-built cases
# ---------------------------------------------------------------------------------------------------------------------
def test_argmax_ties_take_the_lowest_channel_and_the_first_nan_wins():
    nan = np.nan
    v = np.array([[0.2, 0.4, 0.4, 0.0], [0.3, nan, 0.9, nan], [nan, 0.1, 0.1, 0.1], [0.5, 0.5, 0.5, 0.5]], np.float32)
    np.testing.assert_array_equal(sto.argmax(v, 1), [1, 1, 0, 0])


def test_mode_ties_take_the_smallest_label():
    assert sto.mode(np.array([3, 1, 3, 1, 2]), 5) == 1
    assert sto.mode(np.array([4]), 5) == 4
    assert sto.mode(np.array([], np.int64), 5) == -1


def test_selection_orders_by_distance_then_index_with_nan_last():
    d = np.array([2.0, np.nan, 1.0, 2.0, np.inf, 0.5, np.nan], np.float32)
    np.testing.assert_array_equal(sto.select(d, 7), [5, 2, 0, 3, 4, 1, 6])
    np.testing.assert_array_equal(sto.select(d, 3), [5, 2, 0])


def test_the_k_maps_are_summed_before_the_accumulator():
    big, small = np.float32(2.0 ** 24), np.float32(1.0)
    acc = np.full((1, 1, 1), big, np.float32)
    parts = np.array([small, small], np.float32).reshape(2, 1, 1, 1)
    # (1 + 1) + 2^24 is exact; adding each 1 to 2^24 in turn would round both away
    assert sto.accumulate(acc, parts, [0, 1])[0, 0, 0] == big + 2


def _one_channel_template(face_label_of_texels, faces, num_vertices=None):
    """A 1 x 2 label image whose two pixels are labels 0 and 1 of C = 2, faces sampled at one pixel or the other."""
    avg = np.array([[[1.0, 0.0], [0.0, 1.0]]], np.float32)          # [H=1, W=2, C=2]
    x = np.where(np.asarray(face_label_of_texels) == 1, 1.0, -1.0).astype(np.float32)
    sampler = np.stack([x, np.zeros_like(x)], axis=-1)                # [F,T2,2]
    return sto.label(avg, sampler, faces, 0, num_vertices)


def test_a_vertex_on_one_face_takes_its_label_and_a_vertex_on_none_gets_minus_one():
    # face 0 = (0, 1, 2) label 1, face 1 = (1, 2, 3) label 0; vertex 4 is on no face, vertex 0 on face 0 only
    lab = _one_channel_template([[1, 1, 0], [0, 0, 0]], [[0, 1, 2], [1, 2, 3]], num_vertices=5)
    np.testing.assert_array_equal(lab["face_labels"], [1, 0])
    np.testing.assert_array_equal(lab["vertex_labels"], [1, 0, 0, 0, -1])   # 1 and 2: a tie of labels 0 and 1 -> 0
    np.testing.assert_array_equal(lab["part_vertices"][0], [0])


def test_a_face_repeating_a_vertex_counts_once():
    # vertex 0 is on face 0 (label 0) twice and on faces 1 and 2 (label 1): {0, 1, 1} -> 1, where counting face 0's
    # corners twice would tie {0, 0, 1, 1} -> 0
    lab = _one_channel_template([[0], [1], [1], [0]], [[0, 0, 1], [0, 1, 2], [2, 0, 3], [1, 2, 3]])
    assert lab["vertex_labels"][0] == 1


def test_symmetric_faces_take_their_source_faces_samples():
    avg = np.array([[[1.0, 0.0], [0.0, 1.0]]], np.float32)
    sampler = np.array([[[-1.0, 0.0]], [[1.0, 0.0]], [[-1.0, 0.0]]], np.float32)   # F' = 3, labels 0 1 0
    lab = sto.label(avg, sampler, [[0, 1, 2]] * 5, 2)
    np.testing.assert_array_equal(lab["face_labels"], [0, 1, 0, 1, 0])


def test_sampler_matches_grid_sample_align_corners():
    rng = np.random.default_rng(0)
    img = rng.random((3, 7, 9)).astype(np.float32)
    xy = rng.uniform(-1.3, 1.3, (2, 40)).astype(np.float32)
    want = torch.nn.functional.grid_sample(torch.from_numpy(img)[None], torch.from_numpy(xy.T.copy()).view(1, 1, 40, 2),
                                           align_corners=True)[0, :, 0].numpy()
    np.testing.assert_allclose(sto.bilinear(img, xy[0], xy[1]), want, rtol=0, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------------
# C ABI: declaration, export and refusals (no GPU: a refusal comes before any device work)
# ---------------------------------------------------------------------------------------------------------------------
def test_header_declares_exactly_the_bound_symbols():
    src = open(os.path.join(ROOT, "include", "umr_semantic_template.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = set(re.findall(r"\b(umr_[a-z0-9_]+)\s*\(", src))
    assert names == set(_lib.ST_EXPORTS)
    assert '#include "umr_semantic_template.h"' in open(os.path.join(ROOT, "include", "umr_b200.h")).read()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(lib, n)


A = 256          # non-NULL, aligned to 16
BAD_ARG, TOO_LARGE = -2, -3


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _add(*, segs=A, uv=A, ex=A, B=8, C=5, S=64, H=128, W=256, k=5, ws=A, dist=A, sel=A, acc=A):
    return (segs, uv, ex, B, C, S, H, W, k, ws, dist, sel, acc)


def _mean(*, acc=A, C=5, H=128, W=256, count=10, avg=A):
    return (acc, C, H, W, count, avg)


def _labels(*, avg=A, H=128, W=256, C=5, uvs=A, Fs=656, T2=36, nsym=624, rowptr=A, corners=A, V=642, img=A, tex=A,
            face=A, vert=A):
    return (avg, H, W, C, uvs, Fs, T2, nsym, rowptr, corners, V, img, tex, face, vert)


ADD_REFUSALS = (
    [(_add(**{k: None}), BAD_ARG) for k in ("segs", "uv", "ex", "ws", "dist", "sel", "acc")]
    + [(_add(**{k: A + 2}), BAD_ARG) for k in ("segs", "uv", "ex", "ws", "dist", "sel", "acc")]
    + [(_add(**{k: v}), BAD_ARG) for k in ("B", "C", "S", "H", "W", "k") for v in (0, -1)]
    + [(_add(k=9), BAD_ARG), (_add(B=1025, k=5), TOO_LARGE), (_add(C=33), TOO_LARGE),
       (_add(S=2 ** 15), TOO_LARGE), (_add(H=2 ** 15, W=2 ** 15), TOO_LARGE)]
)
MEAN_REFUSALS = (
    [(_mean(**{k: None}), BAD_ARG) for k in ("acc", "avg")] + [(_mean(**{k: A + 1}), BAD_ARG) for k in ("acc", "avg")]
    + [(_mean(**{k: v}), BAD_ARG) for k in ("C", "H", "W", "count") for v in (0, -1)]
    + [(_mean(C=33), TOO_LARGE), (_mean(H=2 ** 15, W=2 ** 15), TOO_LARGE)]
)
LABEL_REFUSALS = (
    [(_labels(**{k: None}), BAD_ARG) for k in ("avg", "uvs", "rowptr", "corners", "img", "tex", "face", "vert")]
    + [(_labels(**{k: A + 2}), BAD_ARG) for k in ("avg", "rowptr", "corners", "tex", "face", "vert")]
    + [(_labels(uvs=A + 4), BAD_ARG)]
    + [(_labels(**{k: v}), BAD_ARG) for k in ("H", "W", "C", "Fs", "T2", "V") for v in (0, -1)]
    + [(_labels(nsym=-1), BAD_ARG), (_labels(nsym=657), BAD_ARG)]
    + [(_labels(C=33), TOO_LARGE), (_labels(H=2 ** 15, W=2 ** 15), TOO_LARGE), (_labels(V=2 ** 30), TOO_LARGE),
       (_labels(Fs=2 ** 28, nsym=2 ** 28), TOO_LARGE), (_labels(Fs=2 ** 20, nsym=0, T2=2 ** 10), TOO_LARGE)]
)


@pytest.mark.parametrize("args,code", ADD_REFUSALS, ids=[str(i) for i in range(len(ADD_REFUSALS))])
def test_average_add_refused_before_device_work(lib, args, code):
    before = lib.umr_launch_count()
    assert lib.umr_st_average_add(*args, None) == code
    assert lib.umr_launch_count() == before


@pytest.mark.parametrize("args,code", MEAN_REFUSALS, ids=[str(i) for i in range(len(MEAN_REFUSALS))])
def test_average_mean_refused_before_device_work(lib, args, code):
    before = lib.umr_launch_count()
    assert lib.umr_st_average_mean(*args, None) == code
    assert lib.umr_launch_count() == before


@pytest.mark.parametrize("args,code", LABEL_REFUSALS, ids=[str(i) for i in range(len(LABEL_REFUSALS))])
def test_labels_refused_before_device_work(lib, args, code):
    before = lib.umr_launch_count()
    assert lib.umr_st_labels(*args, None) == code
    assert lib.umr_launch_count() == before


def test_workspace_bytes(lib):
    assert lib.umr_st_average_workspace_bytes(32, 128, 256) == 32 * 32 * 4
    assert lib.umr_st_average_workspace_bytes(3, 5, 7) == 3 * 4
    for args in ((0, 8, 8), (8, 0, 8), (8, 8, -1), (1025, 8, 8), (8, 2 ** 15, 2 ** 15)):
        assert lib.umr_st_average_workspace_bytes(*args) == 0


# ---------------------------------------------------------------------------------------------------------------------
# Python argument checks (before any device work)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def claims_cuda(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def test_cpu_tensors_are_refused():
    with pytest.raises(TypeError, match="exemplar_uv"):
        st.UVPartAverage(torch.zeros(5, 8, 16))
    with pytest.raises(TypeError, match="avg_prob"):
        st.semantic_template(torch.zeros(8, 16, 5), torch.zeros(1, 4, 1, 2), torch.zeros(6, 3, dtype=torch.long), 2)


@pytest.mark.parametrize("exemplar,k,match", [
    (torch.zeros(5, 8, 16, dtype=torch.float64), 5, "exemplar_uv must be float32"),
    (torch.zeros(1, 5, 8, 16), 5, "exemplar_uv must have 3"),
    (torch.zeros(33, 8, 16), 5, "exemplar_uv must have 1 to 32"),
    (torch.zeros(5, 8, 16), 0, "k must be"),
    (torch.zeros(5, 8, 16), 1025, "k must be"),
    (torch.zeros(5, 8, 16), 2.5, "k must be"),
])
def test_average_constructor_checks(claims_cuda, exemplar, k, match):
    with pytest.raises((TypeError, ValueError), match=match):
        st.UVPartAverage(exemplar, k)


@pytest.mark.parametrize("segs,uv,match", [
    ((8, 5, 32, 32), (8, 2, 8, 17), "uvimage_pred must be"),
    ((8, 4, 32, 32), (8, 2, 8, 16), "part_segs must be"),
    ((8, 5, 32, 31), (8, 2, 8, 16), "part_segs must be"),
    ((4, 5, 32, 32), (4, 2, 8, 16), "k = 5"),
    ((1025, 5, 2, 2), (1025, 2, 8, 16), "k = 5"),
    ((8, 5, 32), (8, 2, 8, 16), "part_segs must have 4"),
])
def test_average_add_checks(claims_cuda, segs, uv, match):
    avg = st.UVPartAverage(torch.zeros(5, 8, 16))
    with pytest.raises(ValueError, match=match):
        avg.add(torch.zeros(segs), torch.zeros(uv))
    assert avg.count == 0


def test_average_add_refuses_mixed_devices_and_dtypes(claims_cuda):
    avg = st.UVPartAverage(torch.zeros(5, 8, 16))
    with pytest.raises(ValueError, match="one device"):
        avg.add(torch.zeros(8, 5, 4, 4, device="meta"), torch.zeros(8, 2, 8, 16))
    with pytest.raises(TypeError, match="uvimage_pred must be float32"):
        avg.add(torch.zeros(8, 5, 4, 4), torch.zeros(8, 2, 8, 16, dtype=torch.float16))


def test_mean_of_nothing_is_refused(claims_cuda):
    with pytest.raises(ValueError, match="no batch"):
        st.UVPartAverage(torch.zeros(5, 8, 16)).mean()


@pytest.mark.parametrize("prob,sampler,faces,nsym,nv,match", [
    ((8, 16, 33), (1, 4, 4, 2), (6, 3), 2, None, "1 to 32 channels"),
    ((8, 16, 5), (4, 4, 2), (6, 3), 2, None, "uv_sampler must have 4"),
    ((8, 16, 5), (2, 4, 4, 2), (6, 3), 2, None, r"uv_sampler must be \[1"),
    ((8, 16, 5), (1, 4, 4, 3), (6, 3), 2, None, r"uv_sampler must be \[1"),
    ((8, 16, 5), (1, 4, 5, 2), (6, 3), 2, None, "tex_size"),
    ((8, 16, 5), (1, 4, 4, 2), (6, 3), 0, None, "num_sym_faces"),
    ((8, 16, 5), (1, 4, 4, 2), (9, 3), 5, None, "num_sym_faces"),
    ((8, 16, 5), (1, 4, 4, 2), (7, 3), 2, None, "faces must be"),
    ((8, 16, 5), (1, 4, 4, 2), (6, 4), 2, None, "faces must be"),
    ((8, 16, 5), (1, 4, 4, 2), (6, 3), 2, 0, "num_vertices"),
])
def test_semantic_template_checks(claims_cuda, prob, sampler, faces, nsym, nv, match):
    with pytest.raises(ValueError, match=match):
        st.semantic_template(torch.zeros(prob), torch.zeros(sampler), torch.zeros(faces, dtype=torch.long), nsym, nv)


def test_semantic_template_refuses_float_faces_and_mixed_devices(claims_cuda):
    with pytest.raises(TypeError, match="faces must be int"):
        st.semantic_template(torch.zeros(8, 16, 5), torch.zeros(1, 4, 4, 2), torch.zeros(6, 3), 2)
    with pytest.raises(ValueError, match="one device"):
        st.semantic_template(torch.zeros(8, 16, 5), torch.zeros(1, 4, 4, 2, device="meta"),
                             torch.zeros(6, 3, dtype=torch.long), 2)
