"""Host-side contract of the deterministic vertex, NMR-texture and sampler backwards (no GPU): the new entry points are
exported, the vertex workspace query follows its header formula (0 for empty or negative sizes), and the device-built
transposed tables (`ops.device_incidence`, `vertex._corner_incidence`) equal a brute-force inversion on CPU tensors."""
import numpy as np
import pytest
import torch

from umr_b200 import _lib, ops, synth
from umr_b200.vertex import _corner_incidence

ENTRY_POINTS = ("umr_project_faces_workspace_bytes_deterministic", "umr_project_faces_backward_deterministic",
                "umr_nmr_backward_textures_deterministic", "umr_bilinear_sample_cells",
                "umr_bilinear_sample_backward_deterministic")


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def test_symbols_exported(lib):
    for name in ENTRY_POINTS:
        assert name in _lib.EXPORTS
        assert getattr(lib, name) is not None


def _vertex_ws(B, V, F):
    """include/umr_b200.h: 4 * B * (9 * F + 3 * V + 7 * ceil(V / 256))"""
    return 4 * B * (9 * F + 3 * V + 7 * ((V + 255) // 256))


@pytest.mark.parametrize("B,V,F", [(1, 1, 1), (1, 3, 1), (2, 255, 256), (16, 256, 1280), (128, 257, 1280), (8, 163842, 327680),
                                   (65535, 642, 1280)])
def test_vertex_workspace_formula(lib, B, V, F):
    assert lib.umr_project_faces_workspace_bytes_deterministic(B, V, F) == _vertex_ws(B, V, F)


def test_vertex_workspace_empty_sizes(lib):
    q = lib.umr_project_faces_workspace_bytes_deterministic
    for args in ((0, 10, 10), (4, 0, 10), (4, 10, 0), (-1, 10, 10), (4, -3, 10), (4, 10, -7)):
        assert q(*args) == 0, args


def brute_force(keys, rows):
    flat = np.asarray(keys).reshape(-1)
    lists = [[k for k in range(flat.size) if flat[k] == r] for r in range(rows)]
    rowptr = np.cumsum([0] + [len(x) for x in lists])
    return rowptr, np.array([k for x in lists for k in x], dtype=np.int64)


def _check_table(table, keys, rows):
    rowptr, pos = table
    assert rowptr.dtype == torch.int32 and pos.dtype == torch.int32
    assert pos.numel() == np.asarray(keys).size   # dropped keys sit after rowptr[rows]
    want_ptr, want_pos = brute_force(keys, rows)
    assert np.array_equal(rowptr.numpy(), want_ptr)
    assert np.array_equal(pos[:int(rowptr[-1])].numpy(), want_pos)
    dropped = sorted(set(range(np.asarray(keys).size)) - set(want_pos.tolist()))
    assert sorted(pos[int(rowptr[-1]):].tolist()) == dropped


def test_device_incidence_shared_faces():
    v, f = synth.icosphere(2)
    faces = torch.from_numpy(f.astype(np.int32))
    _check_table(ops.device_incidence(faces, v.shape[0]), f, v.shape[0])
    _check_table(_corner_incidence(faces[None], v.shape[0], False), f, v.shape[0])


def test_device_incidence_batched_faces_with_keys_to_drop():
    rng = np.random.default_rng(3)
    V, F, Bv = 40, 70, 3
    f = np.stack([rng.permutation(np.stack([rng.permutation(V)[:3] for _ in range(F)])) for _ in range(Bv)]).astype(np.int32)
    f[1, 5, 1] = V          # out of range: must not land in mesh 2's rows
    f[2, 0, 0] = -1
    f[0, 9, 2] = V + 1000
    keys = np.where((f >= 0) & (f < V), f + np.arange(Bv)[:, None, None] * V, -1)
    _check_table(_corner_incidence(torch.from_numpy(f), V, True), keys, Bv * V)
    # keys outside [0, rows) in a plain key list, on both sides
    k = np.array([3, -2, 0, 7, 3, 5, 12, 0, -1], dtype=np.int64)
    _check_table(ops.device_incidence(torch.from_numpy(k), 7), k, 7)


def test_device_incidence_empty_and_one_hub_vertex():
    _check_table(ops.device_incidence(torch.zeros(0, 3, dtype=torch.int32), 5), np.zeros((0, 3), np.int64), 5)
    # a fan: vertex 0 is a corner of every face
    F = 300
    f = np.stack([np.zeros(F, np.int64), 1 + np.arange(F), 1 + (np.arange(F) + 1) % F], 1)
    rowptr, pos = ops.device_incidence(torch.from_numpy(f), F + 1)
    _check_table((rowptr, pos), f, F + 1)
    assert int(rowptr[1]) == F and np.array_equal(pos[:F].numpy(), 3 * np.arange(F))


def test_device_incidence_refuses_int32_overflow():
    with pytest.raises(ValueError):
        ops.device_incidence(torch.zeros(3, dtype=torch.int64), 2 ** 31)
