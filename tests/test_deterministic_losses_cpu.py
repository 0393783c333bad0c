"""Host-side contract of the loss kernels' deterministic mode (no GPU): the new entry points are exported, every workspace
query follows its formula (a function of the sizes only, 0 for an empty size), and the transposed index tables the
deterministic gathers sum over equal a brute-force inversion."""
import numpy as np
import pytest
import torch

from umr_b200 import _lib, ops, synth
from umr_b200 import soft_renderer as sr
from umr_b200.nnutils import loss_utils

ENTRY_POINTS = ("umr_iou_forward_deterministic", "umr_masked_l1_forward_deterministic", "umr_loss_head_forward_deterministic",
                "umr_texcycle_forward_deterministic", "umr_laplacian_forward_deterministic",
                "umr_flatten_forward_deterministic", "umr_flatten_backward_deterministic",
                "umr_chamfer_backward_deterministic", "umr_corr_chamfer_backward_deterministic")


def _cdiv(a, b):
    return (a + b - 1) // b


# query -> bytes for sizes (a, b): one float slot per reduction CTA (IoU: two), or the gathers' per-term arrays
FORMULAS = {
    "umr_iou_workspace_bytes_deterministic": lambda B, N: 8 * B * _cdiv(N, 512 * 4 * 8),
    "umr_masked_l1_workspace_bytes_deterministic": lambda B, HW: 4 * B * _cdiv(HW, 256 * 8),
    "umr_loss_head_workspace_bytes_deterministic": lambda B, HW: 12 * B * _cdiv(HW, 256 * 8),
    "umr_texcycle_workspace_bytes_deterministic": lambda B, F: 4 * _cdiv(B * F, 256),
    "umr_laplacian_workspace_bytes_deterministic": lambda B, V: 4 * B * _cdiv(V, 256),
    "umr_flatten_forward_workspace_bytes_deterministic": lambda B, E: 4 * B * _cdiv(E, 128),
    "umr_flatten_backward_workspace_bytes_deterministic": lambda B, E: 48 * B * E,
    "umr_corr_chamfer_workspace_bytes_deterministic": lambda B, NS: 12 * B * NS,
}


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def test_symbols_exported(lib):
    for name in ENTRY_POINTS + tuple(FORMULAS):
        assert name in _lib.EXPORTS
        assert getattr(lib, name) is not None


@pytest.mark.parametrize("name", list(FORMULAS))
@pytest.mark.parametrize("a,b", [(1, 1), (16, 65536), (256, 262144), (1, 4194304), (3, 1001), (128, 1920), (16, 102400)])
def test_workspace_formula(lib, name, a, b):
    assert getattr(lib, name)(a, b) == FORMULAS[name](a, b)


@pytest.mark.parametrize("name", list(FORMULAS))
def test_workspace_empty_sizes(lib, name):
    q = getattr(lib, name)
    assert q(0, 100) == 0 and q(4, 0) == 0 and q(-1, 100) == 0 and q(4, -5) == 0


def brute_force(index, V):
    flat = np.asarray(index).reshape(-1)
    rows = [[k for k in range(flat.size) if flat[k] == v] for v in range(V)]
    rowptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    return rowptr, np.array([k for r in rows for k in r], np.int32)


def check_table(rowptr, pos, index, V):
    want_ptr, want_pos = brute_force(index, V)
    assert rowptr.dtype == np.int32 and pos.dtype == np.int32
    assert np.array_equal(rowptr, want_ptr)
    assert np.array_equal(pos, want_pos)


def _open_mesh():
    """The upper half of an icosphere: a mesh with boundary edges (only interior edges enter the flatten loss)."""
    v, f = synth.icosphere(2)
    keep = v[f].mean(1)[:, 2] > 0
    return f[keep]


@pytest.mark.parametrize("mesh", ["icosphere3", "open"])
def test_flatten_incidence_table(mesh):
    f = synth.icosphere(3)[1] if mesh == "icosphere3" else _open_mesh()
    m = sr.FlattenLoss(torch.from_numpy(f.astype(np.int64)))
    V = int(f.max()) + 1
    edges = m.edge_table.numpy()
    if mesh == "open":
        assert edges.shape[0] < len({tuple(sorted(e)) for t in f for e in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0]))})
    check_table(m.vert_rowptr.numpy(), m.vert_incidence.numpy(), edges, V)
    # the tables are buffers that follow .to(), but stay out of the state dict
    assert "vert_rowptr" not in m.state_dict() and "vert_incidence" not in m.state_dict()
    assert {n for n, _ in m.named_buffers()} >= {"vert_rowptr", "vert_incidence"}


def test_corr_selection_table_shared_vertex_and_empty_part():
    V = 50
    parts = [torch.tensor([3, 7, 11]), torch.tensor([7, 20, 3, 49]), torch.tensor([], dtype=torch.long), torch.tensor([0, 11])]
    rowptr, pos = loss_utils._vertex_table(parts, V, "cpu")
    sel = torch.cat(parts).numpy()
    check_table(rowptr.numpy(), pos.numpy(), sel, V)
    assert list(pos.numpy()[rowptr[7]:rowptr[8]]) == [1, 3]        # vertex 7 in parts 0 and 1, ascending j
    assert list(pos.numpy()[rowptr[11]:rowptr[12]]) == [2, 8]
    assert int(rowptr[1] - rowptr[0]) == 1 and int(rowptr[2] - rowptr[1]) == 0   # vertex 0 once (part 3), vertex 1 never


def test_vertex_incidence_rejects_out_of_range():
    with pytest.raises(IndexError):
        ops.vertex_incidence(np.array([0, 5]), 5)
    with pytest.raises(IndexError):
        ops.vertex_incidence(np.array([-1, 2]), 5)
    rowptr, pos = ops.vertex_incidence(np.zeros((0, 4), np.int32), 3)
    assert list(rowptr) == [0, 0, 0, 0] and pos.size == 0
