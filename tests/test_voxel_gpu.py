"""`voxelization` on the H100 (csrc/voxel.cu through umr_voxelize): bit-exact against the numpy oracle
(oracle/voxel_oracle.py) and the reference's own extension built with -fmad=false, the FMA build's differences bounded,
the fill's convergence on a labyrinth, CUDA-graph capture, a constant launch count, and the drop-in surface
(`Mesh.voxelize`, `functional.voxelization`, `save_voxel`).  Every call's status word is checked."""
import os
import sys

import numpy as np
import pytest
import torch

import voxel_oracle as vo
from umr_b200 import _lib, ops, synth

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import voxel_bench as vb  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def run(faces, vs, normalize=False):
    out = ops.voxelize(faces, vs, normalize)
    assert ops.voxelize_status(faces.device) == 0, "fill stopped at its sweep cap"
    return out


def bird(B, subdiv, dtype, seed=0):
    v, f = synth.icosphere(subdiv)
    verts = synth.bird_like(v, np.random.default_rng(seed), B).astype(np.float64) * 0.45 + 0.5
    return np.ascontiguousarray(verts[:, f]).astype(dtype)


def soup(B, vs, dtype, seed=0, nonfinite=True):
    """Random triangles in and around the unit cube plus the awkward ones: slivers, det == 0 faces, faces partly and
    wholly outside the grid, vertices on grid planes, NaN / inf coordinates."""
    rng = np.random.default_rng(seed + vs)
    f = rng.uniform(-0.3, 1.3, size=(B, 48, 3, 3))
    f[:, 0, 1] = f[:, 0, 0]                                             # zero area
    f[:, 1, 2] = 2 * f[:, 1, 1] - f[:, 1, 0]                           # collinear
    f[:, 2, 2] = f[:, 2, 0] + 1e-7 * (f[:, 2, 1] - f[:, 2, 0]) + np.array([0, 1e-6, 0])   # slivers
    f[:, 3, 2] = f[:, 3, 0] + 1e-3 * rng.normal(size=(B, 3))
    f[:, 4] = rng.uniform(1.5, 3.0, size=(B, 3, 3))                    # wholly outside
    f[:, 5] = rng.uniform(-1.0, 0.3, size=(B, 3, 3))                   # partly outside
    f[:, 6] = np.round(f[:, 6] * vs) / vs                               # on grid planes
    f[:, 7:12] = f[:, 7:12] * 0.05 + rng.uniform(0, 1, size=(B, 5, 1, 3))  # small faces
    if nonfinite:
        f[:, 12, 0, 2] = np.nan
        f[:, 13, 1, 0] = np.inf
        f[:, 14, 2, 1] = -np.inf
        f[:, 15, :, :] = np.nan
    return f.astype(dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("vs", [1, 2, 3, 31, 32, 64, 65, 128])
@pytest.mark.parametrize("B", [1, 3])
def test_bit_exact_against_oracle(dtype, vs, B):
    for m in (bird(B, 2 if vs >= 64 else 3, dtype, seed=vs), soup(B, vs, dtype)):
        faces = torch.from_numpy(m).to(DEV)
        got = run(faces, vs).cpu().numpy()
        want = vo.voxelization_np(m, vs)
        assert got.dtype == np.int32 and got.shape == (B, vs, vs, vs)
        bad = np.argwhere(got != want)
        assert len(bad) == 0, "%d voxels differ, first %s" % (len(bad), bad[:5].tolist())


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_normalize_true(dtype):
    vs = 48
    m = (bird(2, 3, dtype) * dtype(vs)).astype(dtype)
    got = run(torch.from_numpy(m).to(DEV), vs, normalize=True).cpu().numpy()
    np.testing.assert_array_equal(got, vo.voxelization_np(m, vs, normalize=True))


def labyrinth(vs):
    """Nested boxes, each with a hole on a different side: the gaps form one winding cavity open to the outside."""
    parts, lo, hi, k = [], 1.5, vs - 2.5, 0
    while hi - lo > 6:
        ax, side = k % 3, (k // 3) % 2
        h0, h1 = (lo + 1, lo + 3) if k % 2 else (hi - 3, hi - 1)
        parts.append(vo.box_with_hole(lo, hi, ax, side, h0, h1))
        lo, hi, k = lo + 2, hi - 2, k + 1
    parts.append(vo.box_faces(lo, hi))  # a closed core: filled
    return np.concatenate(parts)[None]


@pytest.mark.parametrize("vs", [40, 64, 100])
def test_labyrinth_converges(vs):
    m = labyrinth(vs).astype(np.float32)
    got = run(torch.from_numpy(m).to(DEV), vs, normalize=True).cpu().numpy()
    want = vo.voxelization_np(m, vs, normalize=True)
    np.testing.assert_array_equal(got, want)
    occ = vo.occupancy_np(m, vs, normalize=True)
    assert (want.astype(bool) & ~occ).sum() > 0          # the closed core is filled
    assert (want[0, 3:vs - 4, 3:vs - 4, 3:vs - 4] == 0).any()  # the winding gaps are not


def test_launch_count_is_independent_of_the_fill():
    lib = _lib.load()
    one = torch.from_numpy(np.asarray([[[[0.2, 0.2, 0.5], [0.8, 0.2, 0.5], [0.2, 0.8, 0.5]]]], np.float32)).to(DEV)
    many = torch.from_numpy(labyrinth(64).astype(np.float32)).to(DEV)
    counts = []
    for faces, norm in ((one, False), (many, True)):
        n0 = lib.umr_launch_count()
        run(faces, 64, norm)
        counts.append(lib.umr_launch_count() - n0)
    assert counts == [3, 3]


def test_graph_capture_replays_the_eager_result():
    faces = torch.from_numpy(bird(3, 3, np.float32)).to(DEV)
    for vs in (64, 96):
        eager = run(faces, vs)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            run(faces, vs)  # warm-up on the capture stream
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = ops.voxelize(faces, vs)
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert ops.voxelize_status(DEV) == 0
        assert torch.equal(out, eager)


def test_input_untouched():
    m = soup(2, 32, np.float32)
    faces = torch.from_numpy(m).to(DEV)
    before = faces.clone()
    run(faces, 32)
    run(faces, 32, normalize=True)
    assert torch.equal(faces.view(torch.int32), before.view(torch.int32))


def test_mesh_voxelize_and_dropin(tmp_path):
    from umr_b200 import compat
    compat.install()
    import soft_renderer as sr
    v, f = synth.icosphere(3)
    verts = torch.from_numpy(synth.bird_like(v, np.random.default_rng(3), 2) * 0.5).to(DEV)
    mesh = sr.Mesh(verts, torch.from_numpy(f).to(DEV).int()[None].repeat(2, 1, 1))
    for vs in (32, 50):
        got = mesh.voxelize(vs)
        assert ops.voxelize_status(DEV) == 0
        fvn = mesh.face_vertices * vs / (vs - 1) + 0.5  # SoftRas/mesh.py:178, same torch ops
        np.testing.assert_array_equal(got.cpu().numpy(), vo.voxelization_np(fvn.cpu().numpy(), vs))
    assert sr.Mesh(verts[:1], torch.from_numpy(f).to(DEV).int()).voxelize().shape == (1, 32, 32, 32)
    out = sr.functional.voxelization(fvn, vs)
    np.testing.assert_array_equal(out.cpu().numpy(), got.cpu().numpy())
    fn = str(tmp_path / "vox.obj")
    sr.functional.save_voxel(fn, out[0])
    n = sum(1 for ln in open(fn) if ln.startswith("v "))
    assert n == int(out[0].sum())


def test_refusals():
    faces = torch.zeros(1, 4, 3, 3, device=DEV)
    with pytest.raises(TypeError):
        ops.voxelize(faces.half(), 8)
    with pytest.raises(ValueError):
        ops.voxelize(faces, 0)
    with pytest.raises(RuntimeError, match="exceeds"):
        ops.voxelize(faces, 1291)
    assert run(faces[:, :0], 4).sum() == 0  # no faces: all empty voxels reach the boundary


# ------------------------------------------------------------------------------------------------------------------
# the reference's own extension (oracle/build_ref_voxel.py)
# ------------------------------------------------------------------------------------------------------------------
REF_NOFMA, REF_FMA = vb.load_ref("voxelization_ref_nofma"), vb.load_ref("voxelization_ref")


@pytest.mark.skipif(REF_NOFMA is None, reason="oracle/_ref/voxelization_ref_nofma.so not built")
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("vs", [2, 31, 64, 65, 128])
def test_bit_exact_against_reference_built_without_fma(dtype, vs):
    # finite inputs only: the reference converts floor(NaN) to int, which is undefined (DESIGN.md §8)
    for m in (bird(3, 3, np.float64, seed=vs), soup(2, vs, np.float64, nonfinite=False)):
        faces = torch.from_numpy(m).to(DEV, dtype)
        assert torch.equal(run(faces, vs), vb.ref_voxelization(REF_NOFMA, faces, vs))


@pytest.mark.skipif(REF_FMA is None, reason="oracle/_ref/voxelization_ref.so not built")
@pytest.mark.parametrize("vs", [32, 64, 128])
def test_fma_build_differs_only_at_the_surface(vs):
    """Contracting a*b+c into FMA changes the last bits of t1, t2 and the depth, so a column on a triangle edge or a depth
    within rounding of an integer can land differently.  The differences must sit next to our surface, and be few."""
    faces = torch.from_numpy(bird(4, 3, np.float32, seed=vs)).to(DEV)
    got, want = run(faces, vs), vb.ref_voxelization(REF_FMA, faces, vs)
    diff = (got != want).cpu().numpy()
    occ = vo.occupancy_np(faces.cpu().numpy(), vs)
    from scipy import ndimage
    near = ndimage.binary_dilation(occ, structure=np.ones((1, 3, 3, 3), bool))
    assert not (diff & ~near).any(), "a difference away from the surface"
    assert diff.sum() <= max(8, occ.sum() // 200), "%d of %d surface voxels differ" % (diff.sum(), occ.sum())
