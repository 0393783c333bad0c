"""CPU checks of `voxelization`: the numpy oracle on hand-computed meshes and against a literal transcription of the
reference's four kernels and host loop, the word-parallel run fill exhaustively at 16 bits, `save_voxel` / `load_obj`,
and the refusals that need no GPU."""
import ctypes
import math

import numpy as np
import pytest
import torch

import voxel_oracle as vo
from umr_b200 import _lib, ops, synth
import umr_b200.soft_renderer as sr
from umr_b200.soft_renderer.functional import obj_io


# ------------------------------------------------------------------------------------------------------------------
# run fill along the packed axis
# ------------------------------------------------------------------------------------------------------------------
def _naive_fill(s, e, bits):
    for _ in range(bits):
        s = s | (((s << np.uint64(1)) | (s >> np.uint64(1))) & e)
    return s


def test_run_fill_exhaustive_16bit():
    """Every (seeds, empty) pair with seeds ⊆ empty over 16 bits (3^16 pairs): fill_runs == bit-by-bit fill."""
    bits = 16
    pw = 3 ** np.arange(bits, dtype=np.int64)
    chunk = 3 ** 12
    for start in range(0, 3 ** bits, chunk):
        n = np.arange(start, start + chunk, dtype=np.int64)
        digit = (n[:, None] // pw[None, :]) % 3  # 0: occupied, 1: empty, 2: empty seed
        weights = (np.uint64(1) << np.arange(bits, dtype=np.uint64))[None, :]
        e = ((digit >= 1).astype(np.uint64) * weights).sum(1).astype(np.uint64)
        s = ((digit == 2).astype(np.uint64) * weights).sum(1).astype(np.uint64)
        np.testing.assert_array_equal(vo.fill_runs(s, e, bits), _naive_fill(s, e, bits))


# ------------------------------------------------------------------------------------------------------------------
# the oracle on hand-computed meshes (normalize=True: coordinates are voxel units)
# ------------------------------------------------------------------------------------------------------------------
def _vox(faces, vs, dtype=np.float32):
    return vo.voxelization_np(np.asarray(faces, dtype)[None], vs, normalize=True)[0]


def test_axis_aligned_triangle():
    tri = [[[0.5, 0.5, 1.5], [2.5, 0.5, 1.5], [0.5, 2.5, 1.5]]]
    got = _vox(tri, 4)
    # the z-projection passes columns (1,1), (1,2), (2,1); each marks itself and its (-1, 0), (0, -1), (-1, -1)
    # neighbours at z = floor(1.5); the other two projections have det == 0; the vertices add nothing new
    want = np.zeros((4, 4, 4), np.int32)
    for c0, c1 in [(0, 0), (0, 1), (0, 2), (1, 0), (1, 1), (1, 2), (2, 0), (2, 1)]:
        want[c0, c1, 1] = 1
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_closed_cube_is_solid(dtype):
    got = _vox(vo.box_faces(0.5, 5.5), 8, dtype)
    want = np.zeros((8, 8, 8), np.int32)
    want[:6, :6, :6] = 1
    np.testing.assert_array_equal(got, want)


def test_open_cube_keeps_its_cavity():
    got = _vox(vo.box_faces(0.5, 5.5, open_side=(2, 1)), 8)
    want = np.zeros((8, 8, 8), np.int32)
    want[:6, :6, :6] = 1
    want[1:5, 1:5, 1:6] = 0  # open at the top: the cavity reaches the outside through z = 5 -> 6
    np.testing.assert_array_equal(got, want)


def test_nested_boxes_fill_the_gap():
    faces = np.concatenate([vo.box_faces(0.5, 9.5), vo.box_faces(3.5, 6.5)])
    got = _vox(faces, 12)
    want = np.zeros((12, 12, 12), np.int32)
    want[:10, :10, :10] = 1
    np.testing.assert_array_equal(got, want)


def test_nonfinite_marks_nothing():
    tri = np.array([[[0.5, 0.5, np.nan], [2.5, 0.5, 1.5], [0.5, 2.5, 1.5]],
                    [[np.inf, 1.0, 1.0], [2.0, 2.0, 2.0], [1.0, 3.0, 1.0]]])
    got = _vox(tri, 4)
    # only finite vertices are marked: (2,0,1), (0,2,1), (2,2,2), (1,3,1)
    want = np.zeros((4, 4, 4), np.int32)
    for c in [(2, 0, 1), (0, 2, 1), (2, 2, 2), (1, 3, 1)]:
        want[c] = 1
    np.testing.assert_array_equal(got, want)


# ------------------------------------------------------------------------------------------------------------------
# literal transcription of the reference (voxelization_cuda_kernel.cu:30-190, functional/voxelization.py:9-58)
# ------------------------------------------------------------------------------------------------------------------
def _ref_sub1(faces, vs):
    dt = faces.dtype.type
    bs, nf = faces.shape[:2]
    vox = np.zeros((bs, vs, vs, vs), np.int32)
    for bn in range(bs):
        for x in range(vs):
            for y in range(vs):
                for fn in range(nf):
                    face = faces[bn, fn].reshape(9)
                    y1d, x1d, z1d = face[3] - face[0], face[4] - face[1], face[5] - face[2]
                    y2d, x2d, z2d = face[6] - face[0], face[7] - face[1], face[8] - face[2]
                    ypd, xpd = dt(y) - face[0], dt(x) - face[1]
                    det = x1d * y2d - x2d * y1d
                    if det == 0:
                        continue
                    t1 = (y2d * xpd - x2d * ypd) / det
                    t2 = (-y1d * xpd + x1d * ypd) / det
                    if t1 < 0 or t2 < 0 or 1 < t1 + t2:
                        continue
                    zf = np.floor(t1 * z1d + t2 * z2d + face[2])
                    if not np.isfinite(zf):  # undefined in the reference (int)floor(NaN): defined as no mark
                        continue
                    zi = int(zf)
                    for yi, xi in ((y, x), (y - 1, x), (y, x - 1), (y - 1, x - 1)):
                        if 0 <= yi < vs and 0 <= xi < vs and 0 <= zi < vs:
                            vox[bn, yi, xi, zi] = 1
    return vox


def _ref_voxelization(faces, size, normalize=False):
    faces = faces.copy()
    if not normalize:
        faces = (faces * faces.dtype.type(size)).astype(faces.dtype)
    vs = size
    grids = []
    for dim in range(3):
        f = faces
        if dim == 0:
            f = np.ascontiguousarray(faces[..., [2, 1, 0]])
        elif dim == 1:
            f = np.ascontiguousarray(faces[..., [0, 2, 1]])
        grids.append(np.swapaxes(_ref_sub1(f, vs), dim + 1, 3))
    v3 = np.zeros_like(grids[0])
    for bn in range(faces.shape[0]):  # voxelize_sub2
        for fn in range(faces.shape[1]):
            for k in range(3):
                c = np.floor(faces[bn, fn, k])
                if not np.isfinite(c).all():
                    continue
                yi, xi, zi = (int(t) for t in c)
                if 0 <= yi < vs and 0 <= xi < vs and 0 <= zi < vs:
                    v3[bn, yi, xi, zi] = 1
    voxels = ((grids[0] + grids[1] + grids[2] + v3) > 0).astype(np.int32)
    visible = np.zeros_like(voxels)
    for bn in range(voxels.shape[0]):  # sub3
        for y in range(vs):
            for x in range(vs):
                for z in range(vs):
                    if (y in (0, vs - 1) or x in (0, vs - 1) or z in (0, vs - 1)) and voxels[bn, y, x, z] == 0:
                        visible[bn, y, x, z] = 1
    total = visible.sum()
    while True:  # sub4, in place in index order (one schedule of the reference's racy sweep)
        for bn in range(voxels.shape[0]):
            for y in range(1, vs - 1):
                for x in range(1, vs - 1):
                    for z in range(1, vs - 1):
                        if voxels[bn, y, x, z] == 0 and visible[bn, y, x, z] == 0:
                            if (visible[bn, y - 1, x, z] or visible[bn, y + 1, x, z] or visible[bn, y, x - 1, z]
                                    or visible[bn, y, x + 1, z] or visible[bn, y, x, z - 1] or visible[bn, y, x, z + 1]):
                                visible[bn, y, x, z] = 1
        if visible.sum() == total:
            break
        total = visible.sum()
    return 1 - visible


def _soup(rng, F, vs, dtype):
    f = rng.uniform(-0.2, 1.2, size=(1, F, 3, 3))
    f[0, 0, 1] = f[0, 0, 0]                                       # zero-area face (det == 0 on every axis)
    f[0, 1, 2] = f[0, 1, 0] + 1e-6 * (f[0, 1, 1] - f[0, 1, 0])    # sliver
    f[0, 2] = rng.uniform(1.5, 3.0, size=(3, 3))                  # wholly outside
    return f.astype(dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("vs", [1, 2, 5, 8])
def test_oracle_equals_reference_transcription(dtype, vs):
    rng = np.random.default_rng(vs)
    meshes = [_soup(rng, 8, vs, dtype)]
    v, f = synth.icosphere(1)
    verts = synth.bird_like(v, rng, 1) * 0.45 + 0.5
    meshes.append(verts[:, f].astype(dtype))
    meshes.append((vo.box_faces(0.1, 0.8)[None]).astype(dtype))
    for m in meshes:
        np.testing.assert_array_equal(vo.voxelization_np(m, vs), _ref_voxelization(m, vs))
    m = meshes[1] * dtype(vs)
    np.testing.assert_array_equal(vo.voxelization_np(m, vs, normalize=True), _ref_voxelization(m, vs, normalize=True))


# ------------------------------------------------------------------------------------------------------------------
# save_voxel / load_obj / Mesh plumbing
# ------------------------------------------------------------------------------------------------------------------
def test_save_voxel_format(tmp_path):
    vox = torch.zeros(2, 3, 4, dtype=torch.int32)
    vox[0, 0, 0] = 1
    vox[1, 2, 3] = 1
    vox[0, 1, 2] = 1
    vox[1, 0, 1] = 2  # only voxels equal to 1 are written
    fn = str(tmp_path / "v.obj")
    sr.functional.save_voxel(fn, vox)
    lines = open(fn).read().split("\n")
    assert lines[:3] == ["# v.obj", "#", ""]
    assert lines[3:] == ["v 0.00000000 0.00000000 0.00000000", "v 0.00000000 0.33333334 0.50000000",
                         "v 0.50000000 0.66666669 0.75000000", "", ""]


def test_load_obj_parses_and_triangulates(tmp_path, monkeypatch):
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)  # the parser, without a GPU
    fn = tmp_path / "m.obj"
    fn.write_text("# quad + triangle\nv 0 0 0\nv 2 0 0\nv 2 1 0\nv 0 1 0.5\n\nf 1/1 2/2 3/3 4/4\nf 1 3 4\n")
    v, f = sr.functional.load_obj(str(fn))
    assert v.dtype == torch.float32 and f.dtype == torch.int32
    np.testing.assert_array_equal(v.numpy(), [[0, 0, 0], [2, 0, 0], [2, 1, 0], [0, 1, 0.5]])
    np.testing.assert_array_equal(f.numpy(), [[0, 1, 2], [0, 2, 3], [0, 2, 3]])
    vn, _ = sr.functional.load_obj(str(fn), normalization=True)
    np.testing.assert_allclose(vn.numpy().max(0) + vn.numpy().min(0), 0, atol=1e-6)
    mesh = sr.Mesh.from_obj(str(fn))
    np.testing.assert_array_equal(mesh.vertices[0].numpy(), v.numpy())
    np.testing.assert_array_equal(mesh.faces[0].numpy(), f.numpy())
    with pytest.raises(ValueError):
        sr.functional.load_obj(str(fn), texture_type="nope")


def test_refusals_without_gpu():
    faces = torch.zeros(1, 2, 3, 3)
    with pytest.raises(TypeError):
        sr.functional.voxelization(faces, 8)
    with pytest.raises(ValueError):
        ops.voxelize(faces, 0)
    mesh = sr.Mesh(torch.zeros(3, 3), torch.tensor([[0, 1, 2]], dtype=torch.int32))
    for bad in (0, 1):
        with pytest.raises(ValueError):
            mesh.voxelize(bad)


def test_c_abi_refusals_without_gpu():
    """Argument checks return before any CUDA call."""
    lib = _lib.load()
    p = ctypes.c_void_p(256)
    assert lib.umr_voxelize(p, 0, p, 1, 1, 0, 1.0, p, None) == -2          # size < 1: UMR_ERR_BAD_ARG
    assert lib.umr_voxelize(p, 2, p, 1, 1, 8, 1.0, p, None) == -2          # unknown dtype
    assert lib.umr_voxelize(p, 0, ctypes.c_void_p(260), 1, 1, 8, 1.0, p, None) == -2  # voxels not 16-byte aligned
    vs = math.ceil(2 ** (31 / 3))                                           # B * vs^3 >= 2^31: UMR_ERR_TOO_LARGE
    assert lib.umr_voxelize(p, 0, p, 1, 1, vs, 1.0, p, None) == -3
    assert lib.umr_voxelize(p, 0, p, 2, 1, 1024, 1.0, p, None) == -3
    assert lib.umr_voxelize_workspace_bytes(1, vs) == 0
    assert lib.umr_voxelize_workspace_bytes(2, 64) >= 256 + 2 * 2 * 64 ** 3 // 8
    assert lib.umr_version() == 204
