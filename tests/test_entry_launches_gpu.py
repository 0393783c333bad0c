"""Kernel launches of every loss, mesh-op, vertex, NMR and voxel C entry point and branch: umr_launch_count() moves by
the number of kernels the accepted call launches (memsets are not counted).

Counts per call:
  sampler forward (C = 1..4, float32 / float64)      1
  sampler backward (float32, with or without image)  1
  sampler cells                                      1
  sampler backward deterministic / float64           1, +1 (the image gather) with grad_image
  IoU forward                                        2 (partial, finalize), every variant;  backward 1
  chamfer forward (D = 2 / 3)                        2 (one nearest-neighbour pass per direction)
  chamfer backward (float32)                         1 per distance gradient given
  chamfer backward deterministic / float64           2 (one gather per point set)
  TexCycle forward                                   float32 1, deterministic / float64 2, +1 (visibility bitmap) with
                                                     face_ids;  backward 1
  masked L1 forward (C = 1 / 3)                      float32 1, deterministic / float64 2;  backward 1
  loss head forward                                  float32 2, deterministic / float64 3;  backward 1
  part head forward                                  kld 2, mse 4 (float32 / float64);  backward 1
  texture image / load textures                      1 each
  Laplacian forward                                  float32 1, deterministic / float64 2;  backward 1
  flatten forward                                    float32 1, deterministic / float64 2
  flatten backward                                   float32 1, deterministic / float64 2 (terms, gather)
  dt barrier                                         2 (columns, rows)
  projection forward                                 1;  backward 2
  projection backward deterministic                  3, +1 (hypothesis sum) with grad_vertices and H > 1, +1 (camera
                                                     finalize) with grad_cams
  CorrLossChamfer forward                            1;  backward float32 1
  CorrLossChamfer backward deterministic / float64   1, +1 (gather) with grad_vertices
  NMR forward                                        2 (prep, z-buffer), +1 (shade) with any shaded output
  NMR texture gradient                               2 (prep, gradient), default and deterministic
  NMR face gradient                                  2 (prep, gradient), +1 (colour plane) with grad_rgb
  lighting forward                                   1;  backward 1, +1 (reduction) with grad_light
  voxelize                                           2 (fill, unpack), +1 (surface) with F > 0
"""
import ctypes

import pytest
import torch

from umr_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
N = 1 << 20          # elements of every buffer: far past what the small shapes below read or write
F32, F64 = torch.float32, torch.float64


_keep = []   # the buffers of the running test


def _hold(t):
    _keep.append(t)
    return t


def Rk(dt=F32):
    """A buffer of uniform [0, 1) values."""
    return _hold(torch.rand(N, dtype=dt, device=DEV)).data_ptr()


def Zk():
    """An int32 buffer of zeros: every index 0, every CSR table empty."""
    return _hold(torch.zeros(N, dtype=torch.int32, device=DEV)).data_ptr()


@pytest.fixture(autouse=True)
def _release():
    yield
    _keep.clear()


def launches(name, *args):
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.umr_launch_count()
    rc = getattr(lib, name)(*args, None)
    torch.cuda.synchronize()
    assert rc == 0, (name, rc)
    return lib.umr_launch_count() - n0


def _ws():
    return _hold(torch.zeros(N * 8, dtype=torch.uint8, device=DEV)).data_ptr()


B = 2


@pytest.mark.parametrize("C", [1, 2, 3, 4])
def test_sampler(C):
    H = W = 8
    for suffix, dt in (("", F32), ("_f64", F64)):
        assert launches("umr_bilinear_sample_forward" + suffix, Rk(dt), Rk(dt), Rk(dt), B, C, H, W, 50) == 1
        assert launches("umr_bilinear_sample_cells" + suffix, Rk(dt), Zk(), B, H, W, 50) == 1
    for gimg in (Rk(), None):
        assert launches("umr_bilinear_sample_backward", Rk(), Rk(), Rk(), Rk(), gimg, B, C, H, W, 50) == 1
    for suffix, dt in (("_deterministic", F32), ("_f64", F64)):
        for gimg, want in ((Rk(dt), 2), (None, 1)):
            assert launches("umr_bilinear_sample_backward" + suffix, Rk(dt), Rk(dt), Rk(dt), Rk(dt), gimg, B, C, H, W, 50,
                            Zk(), Zk()) == want


def test_iou():
    assert launches("umr_iou_forward", Rk(), 64, Rk(), Rk(), Rk(), Rk(), B, 64) == 2
    assert launches("umr_iou_forward_deterministic", Rk(), 64, Rk(), Rk(), Rk(), Rk(), B, 64, _ws()) == 2
    assert launches("umr_iou_forward_f64", Rk(F64), 64, Rk(F64), Rk(F64), Rk(F64), Rk(F64), B, 64, _ws()) == 2
    assert launches("umr_iou_backward", Rk(), Rk(), Rk(), Rk(), Rk(), B, 64) == 1
    assert launches("umr_iou_backward_f64", Rk(F64), Rk(F64), Rk(F64), Rk(F64), Rk(F64), B, 64) == 1


@pytest.mark.parametrize("D", [2, 3])
def test_chamfer(D):
    for suffix, dt in (("", F32), ("_f64", F64)):
        assert launches("umr_chamfer_forward" + suffix, Rk(dt), Rk(dt), Rk(dt), Rk(dt), Zk(), Zk(), B, 30, 20, D) == 2
    for gab, gba in ((Rk(), Rk()), (Rk(), None), (None, Rk()), (None, None)):
        want = (gab is not None) + (gba is not None)
        assert launches("umr_chamfer_backward", Rk(), Rk(), Zk(), Zk(), gab, gba, Rk(), Rk(), B, 30, 20, D) == want
    for suffix, dt in (("_deterministic", F32), ("_f64", F64)):
        assert launches("umr_chamfer_backward" + suffix, Rk(dt), Rk(dt), Zk(), Zk(), Rk(dt), Rk(dt), Rk(dt), Rk(dt), B, 30,
                        20, D) == 2


def test_texcycle():
    Fc, T2, P = 16, 4, 64
    vis = lambda: _hold(torch.ones(N, dtype=torch.uint8, device=DEV)).data_ptr()
    assert launches("umr_texcycle_forward", Rk(), Rk(), Rk(), vis(), Rk(), B, Fc, T2, P) == 2
    assert launches("umr_texcycle_forward", Rk(), Rk(), None, vis(), Rk(), B, Fc, T2, 0) == 1
    for suffix, dt in (("_deterministic", F32), ("_f64", F64)):
        assert launches("umr_texcycle_forward" + suffix, Rk(dt), Rk(dt), Rk(), vis(), Rk(dt), B, Fc, T2, P, _ws()) == 3
        assert launches("umr_texcycle_forward" + suffix, Rk(dt), Rk(dt), None, vis(), Rk(dt), B, Fc, T2, 0, _ws()) == 2
    for suffix, dt in (("", F32), ("_f64", F64)):
        assert launches("umr_texcycle_backward" + suffix, Rk(dt), Rk(dt), vis(), Rk(dt), Rk(dt), B, Fc, T2) == 1


@pytest.mark.parametrize("C", [1, 3])
def test_masked_l1(C):
    HW = 64
    assert launches("umr_masked_l1_forward", Rk(), C * HW, Rk(), HW, Rk(), Rk(), Rk(), B, C, HW) == 1
    assert launches("umr_masked_l1_forward_deterministic", Rk(), C * HW, Rk(), HW, Rk(), Rk(), Rk(), B, C, HW, _ws()) == 2
    assert launches("umr_masked_l1_forward_f64", Rk(F64), C * HW, Rk(F64), HW, Rk(F64), Rk(F64), Rk(F64), B, C, HW,
                    _ws()) == 2
    assert launches("umr_masked_l1_backward", Rk(), C * HW, Rk(), HW, Rk(), Rk(), Rk(), Rk(), Rk(), B, C, HW) == 1
    assert launches("umr_masked_l1_backward_f64", Rk(F64), C * HW, Rk(F64), HW, Rk(F64), Rk(F64), Rk(F64), Rk(F64), Rk(F64),
                    B, C, HW) == 1


def test_loss_head():
    HW = 64
    assert launches("umr_loss_head_forward", Rk(), Rk(), Rk(), Rk(), Rk(), Rk(), B, HW, 1.0, 1.0) == 2
    assert launches("umr_loss_head_forward_deterministic", Rk(), Rk(), Rk(), Rk(), Rk(), Rk(), B, HW, 1.0, 1.0, _ws()) == 3
    assert launches("umr_loss_head_forward_f64", *[Rk(F64) for _ in range(6)], B, HW, 1.0, 1.0, _ws()) == 3
    assert launches("umr_loss_head_backward", *[Rk() for _ in range(6)], B, HW, 1.0, 1.0) == 1
    assert launches("umr_loss_head_backward_f64", *[Rk(F64) for _ in range(6)], B, HW, 1.0, 1.0) == 1


@pytest.mark.parametrize("kld", [1, 0])
@pytest.mark.parametrize("dtype", [0, 1])
def test_part_head(kld, dtype):
    H = 16
    dt = F64 if dtype else F32
    maps = (ctypes.c_void_p * 4)(*[Rk(dt) for _ in range(4)])
    bs = (ctypes.c_int64 * 4)(*[H * H] * 4)
    ws = _ws()
    c0, segs, w = Rk(dt), Rk(dt), _hold(torch.ones(N, dtype=dt, device=DEV)).data_ptr()
    assert launches("umr_part_head_forward", maps, bs, c0, 8, segs, 8, w, Rk(dt), B, H, kld, dtype, ws) == (2 if kld else 4)
    assert launches("umr_part_head_backward", maps, bs, c0, 8, segs, 8, w, ws, Rk(dt), Rk(dt), B, H, kld, dtype) == 1


def test_mesh_ops():
    V, E = 12, 20
    assert launches("umr_create_texture_image", Rk(), Rk(), Rk(), 4, 4, 16, 16, 1e-5) == 1
    assert launches("umr_load_textures", Rk(), Rk(), Zk(), Rk(), 4, 4, 16, 16) == 1
    assert launches("umr_laplacian_forward", Rk(), Zk(), Zk(), Rk(), Rk(), Rk(), B, V) == 1
    assert launches("umr_laplacian_forward_deterministic", Rk(), Zk(), Zk(), Rk(), Rk(), Rk(), B, V, _ws()) == 2
    assert launches("umr_laplacian_forward_f64", Rk(F64), Zk(), Zk(), Rk(F64), Rk(F64), Rk(F64), B, V, _ws()) == 2
    assert launches("umr_laplacian_backward", Rk(), Zk(), Zk(), Rk(), Rk(), Rk(), B, V) == 1
    assert launches("umr_laplacian_backward_f64", Rk(F64), Zk(), Zk(), Rk(F64), Rk(F64), Rk(F64), B, V) == 1
    assert launches("umr_flatten_forward", Rk(), Zk(), Rk(), B, V, E, 1e-6) == 1
    assert launches("umr_flatten_forward_deterministic", Rk(), Zk(), Rk(), B, V, E, 1e-6, _ws()) == 2
    assert launches("umr_flatten_forward_f64", Rk(F64), Zk(), Rk(F64), B, V, E, 1e-6, _ws()) == 2
    assert launches("umr_flatten_backward", Rk(), Zk(), Rk(), Rk(), B, V, E, 1e-6) == 1
    assert launches("umr_flatten_backward_deterministic", Rk(), Zk(), Zk(), Zk(), Rk(), Rk(), B, V, E, 1e-6, _ws()) == 2
    assert launches("umr_flatten_backward_f64", Rk(F64), Zk(), Zk(), Zk(), Rk(F64), Rk(F64), B, V, E, 1e-6, _ws()) == 2
    assert launches("umr_dt_barrier", Rk(), Rk(), _ws(), B, 16, 16, 1.0) == 2


def _proj(H):
    p = _lib.UmrProjectParams()
    p.batch_size, p.num_vertices, p.num_faces, p.num_hypotheses = 2 * H, 12, 20, H
    p.offset_z, p.eye_z, p.viewing_scale = 5.0, 2.732, 1.0
    return p


@pytest.mark.parametrize("H", [1, 2])
def test_projection(H):
    p = ctypes.byref(_proj(H))
    assert launches("umr_project_faces_forward", Rk(), Rk(), Zk(), Rk(), Rk(), p) == 1
    for gv in (Rk(), None):
        for gc in (Rk(), None):
            assert launches("umr_project_faces_backward", Rk(), Rk(), Zk(), Rk(), Rk(), Rk(), gv, gc, p) == 2
            want = 3 + (gv is not None and H > 1) + (gc is not None)
            assert launches("umr_project_faces_backward_deterministic", Rk(), Rk(), Zk(), Rk(), Rk(), Rk(), gv, gc, p, Zk(),
                            Zk(), _ws()) == want


def test_corr_chamfer():
    NS, V = 4, 12
    tc = (ctypes.c_int32 * 4)(3, 3, 3, 3)
    ends = (ctypes.c_int32 * 4)(1, 2, 3, 4)
    for suffix, gather, dt, ct in (("", "_deterministic", F32, ctypes.c_float), ("_f64", "_f64", F64, ctypes.c_double)):
        tp = (ctypes.c_void_p * 4)(*[Rk(dt) for _ in range(4)])
        wt = (ct * 4)(1, 1, 0, 0)
        corr = lambda: (Rk(dt), 3 * V, Rk(dt), Zk(), tp, tc, ends, wt)
        assert launches("umr_corr_chamfer_forward" + suffix, *corr(), Rk(dt), Zk(), Rk(dt), B, NS) == 1
        if suffix == "":
            assert launches("umr_corr_chamfer_backward", *corr(), Rk(), Zk(), Rk(), Rk(), Rk(), Rk(), B, NS, V) == 1
        for gv, want in ((Rk(dt), 2), (None, 1)):
            assert launches("umr_corr_chamfer_backward" + gather, *corr(), Rk(dt), Zk(), Rk(dt), Rk(dt), gv, Rk(dt), B, NS, V,
                            Zk(), Zk(), _ws()) == want


def _nmr(fill_back=1, light_dir=0.5):
    p = _lib.UmrNmrParams()
    p.batch_size, p.num_vertices, p.num_faces, p.texture_res = B, 10, 4, 3
    p.image_size, p.anti_aliasing, p.fill_back, p.shared_textures = 16, 1, fill_back, 1
    p.eye_z, p.near_plane, p.far_plane = 2.732, 0.1, 100.0
    p.light_intensity_ambient, p.light_intensity_directional = 0.5, light_dir
    return p


def test_nmr():
    p = ctypes.byref(_nmr())
    for shaded, want in (((Rk(), Rk(), Rk()), 3), ((Rk(), None, None), 3), ((None, None, None), 2)):
        assert launches("umr_nmr_forward", Rk(), Zk(), Rk(), Zk(), Rk(), *shaded, p, _ws()) == want
    for name in ("umr_nmr_backward_textures", "umr_nmr_backward_textures_deterministic"):
        assert launches(name, Rk(), Zk(), Zk(), Rk(), Rk(), p, _ws()) == 2
    q = ctypes.byref(_nmr(fill_back=0, light_dir=0.0))
    for grgb, want in ((Rk(), 3), (None, 2)):
        assert launches("umr_nmr_backward_faces", Rk(), Zk(), Zk(), Rk(), grgb, Rk(), Rk(), Rk(), q, 1e-8, _ws()) == want


@pytest.mark.parametrize("dtype", [0, 1])
def test_lighting(dtype):
    dt = F64 if dtype else F32
    p = _lib.UmrNmrLightParams()
    p.batch_size, p.num_faces, p.texture_res, p.dtype = B, 3, 2, dtype
    p.intensity_ambient, p.intensity_directional = 0.5, 0.5
    p = ctypes.byref(p)
    assert launches("umr_nmr_lighting_forward", *[Rk(dt) for _ in range(6)], p) == 1
    for gl, want in ((Rk(dt), 2), (None, 1)):
        assert launches("umr_nmr_lighting_backward", *[Rk(dt) for _ in range(6)], Rk(dt), Rk(dt), gl, p, _ws()) == want


@pytest.mark.parametrize("vs", [64, 65])
@pytest.mark.parametrize("F", [0, 6])
def test_voxelize(vs, F):
    vox = _hold(torch.zeros(B * vs ** 3, dtype=torch.int32, device=DEV)).data_ptr()
    faces = Rk() if F else None
    assert launches("umr_voxelize", faces, 0, vox, B, F, vs, 1.0, _ws()) == (1 if F else 0) + 2
