"""The SCOPS semantic template (csrc/semantic_template.cu, DESIGN.md §18) against the numpy restatement
(tests/semantic_template_oracle.py) across the accepted input range.

The averaging pass: distances within the stated rounding bound of float64, the selection in the (distance, index) order
of the returned distances, the accumulator and the mean bitwise the restatement's float32 sums.  The labelling pass:
texel, face and vertex labels and the part lists exactly the restatement's.  Then the round trip through the files the
train_s2 losses read."""
import numpy as np
import pytest
import torch

import semantic_template_oracle as sto
from umr_b200 import _lib, ops, synth
from umr_b200.nnutils import loss_utils
from umr_b200.raster import _stream_ptr
from umr_b200.utils import semantic_template as st

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NUM_SYM, T = 624, 6


def _t(a):
    return torch.as_tensor(np.ascontiguousarray(a), device=DEV)


def _batches(rng, NB, B, C, S, H, W, spread=1.0):
    return [(sto.part_segs(rng, B, C, S), sto.uvimage_pred(rng, B, H, W, spread)) for _ in range(NB)]


def check_average(batches, exemplar, k):
    """Runs every batch through UVPartAverage against the restatement.  Returns the restatement's avg_prob."""
    avg = st.UVPartAverage(_t(exemplar), k)
    acc = np.zeros_like(exemplar)
    C, H, W = exemplar.shape
    for segs, uv in batches:
        dist, sel = avg.add(_t(segs), _t(uv))
        dist, sel = dist.cpu().numpy(), sel.cpu().numpy()
        parts = sto.uv_parts(segs, uv)
        d64 = sto.distances(parts, exemplar)
        np.testing.assert_array_equal(np.isnan(dist), np.isnan(d64))
        fin = ~np.isnan(d64)
        assert (np.abs(dist[fin] - d64[fin]) <= sto.dist_bound(d64[fin], C, H, W)).all()
        np.testing.assert_array_equal(sel, sto.select(dist, k))
        acc = sto.accumulate(acc, parts, sel)
        np.testing.assert_array_equal(avg.acc.cpu().numpy(), acc)
    want = sto.mean(acc, k * len(batches))
    np.testing.assert_array_equal(avg.mean().cpu().numpy(), want)
    return want


@pytest.mark.parametrize("B,C,k", [(5, 5, 5), (33, 5, 5), (33, 2, 7), (33, 32, 5), (1024, 2, 5), (1024, 2, 1024)])
def test_average_matches_the_restatement(B, C, k):
    rng = np.random.default_rng(B * 100 + C)
    H, W, S = (37, 75, 29) if B < 1024 else (9, 13, 7)
    batches = _batches(rng, 2, B, C, S, H, W, spread=1.3)     # UV past [-1, 1]: zero padding
    check_average(batches, sto.part_segs(rng, 1, C, H)[0][:, :, :1].repeat(W, axis=2) * 0.5 + 0.1, k)


def test_cub_shape_average():
    rng = np.random.default_rng(1)
    batches = _batches(rng, 2, 32, 5, 64, 128, 256)
    check_average(batches, sto.uv_parts(*batches[0])[3], 5)


def test_nan_inputs_rank_last():
    rng = np.random.default_rng(2)
    B, C, S, H, W = 8, 5, 17, 11, 21
    segs, uv = _batches(rng, 1, B, C, S, H, W)[0]
    exemplar = sto.uv_parts(segs, uv)[0]
    segs[1, 2, :, 4:6] = np.nan             # image 1: a NaN band every row of UV pixels samples
    uv[4, 0, 5, 6] = np.nan                 # image 4: one NaN UV pixel
    uv[6, 1, 0, 0] = np.nan
    segs[7, :] = np.nan                     # image 7: every sample NaN
    nan_sel = None
    for k in (4, 5):                        # 4 finite images: k = 5 selects a NaN one
        avg = st.UVPartAverage(_t(exemplar), k)
        dist, sel = avg.add(_t(segs), _t(uv))
        dist, sel = dist.cpu().numpy(), sel.cpu().numpy()
        assert np.isnan(dist[[1, 4, 6, 7]]).all() and not np.isnan(dist[[0, 2, 3, 5]]).any()
        np.testing.assert_array_equal(sel, sto.select(dist, k))
        acc = sto.accumulate(np.zeros_like(exemplar), sto.uv_parts(segs, uv), sel)
        np.testing.assert_array_equal(avg.acc.cpu().numpy(), acc)
        nan_sel = sel
    assert nan_sel[-1] == 1 and np.isnan(avg.acc.cpu().numpy()).any()


GUARD = 64


def _guarded(n, dtype, fill):
    return torch.full((2 * GUARD + n,), fill, device=DEV, dtype=dtype)


def _inside(buf, n):
    return buf[GUARD:GUARD + n]


def _untouched(buf, n, fill):
    return bool((buf[:GUARD] == fill).all() and (buf[GUARD + n:] == fill).all())


def test_average_guard_bands_and_launch_counts():
    rng = np.random.default_rng(3)
    B, C, S, H, W, k = 9, 3, 13, 7, 45, 4
    segs, uv = _batches(rng, 1, B, C, S, H, W)[0]
    exemplar = sto.uv_parts(segs, uv)[2] * np.float32(0.9)
    lib = _lib.load()
    N = H * W
    ws_n = lib.umr_st_average_workspace_bytes(B, H, W) // 4
    ws, dist = _guarded(ws_n, torch.float32, -7.0), _guarded(B, torch.float32, -7.0)
    sel, acc = _guarded(k, torch.int32, -7), _guarded(C * N, torch.float32, 0.0)
    acc[:GUARD] = -7.0
    acc[GUARD + C * N:] = -7.0
    s, u, e = _t(segs), _t(uv), _t(exemplar)
    torch.cuda.synchronize()
    before = lib.umr_launch_count()
    assert lib.umr_st_average_add(s.data_ptr(), u.data_ptr(), e.data_ptr(), B, C, S, H, W, k, _inside(ws, ws_n).data_ptr(),
                                  _inside(dist, B).data_ptr(), _inside(sel, k).data_ptr(), _inside(acc, C * N).data_ptr(),
                                  _stream_ptr(DEV)) == 0
    assert lib.umr_launch_count() - before == 2
    avg = _guarded(C * N, torch.float32, -7.0)
    assert lib.umr_st_average_mean(_inside(acc, C * N).data_ptr(), C, H, W, k, _inside(avg, C * N).data_ptr(),
                                   _stream_ptr(DEV)) == 0
    assert lib.umr_launch_count() - before == 3
    torch.cuda.synchronize()
    for buf, n, fill in ((ws, ws_n, -7.0), (dist, B, -7.0), (sel, k, -7), (acc, C * N, -7.0), (avg, C * N, -7.0)):
        assert _untouched(buf, n, fill)
    got_sel = _inside(sel, k).cpu().numpy()
    np.testing.assert_array_equal(got_sel, sto.select(_inside(dist, B).cpu().numpy(), k))
    want = sto.accumulate(np.zeros((C, H, W), np.float32), sto.uv_parts(segs, uv), got_sel)
    np.testing.assert_array_equal(_inside(acc, C * N).cpu().numpy().reshape(C, H, W), want)
    np.testing.assert_array_equal(_inside(avg, C * N).cpu().numpy().reshape(H, W, C), sto.mean(want, k))


def test_average_is_bitwise_repeatable_and_never_syncs():
    rng = np.random.default_rng(4)
    batches = [(_t(s), _t(u)) for s, u in _batches(rng, 3, 32, 5, 64, 64, 128)]
    exemplar = _t(sto.part_segs(rng, 1, 5, 64)[0][:, :, :64].repeat(2, axis=2))
    outs = []
    for _ in range(2):
        avg = st.UVPartAverage(exemplar)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            res = [avg.add(s, u) for s, u in batches]
            m = avg.mean()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        outs.append((res, m))
    for (d0, s0), (d1, s1) in zip(outs[0][0], outs[1][0]):
        assert torch.equal(d0, d1) and torch.equal(s0, s1)
    assert torch.equal(outs[0][1], outs[1][1])


def test_several_adds_capture_in_a_cuda_graph():
    rng = np.random.default_rng(5)
    batches = [(_t(s), _t(u)) for s, u in _batches(rng, 3, 16, 5, 32, 32, 64)]
    exemplar = _t(sto.part_segs(rng, 1, 5, 32)[0].repeat(2, axis=2))
    eager = st.UVPartAverage(exemplar)
    for s, u in batches:
        eager.add(s, u)
    captured = st.UVPartAverage(exemplar)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        sels = [captured.add(s, u)[1] for s, u in batches]
    assert not captured.acc.any()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured.acc, eager.acc) and torch.equal(captured.mean(), eager.mean())
    assert all(s.shape == (5,) for s in sels)


# ---------------------------------------------------------------------------------------------------------------------
# the labelling pass
# ---------------------------------------------------------------------------------------------------------------------
def _check_labels(avg_prob, sampler, faces, nsym, num_vertices=None):
    tpl = st.semantic_template(_t(avg_prob), _t(sampler[None]), _t(faces.astype(np.int64)), nsym, num_vertices)
    want = sto.label(avg_prob, sampler, faces, nsym, num_vertices)
    for name in ("label_image", "texel_labels", "face_labels", "vertex_labels"):
        np.testing.assert_array_equal(getattr(tpl, name).cpu().numpy(), want[name], err_msg=name)
    C = avg_prob.shape[2]
    assert len(tpl.part_vertices) == C - 1
    for got, ref in zip(tpl.part_vertices, want["part_vertices"]):
        assert got.dtype == torch.int64
        np.testing.assert_array_equal(got.cpu().numpy(), ref)
    assert tuple(tpl.stex_one_hot.shape) == (1, faces.shape[0], sampler.shape[1], C)
    return tpl


def _cub_template(tex_size=T):
    v, f = synth.icosphere(3)
    return v, f, sto.uv_sampler(v, f[:f.shape[0] - NUM_SYM], tex_size)


@pytest.mark.parametrize("tex_size", [T, 1])
def test_cub_template_labels_match_the_restatement(tex_size):
    rng = np.random.default_rng(6)
    _, faces, sampler = _cub_template(tex_size)
    avg = check_average(_batches(rng, 2, 16, 5, 64, 128, 256), sto.part_segs(rng, 1, 5, 128)[0].repeat(2, axis=2), 5)
    tpl = _check_labels(avg, sampler, faces, NUM_SYM)
    assert (tpl.vertex_labels >= 0).all()


@pytest.mark.parametrize("C", [2, 32])
def test_channel_counts_and_ties(C):
    rng = np.random.default_rng(7)
    _, faces, sampler = _cub_template()
    avg = rng.random((37, 75, C)).astype(np.float32)
    avg = np.round(avg * 4) / 4                      # many exact channel ties
    avg[3, :7, C // 2] = np.nan                      # NaN channels win where they appear
    _check_labels(avg.astype(np.float32), sampler, faces, NUM_SYM)


def test_unreferenced_vertex_one_face_vertex_and_repeated_corner():
    v, f = synth.icosphere(2)
    faces = np.where(f >= 5, f + 1, f)                                  # vertex 5: on no face
    V = v.shape[0] + 1
    extra = np.array([[0, 1, V], [2, 2, 3]])                            # vertex V: on one face; a repeated corner
    faces = np.concatenate([faces, extra])
    rng = np.random.default_rng(8)
    sampler = rng.uniform(-1.2, 1.2, (faces.shape[0] - 1, 4, 2)).astype(np.float32)
    avg = sto.part_segs(rng, 1, 5, 24)[0].transpose(1, 2, 0).copy()
    tpl = _check_labels(avg, sampler, faces, 1, num_vertices=V + 1)
    assert int(tpl.vertex_labels[5]) == -1 and int(tpl.vertex_labels[V]) == int(tpl.face_labels[-2])
    assert all(5 not in p.tolist() for p in tpl.part_vertices)


def test_label_guard_bands_and_launch_counts():
    rng = np.random.default_rng(9)
    _, faces, sampler = _cub_template()
    H, W, C = 17, 33, 5
    avg = _t(rng.random((H, W, C)).astype(np.float32))
    ft = _t(faces.astype(np.int64))
    V, F, Fs, T2 = 642, faces.shape[0], sampler.shape[0], sampler.shape[1]
    rowptr, corners = ops.device_incidence(ft, V)
    img, tex = _guarded(H * W, torch.uint8, 77), _guarded(F * T2, torch.int32, -9)
    face, vert = _guarded(F, torch.int32, -9), _guarded(V, torch.int32, -9)
    uvs = _t(sampler)
    lib = _lib.load()
    torch.cuda.synchronize()
    before = lib.umr_launch_count()
    assert lib.umr_st_labels(avg.data_ptr(), H, W, C, uvs.data_ptr(), Fs, T2, NUM_SYM, rowptr.data_ptr(),
                             corners.data_ptr(), V, _inside(img, H * W).data_ptr(), _inside(tex, F * T2).data_ptr(),
                             _inside(face, F).data_ptr(), _inside(vert, V).data_ptr(), _stream_ptr(DEV)) == 0
    assert lib.umr_launch_count() - before == 3
    torch.cuda.synchronize()
    for buf, n, fill in ((img, H * W, 77), (tex, F * T2, -9), (face, F, -9), (vert, V, -9)):
        assert _untouched(buf, n, fill)
    want = sto.label(avg.cpu().numpy(), sampler, faces, NUM_SYM)
    np.testing.assert_array_equal(_inside(tex, F * T2).cpu().numpy().reshape(F, T2), want["texel_labels"])
    np.testing.assert_array_equal(_inside(vert, V).cpu().numpy(), want["vertex_labels"])
    # the Python call: the same three launches
    before = lib.umr_launch_count()
    st.semantic_template(avg, uvs[None], ft, NUM_SYM, V)
    assert lib.umr_launch_count() - before == 3


def test_faces_outside_the_vertex_range_are_refused():
    _, faces, sampler = _cub_template()
    with pytest.raises(ValueError, match="faces must index vertices"):
        st.semantic_template(_t(np.ones((8, 16, 5), np.float32)), _t(sampler[None]), _t(faces.astype(np.int64)),
                             NUM_SYM, 600)


# ---------------------------------------------------------------------------------------------------------------------
# round trip through the files train_s2's losses read
# ---------------------------------------------------------------------------------------------------------------------
def test_saved_template_feeds_the_train_s2_losses(tmp_path):
    rng = np.random.default_rng(10)
    verts, faces, sampler = _cub_template()
    avg = st.UVPartAverage(_t(sto.part_segs(rng, 1, 5, 128)[0].repeat(2, axis=2)))
    for segs, uv in _batches(rng, 2, 16, 5, 64, 128, 256):
        avg.add(_t(segs), _t(uv))
    avg_prob = avg.mean()
    uvs = _t(sampler[None])
    tpl = st.semantic_template(avg_prob, uvs, _t(faces.astype(np.int64)), NUM_SYM)
    st.save_semantic_template(str(tmp_path), avg_prob, tpl)
    np.testing.assert_array_equal(np.load(tmp_path / "semantic_prob.npy"), avg_prob.cpu().numpy())

    B, IS = 4, 64
    from_files = loss_utils.part_matching_loss(str(tmp_path), uvs, NUM_SYM, im_size=IS, batch_size=B, tex_size=T).to(DEV)
    from_tensor = loss_utils.part_matching_loss(None, None, 0, im_size=IS, batch_size=B, tex_size=T,
                                                stex_one_hot=tpl.stex_one_hot).to(DEV)
    a, b = dict(from_files.named_buffers()), dict(from_tensor.named_buffers())
    assert set(a) == set(b)
    for name in a:
        assert a[name].dtype == b[name].dtype and torch.equal(a[name], b[name]), name

    corr = loss_utils.CorrLossChamfer(str(tmp_path), IS)
    head, neck, back, belly = tpl.part_vertices
    for got, want in ((corr.head_vertices, head), (corr.neck_vertices, neck), (corr.back_vertices, back),
                      (corr.belly_vertices, belly)):
        assert torch.equal(got, want.cpu())

    # one train_s2-shaped step with both semantic losses built from the files
    vs = torch.from_numpy(synth.bird_like(verts, rng, B)).to(DEV).requires_grad_(True)
    cams = torch.from_numpy(synth.cameras(rng, B)).to(DEV)
    fs = _t(faces.astype(np.int64))[None].repeat(B, 1, 1)
    part_segs = _t(sto.part_segs(rng, B, 5, IS))
    points = [_t(p) for p in synth.part_points(rng, B, sizes=(10, 10, 30, 30))]
    part_loss, _ = from_files(vs, fs, cams, part_segs)
    corr_loss, _ = corr(points[0], points[3], points[1], points[2], vs, cams)
    (part_loss + corr_loss).backward()
    assert torch.isfinite(part_loss) and torch.isfinite(corr_loss)
    assert torch.isfinite(vs.grad).all() and vs.grad.abs().sum() > 0
