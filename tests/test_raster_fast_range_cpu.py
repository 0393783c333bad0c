"""The fast-path scenes of test_raster_fast_range_gpu.py have the properties they claim (no GPU): tile-list segment
lengths either side of LCAP and FWD4_CAP, box edges on the k_raster_fwd4 tile and coarse-bin boundaries, boxes over two
coarse bins, saved records per tile, the face window the recompute fallback crosses and the block cursor of the
16x16-tile forward (raster_range_scenes.fwd3_blocks_wanted, which the GPU test asserts against the pair buffer's header)."""
import numpy as np
import pytest

import raster_range_scenes as rs

F32 = np.float32


@pytest.mark.parametrize("S", [34])
@pytest.mark.parametrize("n", rs.LIST_LENGTHS)
def test_tile_list_segments(n, S):
    fv, _ = rs.crowd_all(S, F32, seed=n + S, F=n)
    box = rs.boxes(fv[0], F32)
    seg = rs.fwd3_segments(box, S)
    # every face is listed, in windows of LCAP coarse entries; a face of one pixel is one pair block
    assert [c for c, _ in seg] == [min(rs.LCAP, n - w) for w in range(0, n, rs.LCAP)]
    assert all(c == b for c, b in seg)
    assert rs.fwd3_blocks_wanted(fv, S) == n + 2 * len(seg)
    want = {511: [511], 512: [512], 513: [512, 1], 1535: [512, 512, 511], 1536: [512] * 3, 1537: [512] * 3 + [1]}
    if n in want:
        assert [c for c, _ in seg] == want[n]
    # the coarse bin of tile (0, 0) lists all n faces: below, at and above k_raster_fwd4's FWD4_CAP
    assert int(rs.tile_hits(box, S, 0, 0, F32, rs.CB).sum()) == n
    for tx in range((S + 15) // 16):
        for ty in range((S + 15) // 16):
            if tx or ty:
                assert not rs.tile_hits(box, S, tx, ty, F32).any()


@pytest.mark.parametrize("S", [1, 2, 17, 31, 33, 18, 34, 66])
def test_fast_edges(S):
    fv, _, meta = rs.edges(S, F32, fast=True)
    box = rs.boxes(fv[0], F32)
    targets = rs.edge_targets(S, fast=True)
    assert {i for _, i, _ in meta} == set(targets)
    for f, (side, i, d) in enumerate(meta):
        assert np.sign(box[f, side] - rs.pixel_centre(i, S, F32)) == d
    if S > rs.CB:
        assert {31, 32, 63, 64} <= set(targets)
        over = [f for f in range(fv.shape[1]) if rs.tile_hits(box[f:f + 1], S, 0, 0, F32, rs.CB)[0]
                and (rs.tile_hits(box[f:f + 1], S, 1, 0, F32, rs.CB)[0] or rs.tile_hits(box[f:f + 1], S, 0, 1, F32, rs.CB)[0])]
        on_bin_edge = [f for f, (side, i, d) in enumerate(meta) if i in (63, 64) and d == 0]
        assert len(on_bin_edge) >= 4 and len(set(on_bin_edge) & set(over)) >= 2 and len(over) >= 8
        print("S=%d: %d boxes over two coarse bins, %d with an edge on pixel 63 or 64 (%d of them over two bins)"
              % (S, len(over), len(on_bin_edge), len(set(on_bin_edge) & set(over))))


@pytest.mark.parametrize("S", [17, 33, 34, 66])
@pytest.mark.parametrize("extra", [0, 1, 2])
def test_saved_records(extra, S):
    fv, _ = rs.records(S, extra)
    recs = rs.tile_records(fv[0], S)
    assert recs[0, 0] == 32 * 8 + extra
    # the covering face: every pixel of every tile, in full 32-record blocks where the tile is whole
    assert int(rs.survivors(fv[0, :1], S).sum()) == S * S
    assert rs.fwd3_segments(rs.boxes(fv[0], F32), S)[0] == (1 + extra, 8 + extra)


def test_window_crossing():
    fv, _, on = rs.window_crossing()
    F = fv.shape[1]
    assert F > rs.FACE_WINDOW and list(on) == [0, rs.FACE_WINDOW - 1, rs.FACE_WINDOW, F - 1]
    box = rs.boxes(fv[0], F32)
    listed = np.flatnonzero(rs.tile_hits(box, 17, 0, 0, F32, rs.CB))
    assert np.array_equal(listed, on)
    assert {int(f) // rs.FACE_WINDOW for f in on} == {0, 1}


def test_many_images():
    fv, tex = rs.many_images(65535)
    assert fv.shape == (65535, 2, 9) and tex.shape == (65535, 2, 1, 3)
    assert len(np.unique(fv[:, 1, 0])) > 60000
