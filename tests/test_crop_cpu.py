"""Batch crop, resize, mirror and normalisation (DESIGN.md §19) without a GPU: the host loader helpers and the numpy
restatement pinned against the reference's own `forward_img` / `set_input` (tests/golden/crop/reference.npz, made by
tests/golden/make_crop_golden.py), the restatement against cv2 over a size sweep, the collate's pack and table, and
every refusal of the C ABI and of the Python arguments, which come before any device work."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import crop_oracle as co
from umr_b200 import _lib
from umr_b200.utils import crop_loader as cl
from umr_b200.utils import image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "crop", "reference.npz")
KP_PERM = np.array([1, 2, 3, 4, 5, 6, 11, 12, 13, 10, 7, 8, 9, 14, 15]) - 1


# ---------------------------------------------------------------------------------------------------------------------
# the loader helpers and the restatement against the reference's own forward_img / set_input
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLDEN)
    return {str(c): {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(str(c) + "/")} for c in z["cases"]}


def host_item(g, S=64):
    """forward_img's host half on a golden case, seeded as the reference was."""
    rot = np.pad(g["sfm_rot"], (0, 1), "constant")
    rot[3, 3] = 1
    sfm = [np.copy(g["sfm_scale"]), np.copy(g["sfm_trans"]), cl.quaternion_from_matrix(rot)]
    np.random.seed(int(g["seed"]))
    pf, jf = g["fracs"]
    return cl.crop_item(g["src"], g["src_mask"], g["bbox"] - 1, g["parts"].T, sfm, S, pf, jf, True, KP_PERM)


def test_golden_covers_the_case_list(golden):
    assert len(golden) == 12
    sides = {int(g["sq_bbox"][2] - g["sq_bbox"][0] + 1) for g in golden.values()}
    assert {1, 64, 127, 128, 129}.issubset(sides) and min(sides - {1}) < 64 and max(sides) > 8 * 64
    assert {bool(g["flip"]) for g in golden.values()} == {False, True}
    assert any(g["src"].ndim == 2 for g in golden.values())
    assert any(np.isnan(g["part_segs"]).any() for g in golden.values() if "part_segs" in g)


def test_boxes_flips_and_points_match_the_reference(golden):
    for name, g in golden.items():
        win, kp, sfm, box = host_item(g)
        assert box == list(g["sq_bbox"]), name
        assert win.flip == bool(g["flip"]), name
        np.testing.assert_array_equal(kp, g["kp"], err_msg=name)
        sfm[0].shape = 1
        np.testing.assert_array_equal(np.concatenate(sfm), g["sfm_pose"], err_msg=name)


def test_pixels_match_the_reference_bitwise(golden):
    for name, g in golden.items():
        win = host_item(g)[0]
        part = g["part_in"][None] if "part_in" in g else None
        imgs, input_imgs, masks, prob, segs = co.batch([win], 64, part)
        assert co.bitwise_equal(imgs[0], g["imgs"]), name
        assert co.bitwise_equal(input_imgs[0], g["input_imgs"]), name
        assert co.bitwise_equal(masks[0], g["masks"]), name
        if part is not None:
            assert co.bitwise_equal(prob[0], g["part_prob"]), name
            assert co.bitwise_equal(segs[0], g["part_segs"]), name


def test_the_window_is_a_slice_of_the_source():
    img = np.arange(5 * 7 * 3, dtype=np.uint8).reshape(5, 7, 3)
    mask = (np.arange(35).reshape(5, 7) % 2).astype(np.uint8)
    w = cl.crop_window(img, mask, [-2, 1, 5.0, 8.0])     # L = 8, overlaps x 0..5, y 1..4
    assert (w.x0, w.y0, w.L) == (2, 0, 8)
    np.testing.assert_array_equal(w.img, img[1:5, 0:6])
    np.testing.assert_array_equal(w.mask, mask[1:5, 0:6])
    assert np.shares_memory(w.img, img)
    g = cl.crop_window(img[..., 0], mask, [0, 0, 2.0, 2.0])
    assert g.img.shape == (3, 3, 1)
    # no overlap: a 1 x 1 window of the background values
    e = cl.crop_window(img, mask, [10, 10, 12.0, 12.0])
    assert (e.img.tolist(), e.mask.tolist(), e.x0, e.y0, e.L) == ([[[255]]], [[0]], 0, 0, 3)
    with pytest.raises(ValueError):
        cl.crop_window(img.astype(np.float64), mask, [0, 0, 2.0, 2.0])
    with pytest.raises(ValueError):
        cl.crop_window(img, mask, [0, 0, 2.0, 3.0])


# ---------------------------------------------------------------------------------------------------------------------
# the restatement against cv2
# ---------------------------------------------------------------------------------------------------------------------
def _ulps(a, b):
    ia = a.astype(np.float32).view(np.int32).astype(np.int64)
    ib = b.astype(np.float32).view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


SWEEP = [(L, S, ch) for S in (64, 128, 256) for L in (1, 2, 3, 7, 63, 64, 65, 100, 127, 129, 255, 257, 310, 511, 600, 1200)
         for ch in (1, 3)]


@pytest.mark.parametrize("L,S,ch", SWEEP)
def test_resize_within_one_ulp_of_cv2(L, S, ch):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(L * 1000 + S + ch)
    src = rng.integers(0, 256, (L, L, ch)).astype(np.float64) / 255.0
    want = cv2.resize(src, (S, S)).reshape(S, S, ch).astype(np.float32)
    got = co.resize(src, S).astype(np.float32)
    d = _ulps(got, want)
    assert d.max() <= 1, (int(d.max()), int((d != 0).sum()))


@pytest.mark.parametrize("S", [64, 128, 256])
def test_resize_at_twice_the_side_within_one_ulp_of_cv2(S):
    # cv2 resizes an exact 2x reduction with INTER_AREA: a 2 x 2 mean where the restatement takes two linear passes
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(S)
    src = rng.integers(0, 256, (2 * S, 2 * S, 3)).astype(np.float64) / 255.0
    want = cv2.resize(src, (S, S)).astype(np.float32)
    got = co.resize(src, S).astype(np.float32)
    d = _ulps(got, want)
    print("2x S=%d: %d of %d elements differ by 1 ulp" % (S, int((d != 0).sum()), d.size))
    assert d.max() <= 1


# ---------------------------------------------------------------------------------------------------------------------
# collate: the pack and the table
# ---------------------------------------------------------------------------------------------------------------------
def test_collate_packs_windows_and_table():
    rng = np.random.default_rng(3)
    wins = [cl.CropWindow(rng.integers(0, 256, (4, 5, 3), dtype=np.uint8), rng.integers(0, 2, (4, 5), dtype=np.uint8),
                          1, 2, 9, True),
            cl.CropWindow(rng.integers(0, 256, (2, 3, 1), dtype=np.uint8), rng.integers(0, 2, (2, 3), dtype=np.uint8),
                          0, 0, 3, False)]
    batch = [{"crop": w, "kp": np.full((15, 3), i, np.float64), "inds": i} for i, w in enumerate(wins)]
    out = cl.collate(batch)
    assert set(out) == {"crop_pack", "crop_table", "kp", "inds"}
    assert out["kp"].shape == (2, 15, 3) and out["inds"].tolist() == [0, 1]
    pack, table = out["crop_pack"].numpy(), out["crop_table"]
    assert table.dtype == torch.int32 and table.tolist() == [[0, 4, 5, 3, 1, 2, 9, 1], [80, 2, 3, 1, 0, 0, 3, 0]]
    assert pack.dtype == np.uint8 and pack.size == 80 + 12
    np.testing.assert_array_equal(pack[:60], wins[0].img.reshape(-1))
    np.testing.assert_array_equal(pack[60:80], wins[0].mask.reshape(-1))
    np.testing.assert_array_equal(pack[80:86], wins[1].img.reshape(-1))
    np.testing.assert_array_equal(pack[86:], wins[1].mask.reshape(-1))


def test_collate_as_a_dataloader_collate_fn():
    class Items(torch.utils.data.Dataset):
        def __len__(self):
            return 4

        def __getitem__(self, i):
            np.random.seed(i)
            img = np.full((20, 30, 3), i, np.uint8)
            mask = np.ones((20, 30), np.uint8)
            sfm = [np.float64(100.0), np.array([10.0, 5.0]), np.array([1.0, 0, 0, 0])]
            win, kp, sfm, _ = cl.crop_item(img, mask, [2.0, 3.0, 25.0, 15.0], np.ones((15, 3)), sfm, 16, 0.05, 0.05,
                                           True, KP_PERM)
            return {"crop": win, "kp": kp}
    out = next(iter(torch.utils.data.DataLoader(Items(), batch_size=4, collate_fn=cl.collate)))
    assert out["crop_table"].shape == (4, 8) and out["kp"].shape == (4, 15, 3)


# ---------------------------------------------------------------------------------------------------------------------
# C ABI: declaration, export and refusals (no GPU: a refusal comes before any device work)
# ---------------------------------------------------------------------------------------------------------------------
def test_header_declares_exactly_the_bound_symbols():
    src = open(os.path.join(ROOT, "include", "umr_crop.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = set(re.findall(r"\b(umr_[a-z0-9_]+)\s*\(", src))
    assert names == set(_lib.CROP_EXPORTS)
    assert '#include "umr_crop.h"' in open(os.path.join(ROOT, "include", "umr_b200.h")).read()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(lib, n)


A = 256          # non-NULL, 4-byte aligned
BAD_ARG, TOO_LARGE = -2, -3
ROW = (0, 10, 12, 3, 2, 1, 20, 1)   # a 10 x 12 RGB window at (2, 1) in a 20 frame: 480 bytes


def _call(*, pack=A, nbytes=480, tdev=A, rows=(ROW,), B=None, S=64, part=0, C=5, imgs=A, inp=A, masks=A, pout=A,
          segs=A):
    tab = (ctypes.c_int32 * (8 * len(rows)))(*[v for r in rows for v in r]) if rows is not None else None
    return (pack, nbytes, tdev, tab, len(rows or ()) if B is None else B, S, part, C, imgs, inp, masks, pout, segs)


def _row(**kw):
    cols = dict(zip(("off", "h", "w", "ch", "x0", "y0", "L", "flip"), ROW))
    cols.update(kw)
    return (tuple(cols.values()),)


REFUSALS = (
    [(_call(**{k: None}), BAD_ARG) for k in ("pack", "tdev", "rows", "imgs", "inp", "masks")]
    + [(_call(part=A, **{k: None}), BAD_ARG) for k in ("pout", "segs")]
    + [(_call(B=v), BAD_ARG) for v in (0, -1)] + [(_call(S=v), BAD_ARG) for v in (0, -1)]
    + [(_call(nbytes=0), BAD_ARG)]
    + [(_call(part=A, C=c), BAD_ARG) for c in (0, 9)]
    + [(_call(**{k: A + 2}), BAD_ARG) for k in ("tdev", "imgs", "inp", "masks")]
    + [(_call(part=A + 2), BAD_ARG), (_call(part=A, pout=A + 1), BAD_ARG), (_call(part=A, segs=A + 3), BAD_ARG)]
    # per image: window dims, position, fit, channels, offset, pack size, flag
    + [(_call(rows=_row(**{k: v})), BAD_ARG) for k in ("h", "w", "L") for v in (0, -1)]
    + [(_call(rows=_row(x0=-1)), BAD_ARG), (_call(rows=_row(y0=-1)), BAD_ARG)]
    + [(_call(rows=_row(x0=9)), BAD_ARG), (_call(rows=_row(y0=11)), BAD_ARG), (_call(rows=_row(L=11)), BAD_ARG)]
    + [(_call(rows=_row(ch=c)), BAD_ARG) for c in (0, 2, 4)]
    + [(_call(rows=_row(off=-1)), BAD_ARG), (_call(rows=_row(off=1)), BAD_ARG), (_call(nbytes=479), BAD_ARG)]
    + [(_call(rows=(ROW, _row(off=1)[0])), BAD_ARG), (_call(rows=_row(flip=2)), BAD_ARG)]
    # caps: S, L
    + [(_call(S=4097), TOO_LARGE), (_call(rows=_row(L=65537, h=1, w=1)), TOO_LARGE)]
)


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


@pytest.mark.parametrize("args,code", REFUSALS, ids=[str(i) for i in range(len(REFUSALS))])
def test_refused_before_device_work(lib, args, code):
    before = lib.umr_launch_count()
    assert lib.umr_crop_batch(*args, None) == code
    assert lib.umr_launch_count() == before


# ---------------------------------------------------------------------------------------------------------------------
# Python argument checks (before any device work)
# ---------------------------------------------------------------------------------------------------------------------
def _table(B=2):
    return torch.tensor([ROW] * B, dtype=torch.int32)


@pytest.mark.parametrize("pack,table,size", [
    (torch.zeros(480, dtype=torch.uint8), _table().to(torch.int64), 64),        # table dtype
    (torch.zeros(480, dtype=torch.uint8), _table()[:, :7], 64),                  # table columns
    (torch.zeros(480, dtype=torch.uint8), _table()[0], 64),                      # table rank
    (torch.zeros(480, dtype=torch.uint8), torch.zeros(0, 8, dtype=torch.int32), 64),
    (torch.zeros(480, dtype=torch.float32), _table(), 64),                       # pack dtype
    (torch.zeros(0, dtype=torch.uint8), _table(), 64),                           # empty pack
    (torch.zeros(480, dtype=torch.uint8), _table(), 0),
    (torch.zeros(480, dtype=torch.uint8), _table(), 1.5),
    (torch.zeros(480, dtype=torch.uint8), _table(), True),
])
def test_argument_checks(pack, table, size):
    with pytest.raises(ValueError):
        image.crop_batch(pack, table, size)


def test_part_prob_checks(monkeypatch):
    pack = torch.zeros(480, dtype=torch.uint8)
    with pytest.raises(TypeError):   # a host part map
        image.crop_batch(pack, _table(), 8, torch.zeros(2, 8, 8, 5))
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: self.dtype != torch.int32))   # all but the table
    with pytest.raises(TypeError):
        image.crop_batch(pack, _table(), 8, torch.zeros(2, 8, 8, 5, dtype=torch.float64))
    for shape in ((2, 8, 8), (3, 8, 8, 5), (2, 8, 9, 5), (2, 8, 8, 0), (2, 8, 8, 9), (2, 4, 4, 5)):
        with pytest.raises(ValueError):
            image.crop_batch(pack, _table(), 8, torch.zeros(shape))
