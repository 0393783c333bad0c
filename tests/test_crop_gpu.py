"""Batch crop, resize, mirror and normalisation on the GPU (DESIGN.md §19): `utils.image.crop_batch` against the numpy
restatement (tests/crop_oracle.py) and the reference's recorded float32 outputs (tests/golden/crop/reference.npz), bit
for bit, with guard bands, launch counts, CUDA-graph capture, run-to-run reproducibility and the set_input composition
with compute_dt_barrier and part_points."""
import ctypes
import os

import numpy as np
import pytest
import torch

import crop_oracle as co
from umr_b200 import _lib
from umr_b200.utils import crop_loader as cl
from umr_b200.utils import image

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "crop", "reference.npz")
KP_PERM = np.array([1, 2, 3, 4, 5, 6, 11, 12, 13, 10, 7, 8, 9, 14, 15]) - 1
DEV = torch.device("cuda:0")


def random_windows(rng, B, S):
    """B windows over the frame sides of the case list, 1 or 3 channels, either flip, some overlapping no pixel."""
    sides = [1, 2, 17, S // 2, S - 1, S, S + 1, 2 * S - 1, 2 * S, 2 * S + 1, 5 * S + 3, 310]
    wins = []
    for b in range(B):
        L = sides[b % len(sides)] if b < len(sides) else int(rng.integers(1, 3 * S))
        ch = int(rng.choice([1, 3]))
        flip = bool(rng.integers(2))
        if b % 7 == 3:
            wins.append(cl.CropWindow(np.full((1, 1, 1), 255, np.uint8), np.zeros((1, 1), np.uint8), 0, 0, L, flip))
            continue
        h, w = int(rng.integers(1, L + 1)), int(rng.integers(1, L + 1))
        x0, y0 = int(rng.integers(0, L - w + 1)), int(rng.integers(0, L - h + 1))
        wins.append(cl.CropWindow(rng.integers(0, 256, (h, w, ch), dtype=np.uint8),
                                  (rng.random((h, w)) < 0.6).astype(np.uint8), x0, y0, L, flip))
    return wins


def part_maps(rng, B, S, C):
    p = rng.random((B, S, S, C)).astype(np.float32)
    p[0, ..., C - 1] = 0.0                  # a channel zero everywhere: 0 / 0
    if B > 1:
        p[1, 3, 5, 0] = np.nan              # NaN propagates through the max
    return p


def run(wins, S, part=None):
    batch = cl.collate([{"crop": w} for w in wins])
    pack = batch["crop_pack"].to(DEV)
    prob = torch.from_numpy(part).to(DEV) if part is not None else None
    out = image.crop_batch(pack, batch["crop_table"], S, prob)
    return [o.cpu().numpy() if o is not None else None for o in out]


def assert_outputs_equal(got, want):
    for name, g, w in zip(("imgs", "input_imgs", "masks", "part_prob", "part_segs"), got, want):
        if w is None:
            assert g is None, name
        else:
            assert co.bitwise_equal(g, w), name


@pytest.mark.parametrize("S,B", [(64, 1), (64, 64), (256, 5), (256, 32)])
@pytest.mark.parametrize("with_parts", [False, True])
def test_kernel_matches_the_restatement_bitwise(S, B, with_parts):
    rng = np.random.default_rng(S * 100 + B + with_parts)
    wins = random_windows(rng, B, S)
    part = part_maps(rng, B, S, 5) if with_parts else None
    assert_outputs_equal(run(wins, S, part), co.batch(wins, S, part))


@pytest.mark.parametrize("C", [1, 3, 8])
def test_part_channel_counts(C):
    rng = np.random.default_rng(C)
    wins = random_windows(rng, 4, 64)
    part = part_maps(rng, 4, 64, C)
    assert_outputs_equal(run(wins, 64, part), co.batch(wins, 64, part))


def test_kernel_matches_the_reference_golden():
    z = np.load(GOLDEN)
    for name in z["cases"]:
        g = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(str(name) + "/")}
        rot = np.pad(g["sfm_rot"], (0, 1), "constant")
        rot[3, 3] = 1
        sfm = [np.copy(g["sfm_scale"]), np.copy(g["sfm_trans"]), cl.quaternion_from_matrix(rot)]
        np.random.seed(int(g["seed"]))
        win = cl.crop_item(g["src"], g["src_mask"], g["bbox"] - 1, g["parts"].T, sfm, 64, g["fracs"][0], g["fracs"][1],
                           True, KP_PERM)[0]
        imgs, input_imgs, masks, prob, segs = run([win], 64, g["part_in"][None] if "part_in" in g else None)
        assert co.bitwise_equal(imgs[0], g["imgs"]), name
        assert co.bitwise_equal(input_imgs[0], g["input_imgs"]), name
        assert co.bitwise_equal(masks[0], g["masks"]), name
        if "part_in" in g:
            assert co.bitwise_equal(prob[0], g["part_prob"]), name
            assert co.bitwise_equal(segs[0], g["part_segs"]), name


def test_guard_bands_and_launch_counts():
    rng = np.random.default_rng(5)
    B, S, C, G = 6, 64, 5, 4096
    wins = random_windows(rng, B, S)
    part = part_maps(rng, B, S, C)
    batch = cl.collate([{"crop": w} for w in wins])
    pack = batch["crop_pack"].to(DEV)
    table = batch["crop_table"]
    tab_dev = table.to(DEV)
    sizes = {"imgs": B * 3 * S * S, "inp": B * 3 * S * S, "masks": B * S * S, "pout": B * S * S * C, "segs": B * C * S * S}
    sentinel = -12345.5
    bufs = {k: torch.full((n + 2 * G,), sentinel, device=DEV) for k, n in sizes.items()}
    prob = torch.from_numpy(part).to(DEV)
    lib = _lib.load()
    host = ctypes.cast(table.data_ptr(), ctypes.POINTER(ctypes.c_int32))
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ptr = lambda k: ctypes.c_void_p(bufs[k].data_ptr() + 4 * G)   # noqa: E731
    for with_parts, launches in ((False, 1), (True, 2)):
        before = lib.umr_launch_count()
        code = lib.umr_crop_batch(ctypes.c_void_p(pack.data_ptr()), pack.numel(), ctypes.c_void_p(tab_dev.data_ptr()), host,
                                  B, S, ctypes.c_void_p(prob.data_ptr() if with_parts else 0), C if with_parts else 0,
                                  ptr("imgs"), ptr("inp"), ptr("masks"), ptr("pout") if with_parts else None,
                                  ptr("segs") if with_parts else None, stream)
        assert code == 0
        assert lib.umr_launch_count() - before == launches
    torch.cuda.synchronize()
    want = co.batch(wins, S, part)
    for (k, n), w in zip(sizes.items(), want):
        buf = bufs[k].cpu().numpy()
        assert (buf[:G] == sentinel).all() and (buf[G + n:] == sentinel).all(), k
        assert co.bitwise_equal(buf[G:G + n], w.reshape(-1)), k


def test_part_path_on_and_off_agree_on_the_images():
    rng = np.random.default_rng(9)
    wins = random_windows(rng, 8, 64)
    on = run(wins, 64, part_maps(rng, 8, 64, 5))
    off = run(wins, 64)
    for a, b in zip(on[:3], off[:3]):
        assert co.bitwise_equal(a, b)
    assert off[3] is None and off[4] is None


def test_two_runs_are_bitwise_equal():
    rng = np.random.default_rng(11)
    wins = random_windows(rng, 32, 256)
    part = part_maps(rng, 32, 256, 5)
    assert_outputs_equal(run(wins, 256, part), run(wins, 256, part))


def test_cuda_graph_capture_for_a_fixed_packing():
    rng = np.random.default_rng(13)
    B, S = 16, 64
    wins = random_windows(rng, B, S)
    part = part_maps(rng, B, S, 5)
    batch = cl.collate([{"crop": w} for w in wins])
    pack = batch["crop_pack"].to(DEV)
    table = batch["crop_table"].pin_memory()
    prob = torch.from_numpy(part).to(DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        image.crop_batch(pack, table, S, prob)        # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = image.crop_batch(pack, table, S, prob)
    # new pixels and part maps in the same buffers, same packing
    wins2 = [w._replace(img=rng.integers(0, 256, w.img.shape, dtype=np.uint8)) for w in wins]
    pack.copy_(cl.collate([{"crop": w} for w in wins2])["crop_pack"].to(DEV))
    part2 = part_maps(rng, B, S, 5)
    prob.copy_(torch.from_numpy(part2))
    g.replay()
    torch.cuda.synchronize()
    assert_outputs_equal([o.cpu().numpy() for o in out], co.batch(wins2, S, part2))


def test_set_input_composition():
    # the kernel's masks and mirrored part maps feed compute_dt_barrier and part_points exactly as the restatement's do
    rng = np.random.default_rng(17)
    B, S = 4, 256
    wins = []
    for b in range(B):
        L = 310 + 7 * b
        img = rng.integers(0, 256, (L - 20, L - 40, 3), dtype=np.uint8)
        yy, xx = np.mgrid[:L - 20, :L - 40]
        mask = ((yy - L / 2) ** 2 + (xx - L / 2) ** 2 < (L / 3) ** 2).astype(np.uint8)
        wins.append(cl.CropWindow(img, mask, 10, 5, L, bool(b % 2)))
    part = rng.random((B, S, S, 5)).astype(np.float32) + 0.01
    got = run(wins, S, part)
    want = co.batch(wins, S, part)
    assert_outputs_equal(got, want)
    outs = []
    for masks, prob in ((got[2], got[3]), (want[2], want[3])):
        m = torch.from_numpy(np.ascontiguousarray(masks)).to(DEV)
        p = torch.from_numpy(np.ascontiguousarray(prob)).to(DEV)
        dt = image.compute_dt_barrier(m)
        gen = torch.Generator(device=DEV)
        gen.manual_seed(3)
        centres, points = image.part_points(p, m, generator=gen)
        outs.append([dt.cpu().numpy(), centres.cpu().numpy()] + [q.cpu().numpy() for q in points])
    for a, b in zip(*outs):
        assert co.bitwise_equal(a, b)
