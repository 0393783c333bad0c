"""SCOPS part centres and part points (DESIGN.md §17) without a GPU: the numpy restatement pinned against the reference's
own `prob2center` / `sample_prob` (tests/golden/part_points/reference.npz, made by tests/golden/make_part_points_golden.py),
the Efraimidis-Spirakis draw against the exact law of torch.multinomial without replacement, and every refusal of the C
ABI and of the Python arguments, which come before any device work."""
import ctypes
import os
import re

import numpy as np
import pytest
import scipy.stats
import torch

import part_points_oracle as ppo
from umr_b200 import _lib
from umr_b200.utils import image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "part_points", "reference.npz")


# ---------------------------------------------------------------------------------------------------------------------
# the restatement against the reference's own functions
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_centres_match_the_reference(golden):
    prob, mask = golden["part_prob"], golden["mask"].astype(np.float64)
    for b in range(prob.shape[0]):
        for k, ch in enumerate(golden["channels"]):
            np.testing.assert_allclose(ppo.centre(prob[b], mask[b], int(ch)), golden["centres"][b, k], rtol=0, atol=1e-6)


def test_nearest_selection_matches_the_reference_on_its_draws(golden):
    prob, mask = golden["part_prob"], golden["mask"].astype(np.float64)
    S = prob.shape[1]
    for b in range(prob.shape[0]):
        for k, (ch, n) in enumerate(zip(golden["channels"], golden["num_samples"])):
            draws = golden["draws_%d" % k][b]
            assert len(draws) == ppo.n_draws(int(n)) and len(set(draws.tolist())) == len(draws)
            q = (prob[b, :, :, ch] * mask[b]).reshape(-1)
            assert (q[draws] > 0).all()
            c = ppo.centre(prob[b], mask[b], int(ch))
            got = ppo.nearest(draws, c, S, int(n), np.float32)
            np.testing.assert_array_equal(got, golden["points_%d" % k][b])


def test_coordinates_keep_the_reference_constant():
    # x = k % S, y = k // S, mapped by c / 256 * 2 - 1 whatever S is
    np.testing.assert_array_equal(ppo.coords([0, 65, 64 * 64 - 1], 64, np.float64),
                                  [[-1, -1], [1 / 128 - 1, 1 / 128 - 1], [63 / 128 - 1, 63 / 128 - 1]])
    np.testing.assert_array_equal(ppo.coords([255 * 256 + 3], 256, np.float32), [[3 / 128 - 1, 255 / 128 - 1]])


def test_nearest_breaks_distance_ties_by_pixel_index():
    # centre on pixel (2, 2) of an 8 x 8 map: its four neighbours are equidistant
    c = ppo.coords([2 * 8 + 2], 8, np.float64)[0]
    got = ppo.nearest([3 * 8 + 2, 2 * 8 + 3, 2 * 8 + 1, 1 * 8 + 2, 2 * 8 + 2], c, 8, 5, np.float64)
    np.testing.assert_array_equal(got, ppo.coords([2 * 8 + 2, 1 * 8 + 2, 2 * 8 + 1, 2 * 8 + 3, 3 * 8 + 2], 8, np.float64))


# ---------------------------------------------------------------------------------------------------------------------
# the draw's law: exact subset probabilities of sequential sampling without replacement
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("S,m", [(3, 2), (3, 3), (4, 2), (4, 3)])
def test_gumbel_top_k_has_the_law_of_multinomial_without_replacement(S, m, dtype):
    rng = np.random.default_rng(100 * S + m)
    p = rng.uniform(0.05, 1.0, S * S)
    p[rng.integers(S * S)] = 0.0          # never drawn
    p[rng.integers(S * S)] *= 8           # one heavy pixel
    q = p.astype(dtype)
    exact = ppo.subset_probabilities(q.astype(np.float64), m)
    trials = 200000
    u = rng.random((trials, S * S)).astype(dtype)
    with np.errstate(divide="ignore"):
        lg = np.log(u.astype(np.float64)).astype(dtype)
        key = np.where(q > 0, lg / np.where(q > 0, q, dtype(1)), -np.inf)
    top = np.argsort(-key.astype(np.float64), axis=1, kind="stable")[:, :m]
    assert (q[top] > 0).all()
    codes = (np.int64(1) << top).sum(axis=1)
    subsets = sorted(exact)
    index = {sum(1 << i for i in s): j for j, s in enumerate(subsets)}
    observed = np.bincount([index[c] for c in codes], minlength=len(subsets))
    expected = np.array([exact[s] for s in subsets]) * trials
    assert observed.sum() == trials
    # pool cells expected below 5 into one, as the chi-square approximation wants
    small = expected < 5
    obs = np.append(observed[~small], observed[small].sum())
    exp = np.append(expected[~small], expected[small].sum())
    obs, exp = (obs, exp) if small.any() else (obs[:-1], exp[:-1])
    assert scipy.stats.chisquare(obs, exp * obs.sum() / exp.sum()).pvalue > 1e-3
    # and so each pixel's inclusion frequency
    incl = np.bincount(top.reshape(-1), minlength=S * S) / trials
    want = np.zeros(S * S)
    for s, pr in exact.items():
        want[list(s)] += pr
    assert (np.abs(incl - want) <= 5 * np.sqrt(want * (1 - want) / trials) + 1e-12).all(), (incl, want)


# ---------------------------------------------------------------------------------------------------------------------
# C ABI: declaration, export and refusals (no GPU: a refusal comes before any device work)
# ---------------------------------------------------------------------------------------------------------------------
def test_header_declares_exactly_the_bound_symbols():
    src = open(os.path.join(ROOT, "include", "umr_part_points.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = set(re.findall(r"\b(umr_[a-z0-9_]+)\s*\(", src))
    assert names == set(_lib.PP_EXPORTS)
    assert '#include "umr_part_points.h"' in open(os.path.join(ROOT, "include", "umr_b200.h")).read()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(lib, n)


A = 256          # non-NULL, aligned to 16
BAD_ARG, TOO_LARGE = -2, -3


def _call(*, prob=A, mask=A, u=A, B=2, S=64, C=5, K=4, channels=(1, 2, 3, 4), ns=(10, 10, 30, 30), dtype=0, cin=0,
          centers=A, points=(A,) * 4, drawn=None, status=A):
    ch = (ctypes.c_int32 * len(channels))(*channels) if channels is not None else None
    n = (ctypes.c_int32 * len(ns))(*ns) if ns is not None else None
    pts = (ctypes.c_void_p * len(points))(*points) if points is not None else None
    dr = (ctypes.c_void_p * len(drawn))(*drawn) if drawn is not None else None
    return (prob, mask, u, B, S, C, K, ch, n, dtype, cin, centers, pts, dr, status)


REFUSALS = (
    [(_call(**{k: None}), BAD_ARG) for k in ("prob", "mask", "u", "channels", "ns", "centers", "points", "status")]
    + [(_call(points=(A, A, None, A)), BAD_ARG)]
    + [(_call(**{k: v}), BAD_ARG) for k in ("B", "S", "C", "K") for v in (0, -1)]
    + [(_call(K=9, channels=(1,) * 9, ns=(10,) * 9, points=(A,) * 9), BAD_ARG)]
    + [(_call(channels=(1, 2, 3, c)), BAD_ARG) for c in (-1, 5)]
    + [(_call(ns=(10, 10, 0, 30)), BAD_ARG), (_call(ns=(10, -3, 30, 30)), BAD_ARG), (_call(dtype=2), BAD_ARG)]
    # misaligned: element size for the maps, twice it for centres and points, 4 bytes for status and drawn
    + [(_call(**{k: A + 2}), BAD_ARG) for k in ("prob", "mask", "u", "centers", "cin", "status")]
    + [(_call(dtype=1, **{k: A + 4}), BAD_ARG) for k in ("prob", "mask", "u")]
    + [(_call(centers=A + 4), BAD_ARG), (_call(dtype=1, centers=A + 8), BAD_ARG), (_call(dtype=1, cin=A + 8), BAD_ARG)]
    + [(_call(points=(A, A + 4, A, A)), BAD_ARG), (_call(drawn=(A, A, A + 2, A)), BAD_ARG)]
    # m = floor(1.5 n) above 1024 (n = 683 draws exactly 1024), sides above 4096
    + [(_call(ns=(10, 10, 30, 684)), TOO_LARGE), (_call(ns=(100000,) * 4), TOO_LARGE), (_call(S=4097), TOO_LARGE)]
)


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


@pytest.mark.parametrize("args,code", REFUSALS, ids=[str(i) for i in range(len(REFUSALS))])
def test_refused_before_device_work(lib, args, code):
    before = lib.umr_launch_count()
    assert lib.umr_part_points(*args, None) == code
    assert lib.umr_launch_count() == before


# ---------------------------------------------------------------------------------------------------------------------
# Python argument checks (before any device work)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def claims_cuda(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def test_cpu_tensors_are_refused():
    with pytest.raises(TypeError):
        image.part_points(torch.zeros(2, 8, 8, 5), torch.zeros(2, 8, 8))


def test_inputs_on_different_devices_are_refused(claims_cuda):
    p = torch.zeros(2, 8, 8, 5)
    with pytest.raises(ValueError, match="one device"):
        image._part_points(p, torch.zeros(2, 8, 8, device="meta"), torch.zeros(2, 4, 64), (10,) * 4, (1, 2, 3, 4))


@pytest.mark.parametrize("prob,mask,u,ns,chs", [
    ((2, 8, 9, 5), (2, 8, 9), (2, 4, 72), (1,) * 4, (1, 2, 3, 4)),      # not square
    ((2, 8, 8), (2, 8, 8), (2, 4, 64), (1,) * 4, (1, 2, 3, 4)),         # no channel axis
    ((2, 8, 8, 5), (3, 8, 8), (2, 4, 64), (1,) * 4, (1, 2, 3, 4)),      # B differs
    ((2, 8, 8, 5), (2, 8, 8, 1), (2, 4, 64), (1,) * 4, (1, 2, 3, 4)),   # mask keeps its singleton axis
    ((2, 8, 8, 5), (2, 8, 8), (2, 3, 64), (1,) * 4, (1, 2, 3, 4)),      # uniforms for 3 channels
    ((2, 8, 8, 5), (2, 8, 8), (2, 4, 64), (1,) * 3, (1, 2, 3, 4)),      # counts differ
    ((2, 8, 8, 5), (2, 8, 8), (2, 4, 64), (1,) * 4, (1, 2, 3, 5)),      # no channel 5
    ((2, 8, 8, 5), (2, 8, 8), (2, 4, 64), (1, 1, 0, 1), (1, 2, 3, 4)),
    ((2, 8, 8, 5), (2, 8, 8), (2, 4, 64), (1, 1, 684, 1), (1, 2, 3, 4)),  # 1026 draws
    ((2, 8, 8, 5), (2, 8, 8), (2, 9, 64), (1,) * 9, tuple(range(9))),   # 9 channels
    ((2, 8, 8, 5), (2, 8, 8), (2, 0, 64), (), ()),
])
def test_argument_checks(claims_cuda, prob, mask, u, ns, chs):
    with pytest.raises(ValueError):
        image._part_points(torch.zeros(prob), torch.zeros(mask), torch.zeros(u), ns, chs)


def test_half_precision_is_refused(claims_cuda):
    with pytest.raises(TypeError):
        image._part_points(torch.zeros(2, 8, 8, 5, dtype=torch.float16), torch.zeros(2, 8, 8), torch.zeros(2, 4, 64),
                           (1,) * 4, (1, 2, 3, 4))
