"""Host-side contract of the part_matching_loss head kernels (no GPU): the entry points are exported and declared, the
workspace formula, every refusal before the device is touched, and which inputs `part_matching_loss` sends to the kernels
and which to the torch composition -- with the op replaced by a torch restatement of its per-image terms, so the
O(B) combination of those terms is checked against the composition on CPU tensors."""
import ctypes
import os
import re

import pytest
import torch

from umr_b200 import _lib, ops
from umr_b200.nnutils import loss_utils

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("umr_part_head_workspace_bytes", "umr_part_head_forward", "umr_part_head_backward")
UMR_ERR_BAD_ARG, UMR_ERR_TOO_LARGE = -2, -3
FAKE = 4096                     # a non-NULL, aligned device address: every case below is refused before it is read
INT_MAX = 2 ** 31 - 1


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def test_symbols_exported_and_declared(lib):
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "umr_b200.h")).read(), flags=re.S)
    for name in NAMES:
        assert name in _lib.EXPORTS
        assert getattr(lib, name) is not None
        assert re.search(r"\b%s\s*\(" % name, header), name
        # one symbol per operation: float64 through the dtype argument; no atomics, so no deterministic twin
        assert name + "_f64" not in _lib.EXPORTS and name + "_deterministic" not in _lib.EXPORTS


def _ns(H):
    return (H * H + 2047) // 2048


@pytest.mark.parametrize("dtype,size", [(0, 4), (1, 8)])
def test_workspace_formula(lib, dtype, size):
    fn = lib.umr_part_head_workspace_bytes
    for B, H in ((1, 1), (2, 3), (17, 31), (16, 256), (32, 512), (65535, 2), (3, 46340)):
        ns = _ns(H)
        assert fn(B, H, dtype) == B * ((ns + 1) * 40 * size + (8 + ns * 10) * 4), (B, H)
    for B, H in ((0, 8), (-1, 8), (2, 0), (2, -4), (65536, 2), (1, 46341)):
        assert fn(B, H, dtype) == 0, (B, H)
    for bad in (-1, 2, 3):
        assert fn(2, 8, bad) == 0


def _maps(addrs=(FAKE,) * 4, strides=(64,) * 4):
    return (ctypes.c_void_p * 4)(*addrs), (ctypes.c_int64 * 4)(*strides)


def _fwd(lib, dtype, maps=None, c0=FAKE, c0_bs=64, segs=FAKE, segs_bs=320, w=FAKE, terms=FAKE, B=2, H=8, kld=0,
         ws=FAKE):
    mp, mb = maps if maps is not None else _maps()
    return lib.umr_part_head_forward(mp, mb, c0, c0_bs, segs, segs_bs, w, terms, B, H, kld, dtype, ws, None)


def _bwd(lib, dtype, maps=None, c0=FAKE, c0_bs=64, segs=FAKE, segs_bs=320, w=FAKE, ws=FAKE, g=FAKE, gm=FAKE, B=2, H=8,
         kld=0):
    mp, mb = maps if maps is not None else _maps()
    return lib.umr_part_head_backward(mp, mb, c0, c0_bs, segs, segs_bs, w, ws, g, gm, B, H, kld, dtype, None)


@pytest.mark.parametrize("dtype,size", [(0, 4), (1, 8)])
@pytest.mark.parametrize("call", [_fwd, _bwd])
def test_refusals(lib, dtype, size, call):
    odd = FAKE + size // 2
    bufs = ("c0", "segs", "w", "ws") + (("terms",) if call is _fwd else ("g", "gm"))
    for k in bufs:
        assert call(lib, dtype, **{k: None}) == UMR_ERR_BAD_ARG, k
        assert call(lib, dtype, **{k: odd}) == UMR_ERR_BAD_ARG, k
    for i in range(4):
        addrs = [FAKE] * 4
        addrs[i] = None
        assert call(lib, dtype, maps=_maps(addrs)) == UMR_ERR_BAD_ARG
        addrs[i] = odd
        assert call(lib, dtype, maps=_maps(addrs)) == UMR_ERR_BAD_ARG
        strides = [64] * 4
        strides[i] = -1
        assert call(lib, dtype, maps=_maps(strides=strides)) == UMR_ERR_BAD_ARG
    fn = lib.umr_part_head_forward if call is _fwd else lib.umr_part_head_backward
    mp, mb = _maps()
    args = [mp, mb, FAKE, 64, FAKE, 320, FAKE] + ([FAKE] if call is _fwd else [FAKE, FAKE, FAKE])
    tail = [FAKE, None] if call is _fwd else [None]
    assert fn(None, mb, *args[2:], 2, 8, 0, dtype, *tail) == UMR_ERR_BAD_ARG
    assert fn(mp, None, *args[2:], 2, 8, 0, dtype, *tail) == UMR_ERR_BAD_ARG
    for bad in (-1, 2):
        assert fn(*args, 2, 8, 0, bad, *tail) == UMR_ERR_BAD_ARG
    for kw in (dict(B=0), dict(B=-3), dict(H=0), dict(H=-1), dict(kld=2), dict(kld=-1), dict(c0_bs=-1), dict(segs_bs=-5)):
        assert call(lib, dtype, **kw) == UMR_ERR_BAD_ARG, kw
    assert call(lib, dtype, B=65536) == UMR_ERR_TOO_LARGE
    assert call(lib, dtype, H=46341) == UMR_ERR_TOO_LARGE
    assert call(lib, dtype, B=65536, c0=None) == UMR_ERR_BAD_ARG   # argument checks come first


def test_op_refuses_cpu_tensors():
    x = torch.zeros(1, 1, 4, 4)
    with pytest.raises(TypeError):
        ops.part_matching_head([x] * 4, x, torch.zeros(1, 5, 4, 4), torch.ones(5), False)


# --- which path part_matching_loss takes -------------------------------------------------------------------------------
class _T(object):
    """The attributes part_head_on_device reads, for any device."""

    def __init__(self, shape, cuda=True, grad=False):
        self.shape, self.is_cuda, self.requires_grad = shape, cuda, grad

    def dim(self):
        return len(self.shape)

    def size(self, i):
        return self.shape[i]


@pytest.mark.parametrize("case,kernels", [
    (dict(), True),
    (dict(segs_cpu=True), False),
    (dict(map_cpu=2), False),
    (dict(c0_cpu=True), False),
    (dict(segs_grad=True), False),
    (dict(W=9), False),
    (dict(B=65535), True),
    (dict(B=65536), False),
])
def test_dispatch(case, kernels):
    B, H, W = case.get("B", 2), 8, case.get("W", 8)
    maps = [_T((B, 1, H, W), cuda=case.get("map_cpu") != k) for k in range(4)]
    c0 = _T((B, 1, H, W), cuda=not case.get("c0_cpu"))
    segs = _T((B, 5, H, W), cuda=not case.get("segs_cpu"), grad=case.get("segs_grad", False))
    assert loss_utils.part_head_on_device(maps, c0, segs) == kernels


def _terms_torch(projs, c0, segs, weights, kld):
    """The op's per-image terms restated in torch: what the kernels compute."""
    bs = segs.size(0)
    proj = torch.cat([c0] + list(projs), 1)
    cp = loss_utils.batch_get_centers(torch.softmax(proj, 1)[:, 1:])
    cq = loss_utils.batch_get_centers(torch.softmax(segs, 1)[:, 1:])
    L = ((cp - cq) ** 2).sum((1, 2))
    if kld:
        r = torch.softmax(segs, 1)
        E = (torch.xlogy(r, r) - r * torch.log_softmax(proj, 1)).sum((1, 2, 3))
    else:
        mp = proj.view(bs, 5, -1).max(2)[0].clamp_min(1e-5).view(bs, 5, 1, 1)
        mq = segs.view(bs, 5, -1).max(2)[0].clamp_min(1e-5).view(bs, 5, 1, 1)
        E = (((proj / mp - segs / mq) ** 2) * weights.view(1, 5, 1, 1)).sum((1, 2, 3))
    return torch.stack((L, E), 1)


def _module(n, im_size, loss_type):
    one_hot = torch.zeros(1, 3, 1, 5)
    one_hot[..., 0] = 1
    m = loss_utils.part_matching_loss(None, None, 0, im_size=im_size, batch_size=n, tex_size=1, loss_type=loss_type,
                                      stex_one_hot=one_hot)
    return m.double()


@pytest.mark.parametrize("loss_type", ["mse", "kld"])
@pytest.mark.parametrize("avg", [True, False])
@pytest.mark.parametrize("num_cam", [1, 8])
def test_kernel_path_combines_the_terms_as_the_composition(monkeypatch, loss_type, avg, num_cam):
    B, H = 2, 6
    n = B * num_cam
    m = _module(n, H, loss_type)
    m.proj[:, 0].uniform_(0.05, 0.2, generator=torch.Generator().manual_seed(1))
    g = torch.Generator().manual_seed(2)
    projs = [torch.rand(n, 1, H, H, generator=g, dtype=torch.float64).requires_grad_(True) for _ in range(4)]
    segs = torch.rand(n, 5, H, H, generator=g, dtype=torch.float64)
    probs = torch.softmax(torch.rand(B, num_cam, generator=g, dtype=torch.float64), 1).requires_grad_(True)
    cp = None if avg else probs
    ref = m.head(projs, segs, cp, avg)           # CPU tensors: the torch composition
    ref_g = torch.autograd.grad(ref, projs + ([] if avg else [probs]))
    calls = []

    def fake(maps, c0, part_segs, weights, kld):
        calls.append(kld)
        return _terms_torch(maps, c0, part_segs, weights, kld)
    monkeypatch.setattr(loss_utils, "part_head_on_device", lambda *a: True)
    monkeypatch.setattr(ops, "part_matching_head", fake)
    got = m.head(projs, segs, cp, avg)
    got_g = torch.autograd.grad(got, projs + ([] if avg else [probs]))
    assert calls == [loss_type == "kld"]
    assert torch.allclose(got, ref, rtol=1e-12, atol=0)
    for a, b in zip(got_g, ref_g):
        assert torch.allclose(a, b, rtol=1e-9, atol=1e-14 * float(b.abs().max()))


def test_cpu_module_takes_the_composition(monkeypatch):
    m = _module(2, 4, "mse")
    monkeypatch.setattr(ops, "part_matching_head", lambda *a: pytest.fail("the kernels were called for CPU tensors"))
    g = torch.Generator().manual_seed(0)
    projs = [torch.rand(2, 1, 4, 4, generator=g, dtype=torch.float64) for _ in range(4)]
    segs = torch.rand(2, 5, 4, 4, generator=g, dtype=torch.float64)
    assert torch.equal(m.head(projs, segs), loss_utils.part_head_torch(projs, m.proj[:2], segs, m.weights, False))
