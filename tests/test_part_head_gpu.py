"""The part_matching_loss head kernels on the GPU against `loss_utils.part_head_torch`, the torch composition they
replace: float64 at 1e-12 and by gradcheck, float32 within float32 summation error of the double composition, torch's
arg-max on plateaus and clamped maxima, the accepted range of sizes and layouts with guard bands around the outputs,
all three render branches of `part_matching_loss`, reproducibility, CUDA-graph capture, launch counts and memory."""
import ctypes

import numpy as np
import pytest
import torch

from umr_b200 import _lib, ops, synth
from umr_b200.nnutils import loss_utils
from util import rel_report

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D = torch.float64


def _module(n, H, loss_type="mse", T=1, one_hot=None):
    if one_hot is None:
        one_hot = torch.zeros(1, 3, T * T, 5)
        one_hot[..., 0] = 1
    return loss_utils.part_matching_loss(None, None, 0, im_size=H, batch_size=n, tex_size=T, loss_type=loss_type,
                                         stex_one_hot=one_hot).to(DEV)


def _inputs(B, H, dtype=D, seed=0, layout="single"):
    """Blob-shaped part maps (centroids away from 0 and from each other) with noise, and part_segs; the maps as
    standalone [B,1,H,H] tensors, or as channels of a [B,4,H,H] / [B,5,H,H] render."""
    g = torch.Generator().manual_seed(seed)
    ii = torch.arange(H, dtype=D).view(H, 1) / max(H, 1)
    jj = torch.arange(H, dtype=D).view(1, H) / max(H, 1)
    planes = []
    for k in range(9):
        cy, cx = torch.rand(B, 1, 1, generator=g, dtype=D), torch.rand(B, 1, 1, generator=g, dtype=D)
        blob = torch.exp(-((ii - cy) ** 2 + (jj - cx) ** 2) * 8)
        planes.append(blob * (0.7 + 0.3 * torch.rand(B, H, H, generator=g, dtype=D)))
    maps = torch.stack(planes[:4], 1).to(dtype)
    segs = torch.stack(planes[4:], 1).mul(3).to(dtype).to(DEV)
    if layout == "single":
        projs = [maps[:, k:k + 1].clone().to(DEV) for k in range(4)]
    else:
        C = 4 if layout == "render4" else 5
        r = torch.rand(B, C, H, H, generator=g, dtype=dtype)
        r[:, C - 4:] = maps
        r = r.to(DEV)
        projs = [r[:, C - 4 + k:C - 3 + k] for k in range(4)]
    return projs, segs


def _leaves(projs):
    return [p.detach().clone().requires_grad_(True) for p in projs]


def _run(m, projs, segs, probs, avg, kernels):
    """(loss, grads of maps [+ probs]) through part_matching_loss.head on the kernels or on the torch composition."""
    leaves = _leaves(projs)
    cp = None if avg else probs.detach().clone().requires_grad_(True)
    if kernels:
        loss = m.head(leaves, segs, cp, avg)
    else:
        c0 = m.proj[:segs.shape[0]].detach()
        loss = loss_utils.part_head_torch(leaves, c0, segs, m.weights, m.loss_type in "kld", cp, avg)
    grads = torch.autograd.grad(loss, leaves + ([] if avg else [cp]))
    return loss.detach(), [g.detach() for g in grads]


def _cmp(name, got, ref, rtol, ascale):
    got, ref = got.detach().double().cpu().numpy(), ref.detach().double().cpu().numpy()
    ok, msg = rel_report(name, got, ref, rtol, ascale * float(np.abs(ref).max()) + 1e-300)
    assert ok and np.isfinite(got).all(), msg


def _probs(n, num_cam=1, dtype=D):
    return torch.softmax(torch.linspace(-1, 1, n, dtype=dtype).view(n // num_cam, num_cam), 1).to(DEV)


def _terms_ref(projs, c0, segs, w, kld):
    """The op's per-image terms from the composition's own pieces (batch_get_centers, softmax, max), in double."""
    bs = segs.size(0)
    proj = torch.cat([c0.double()] + [p.double() for p in projs], 1)
    segs = segs.double()
    cp = loss_utils.batch_get_centers(torch.softmax(proj, 1)[:, 1:])
    cq = loss_utils.batch_get_centers(torch.softmax(segs, 1)[:, 1:])
    L = ((cp - cq) ** 2).sum((1, 2))
    if kld:
        r = torch.softmax(segs, 1)
        E = (torch.xlogy(r, r) - r * torch.log_softmax(proj, 1)).sum((1, 2, 3))
    else:
        mp = proj.view(bs, 5, -1).max(2)[0].clamp_min(1e-5).view(bs, 5, 1, 1)
        mq = segs.view(bs, 5, -1).max(2)[0].clamp_min(1e-5).view(bs, 5, 1, 1)
        E = (((proj / mp - segs / mq) ** 2) * w.double().view(1, 5, 1, 1)).sum((1, 2, 3))
    return torch.stack((L, E), 1)


# --- float64 ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("loss_type", ["mse", "kld"])
@pytest.mark.parametrize("avg", [True, False])
@pytest.mark.parametrize("B,H", [(2, 64), (3, 61)])
def test_float64_matches_the_composition(loss_type, avg, B, H):
    m = _module(B, H, loss_type)
    m.weights.copy_(torch.tensor([0.5, 5.0, 1.0, 2.0, 5.0]).view(1, 5, 1, 1))
    projs, segs = _inputs(B, H)
    probs = _probs(B)
    got, ref = _run(m, projs, segs, probs, avg, True), _run(m, projs, segs, probs, avg, False)
    _cmp("loss", got[0], ref[0], 1e-12, 0)
    for k, (a, b) in enumerate(zip(got[1], ref[1])):
        _cmp("grad%d" % k, a, b, 1e-12, 1e-12)
    terms = ops.part_matching_head(projs, m.proj[:B], segs, m.weights, loss_type == "kld")
    assert terms.dtype == D
    _cmp("terms", terms, _terms_ref(projs, m.proj[:B], segs, m.weights, loss_type == "kld"), 1e-12, 0)


@pytest.mark.parametrize("loss_type,avg", [("mse", True), ("mse", False), ("kld", True)])
def test_gradcheck(loss_type, avg):
    B, H = 2, 5
    m = _module(B, H, loss_type)
    m.weights.copy_(torch.tensor([0.5, 5.0, 1.0, 2.0, 5.0]).view(1, 5, 1, 1))
    projs, segs = _inputs(B, H, seed=3)
    leaves = _leaves(projs)
    probs = _probs(B).requires_grad_(True)

    def f(*xs):
        return m.head(list(xs[:4]), segs, None if avg else xs[4], avg)
    assert torch.autograd.gradcheck(f, tuple(leaves) + (() if avg else (probs,)), eps=1e-6, atol=1e-8, rtol=1e-6)


# --- float32 ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("loss_type", ["mse", "kld"])
@pytest.mark.parametrize("avg", [True, False])
def test_float32_within_summation_error_of_double(loss_type, avg):
    B, H = 4, 128
    m = _module(B, H, loss_type)
    projs, segs = _inputs(B, H, dtype=torch.float32, seed=5)
    probs = _probs(B, dtype=torch.float32)
    got = _run(m, projs, segs, probs, avg, True)
    ref = _run(m, [p.double() for p in projs], segs.double(), probs.double(), avg, False)
    assert got[0].dtype == torch.float32
    # float32 sums of H*H positive terms: relative error below sqrt(H*H) * 2^-24 by far in practice; 1e-5 bounds it here
    _cmp("loss", got[0], ref[0], 1e-5, 0)
    for k, (a, b) in enumerate(zip(got[1], ref[1])):
        _cmp("grad%d" % k, a, b, 1e-4, 1e-5)


# --- the max's gradient -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, D])
def test_plateau_and_clamped_maxima(dtype):
    B, H = 2, 32
    m = _module(B, H, "mse")
    m.weights.copy_(torch.tensor([0.5, 5.0, 1.0, 2.0, 5.0]).view(1, 5, 1, 1))
    projs, segs = _inputs(B, H, dtype=dtype, seed=7)
    projs = [p.clone() for p in projs]
    projs[0][0, 0, 3:9, 4:12] = 2.0        # a plateau at the maximum, starting mid-row
    projs[0][1, 0, 20:, :] = 2.0           # a plateau over whole rows
    projs[1][:, 0, 5, 7] = 3.0             # two separated maxima of equal value
    projs[1][:, 0, 17, 2] = 3.0
    projs[2].zero_()                       # not visible: the max is clamped to 1e-5 and passes no gradient
    projs[3][1].fill_(0.5)                 # one whole image at the maximum
    probs = _probs(B, dtype=dtype)
    got = _run(m, projs, segs, probs, True, True)
    ref = _run(m, [p.double() for p in projs], segs.double(), probs.double(), True, False)
    tol = 1e-12 if dtype == D else 1e-4
    for k, (a, b) in enumerate(zip(got[1], ref[1])):
        _cmp("grad%d" % k, a, b, tol, tol / 10)   # a max adjoint on another plateau pixel would differ by far more


# --- range --------------------------------------------------------------------------------------------------------------
def _guarded(n, dtype, guard=64):
    buf = torch.full((n + 2 * guard,), 1234.5, device=DEV, dtype=dtype)
    return buf, buf[guard:guard + n]


def _raw(projs, c0, segs, w, kld, gterms):
    """The C entry points on guard-banded outputs: (terms, grad_maps), each checked for untouched guards."""
    dt = 1 if segs.dtype == D else 0
    lib = _lib.load()
    B, _, H, _ = segs.shape
    planes = [ops._planes(p, H * H, segs.dtype) for p in projs]
    cz, cbs = ops._planes(c0, H * H, segs.dtype)
    w = w.detach().reshape(-1).to(segs.dtype).contiguous()
    tbuf, terms = _guarded(B * 2, segs.dtype)
    gbuf, gm = _guarded(B * 4 * H * H, segs.dtype)
    ws = torch.empty(lib.umr_part_head_workspace_bytes(B, H, dt), device=DEV, dtype=torch.uint8)
    mp = (ctypes.c_void_p * 4)(*[v.data_ptr() for v, _ in planes])
    mb = (ctypes.c_int64 * 4)(*[bs for _, bs in planes])
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    assert lib.umr_part_head_forward(mp, mb, p(cz), cbs, p(segs), 5 * H * H, p(w), p(terms), B, H, kld, dt, p(ws), st) == 0
    g = gterms.to(segs.dtype).contiguous()
    assert lib.umr_part_head_backward(mp, mb, p(cz), cbs, p(segs), 5 * H * H, p(w), p(ws), p(g), p(gm), B, H, kld, dt,
                                      st) == 0
    torch.cuda.synchronize()
    for buf, n in ((tbuf, B * 2), (gbuf, B * 4 * H * H)):
        assert torch.all(buf[:64] == 1234.5) and torch.all(buf[64 + n:] == 1234.5)
    return terms.view(B, 2), gm.view(B, 4, H, H)


@pytest.mark.parametrize("H", [1, 2, 3, 31, 61, 64, 256, 512])
@pytest.mark.parametrize("B", [1, 2, 17])
@pytest.mark.parametrize("kld", [0, 1])
def test_range(H, B, kld):
    layout = ("single", "render4", "render5")[(H + B) % 3]
    projs, segs = _inputs(B, H, dtype=torch.float32, seed=H + B, layout=layout)
    m = _module(B, H, "kld" if kld else "mse")
    gterms = torch.rand(B, 2, generator=torch.Generator().manual_seed(H), dtype=D).to(DEV) - 0.5
    terms, gm = _raw(projs, m.proj[:B], segs, m.weights, kld, gterms)
    leaves = [p.detach().double().requires_grad_(True) for p in projs]
    ref = _terms_ref(leaves, m.proj[:B], segs, m.weights, kld)
    gref = torch.autograd.grad(ref, leaves, gterms)
    _cmp("terms", terms, ref, 2e-5, 1e-6)
    for k in range(4):
        _cmp("grad%d" % k, gm[:, k], gref[k][:, 0], 1e-3, 1e-5)
    # float64 at the same shape and layout
    projs64 = [p.double() for p in projs]
    t64, g64 = _raw(projs64, m.proj[:B], segs.double(), m.weights, kld, gterms)
    ref64 = _terms_ref(projs64, m.proj[:B], segs, m.weights, kld)
    _cmp("terms64", t64, ref64, 1e-10, 1e-12)
    for k in range(4):
        _cmp("grad64_%d" % k, g64[:, k], gref[k][:, 0], 1e-9, 1e-11)


@pytest.mark.parametrize("dtype", [torch.float32, D])
def test_largest_batch_and_offset_views(dtype):
    B, H = 65535, 2
    projs, segs = _inputs(B, H, dtype=dtype, seed=9)
    flat = torch.zeros(B * H * H + 1, device=DEV, dtype=dtype)          # a view at an odd element offset
    flat[1:] = projs[0].reshape(-1)
    projs[0] = flat[1:].view(B, 1, H, H)
    m = _module(B, H, "mse")
    gterms = torch.rand(B, 2, generator=torch.Generator().manual_seed(1), dtype=D).to(DEV)
    terms, gm = _raw(projs, m.proj[:B], segs, m.weights, 0, gterms)
    leaves = [p.detach().double().requires_grad_(True) for p in projs]
    ref = _terms_ref(leaves, m.proj[:B], segs, m.weights, 0)
    gref = torch.autograd.grad(ref, leaves, gterms)
    tol = (1e-11, 1e-13) if dtype == D else (2e-5, 1e-6)
    _cmp("terms", terms, ref, *tol)
    for k in range(4):
        _cmp("grad%d" % k, gm[:, k], gref[k][:, 0], tol[0] * 100, tol[1] * 100)


# --- part_matching_loss -------------------------------------------------------------------------------------------------
def _scene(n, IS=32, T=2, seed=11):
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(2)
    part = rng.integers(0, 5, size=(f.shape[0], T * T))
    one_hot = torch.zeros(1, f.shape[0], T * T, 5)
    one_hot.scatter_(3, torch.from_numpy(part)[None, :, :, None], 1.0)
    verts = torch.from_numpy(synth.bird_like(v, rng, n)).to(DEV)
    faces = torch.from_numpy(f.astype(np.int64))[None].repeat(n, 1, 1).to(DEV)
    cams = torch.from_numpy(synth.cameras(rng, n)).to(DEV)
    segs = torch.rand(n, 5, IS, IS, generator=torch.Generator().manual_seed(seed)).to(DEV)
    return one_hot, verts, faces, cams, segs


def _module_step(monkeypatch, branch, loss_type, avg, num_cam, kernels):
    B, IS, T = 2, 32, 2
    n = B * num_cam
    one_hot, verts, faces, cams, segs = _scene(n, IS, T)
    m = _module(n, IS, loss_type, T=T, one_hot=one_hot)
    with monkeypatch.context() as mp:
        if branch == "four":
            m.pack_parts = False
        elif branch == "two":
            mp.setattr(m.renderer, "_fusable", lambda v: False)
        if not kernels:
            mp.setattr(loss_utils, "part_head_on_device", lambda *a: False)
        vv, cc = verts.clone().requires_grad_(True), cams.clone().requires_grad_(True)
        probs = _probs(n, num_cam, torch.float32)
        loss, projs = m(vv, faces, cc, segs, cam_probs=None if avg else probs, avg=avg)
        gv, gc = torch.autograd.grad(loss, (vv, cc))
    return loss.detach(), [p.detach() for p in projs], gv, gc


@pytest.mark.parametrize("branch", ["packed", "two", "four"])
@pytest.mark.parametrize("loss_type", ["mse", "kld"])
@pytest.mark.parametrize("avg,num_cam", [(True, 1), (False, 1), (False, 8)])
def test_module_branches(monkeypatch, branch, loss_type, avg, num_cam):
    got = _module_step(monkeypatch, branch, loss_type, avg, num_cam, True)
    ref = _module_step(monkeypatch, branch, loss_type, avg, num_cam, False)
    for a, b in zip(got[1], ref[1]):
        assert torch.equal(a, b)                  # projs: today's values bit for bit
    assert abs(float(got[0]) - float(ref[0])) <= 1e-6 * max(1.0, abs(float(ref[0])))
    _cmp("d/dverts", got[2], ref[2], 1e-3, 1e-5)
    _cmp("d/dcams", got[3], ref[3], 1e-3, 1e-5)


def test_projs_stay_differentiable(monkeypatch):
    one_hot, verts, faces, cams, segs = _scene(2)
    m = _module(2, 32, T=2, one_hot=one_hot)
    vv = verts.clone().requires_grad_(True)
    _, projs = m(vv, faces, cams, segs)
    assert all(p.requires_grad for p in projs)
    assert torch.autograd.grad(sum(p.sum() for p in projs), vv)[0].abs().sum() > 0


# --- reproducibility, capture, launches, memory -------------------------------------------------------------------------
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("loss_type", ["mse", "kld"])
def test_bitwise_reproducible(det, loss_type):
    B, H = 16, 256
    m = _module(B, H, loss_type)
    projs, segs = _inputs(B, H, dtype=torch.float32, seed=13)
    probs = _probs(B, dtype=torch.float32)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        a = _run(m, projs, segs, probs, False, True)
        b = _run(m, projs, segs, probs, False, True)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert torch.equal(a[0], b[0]) and all(torch.equal(x, y) for x, y in zip(a[1], b[1]))


@pytest.mark.parametrize("loss_type", ["mse", "kld"])
def test_cuda_graph_capture(loss_type):
    B, H = 4, 64
    m = _module(B, H, loss_type)
    projs, segs = _inputs(B, H, dtype=torch.float32, seed=17)
    leaves = _leaves(projs)
    probs = _probs(B, dtype=torch.float32)

    def step():
        loss = m.head(leaves, segs, probs, False)
        return (loss,) + torch.autograd.grad(loss, leaves)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    graph.replay()
    torch.cuda.synchronize()
    eager = step()
    assert all(torch.equal(a, b) for a, b in zip(out, eager))


@pytest.mark.parametrize("loss_type,fwd", [("mse", 4), ("kld", 2)])
def test_launch_counts(loss_type, fwd):
    lib = _lib.load()
    B, H = 2, 64
    m = _module(B, H, loss_type)
    projs, segs = _inputs(B, H, dtype=torch.float32)
    leaves = _leaves(projs)
    n0 = lib.umr_launch_count()
    terms = ops.part_matching_head(leaves, m.proj[:B], segs, m.weights, loss_type == "kld")
    n1 = lib.umr_launch_count()
    torch.autograd.grad(terms.sum(), leaves)
    n2 = lib.umr_launch_count()
    assert (n1 - n0, n2 - n1) == (fwd, 1)
    assert fwd <= 4


def test_peak_memory():
    B, H = 16, 256
    m = _module(B, H, "mse")
    projs, segs = _inputs(B, H, dtype=torch.float32, seed=19)
    leaves = _leaves(projs)
    probs = _probs(B, dtype=torch.float32)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    loss = m.head(leaves, segs, probs, False)
    grads = torch.autograd.grad(loss, leaves)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    plane = B * H * H * 4
    assert peak <= 4 * plane + 5 * plane, (peak, plane)   # the four map gradients + one [B,5,H,W] tensor
    assert len(grads) == 4
