"""The float64 loss kernels (umr_b200/csrc/losses_f64.cu, DESIGN.md §10) on the GPU.

* Values against float64 CPU references: oracle/loss_ref.py where it offers a magnitude evaluation (IoU, masked L1,
  chamfer, TexCycle, Laplacian), with the bound gamma_n * magnitude at u = 2^-53 and n counted generously from the
  kernel's longest chain of roundings plus the reference's own; the other values and every gradient against the same
  references (oracle/losses.py, torch's grid_sample in double, autograd) within tolerances a few hundred ulp wide.
* The sampler's forward against torch.nn.functional.grid_sample in double on the GPU: within a few ulp on dyadic
  coordinates, plus the rounding of the coordinate map on random ones.
* torch.autograd.gradcheck with nondet_tol=0 for every differentiable input.
* Bitwise reproducibility across runs, the deterministic flag on and off, host threads on side streams and CUDA-graph
  replay.
* The dtype rule: mixed float32 / float64 inputs compute in float64 and give each gradient in its input's dtype, half
  inputs still give float32, and a float32 call gives the same bytes before and after a float64 call.
* End to end: the train_s2-shaped loss step with float64 leaves is float64, finite and bitwise reproducible; gradcheck of
  MultiTextureLoss with respect to the texture flow and the camera probabilities.
"""
import threading

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

import loss_ref as R
import losses as LO
from umr_b200 import ops, synth
from umr_b200 import soft_renderer as sr
from umr_b200.nnutils import chamfer_python, geom_utils, loss_utils
from util import rel_report

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D = torch.float64
U64 = 2.0 ** -53


def g64(n):
    return n * U64 / (1 - n * U64)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _leaves(*ts):
    return [t.to(DEV, D).requires_grad_(True) for t in ts]


def _bound(name, got, ref, mag, n):
    """|got - ref| <= gamma_n(2^-53) * mag everywhere (NaN fails); prints the largest error / bound ratio."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    bound = g64(n) * mag.detach().double().cpu().expand_as(ref) + 1e-300
    err = (got - ref).abs()
    ratio = float((err / bound).max()) if err.numel() else 0.0
    print("%-48s max err/bound = %.3e" % (name, ratio))
    assert bool(torch.isfinite(got).all()), name + ": non-finite"
    assert ratio <= 1.0, "%s: outside gamma_%d bound, ratio %.3g" % (name, n, ratio)


def _within(name, got, ref, bound):
    """|got - ref| <= bound everywhere (NaN fails)."""
    err = (got.detach().double().cpu() - ref.detach().double().cpu()).abs()
    ratio = float((err / (bound.detach().double().cpu() + 1e-300)).max())
    print("%-48s max err/bound = %.3e" % (name, ratio))
    assert bool(torch.isfinite(got).all()) and ratio <= 1.0, "%s: ratio %.3g" % (name, ratio)


def _close(name, got, ref, rtol=1e-12, ascale=1e-13):
    """A tolerance of a few hundred to a few thousand float64 ulp of the largest reference value."""
    got, ref = got.detach().double().cpu().numpy(), ref.detach().double().cpu().numpy()
    ok, msg = rel_report(name, got, ref, rtol, ascale * float(np.abs(ref).max()) + 1e-300)
    print(msg)
    assert ok and np.isfinite(got).all(), msg


# -------------------------------------------------------------------------------------------------
# per-op cases: fn(*leaves) -> [outputs..., leaf gradients...] (the thing compared bitwise); check(outs) compares with
# the float64 CPU reference
# -------------------------------------------------------------------------------------------------
def sampler_case(C, H, W, N=1000, B=2):
    g = _gen(C * 100 + H * 10 + W)
    img = torch.rand(B, C, H, W, generator=g, dtype=D) * 2 - 1
    flow = torch.rand(B, N, 2, generator=g, dtype=D) * 2.4 - 1.2
    flow[:, :8] = torch.tensor([[-1.0, -1.0], [1.0, 1.0], [1.0, -1.0], [-1.0, 1.0], [0.0, 0.0], [1e6, 0.5], [-1e6, -1e6],
                                [0.3, 1.0 + 2 ** -40]], dtype=D)
    w = torch.rand(B, N, C, generator=g, dtype=D)
    wd = w.to(DEV)

    def fn(x, f):
        x.grad = f.grad = None
        out = ops.bilinear_sample(x, f)
        (out * wd).sum().backward()
        return [out, x.grad, f.grad]

    def check(outs):
        out, gi, gf = outs
        xr, fr = img.clone().requires_grad_(True), flow.clone().requires_grad_(True)
        ref = TF.grid_sample(xr, fr[:, :, None], mode="bilinear", padding_mode="zeros", align_corners=True)[..., 0]
        (ref.permute(0, 2, 1) * w).sum().backward()
        mag = TF.grid_sample(img.abs(), flow[:, :, None], align_corners=True)[..., 0].permute(0, 2, 1)
        # torch's CPU kernel maps coordinates as (x + 1) * ((W - 1) / 2): the weights then differ by ~u * |ix|
        k = 4 * max(H, W)
        _bound("sampler C%d %dx%d value" % (C, H, W), out, ref.permute(0, 2, 1), mag, 8 + k)
        xm = img.abs().clone().requires_grad_(True)
        (TF.grid_sample(xm, flow[:, :, None], align_corners=True)[..., 0].permute(0, 2, 1) * w).sum().backward()
        _bound("sampler C%d %dx%d grad_image" % (C, H, W), gi, xr.grad, xm.grad, N + 16 + k)
        scale = torch.tensor([(W - 1) / 2, (H - 1) / 2], dtype=D)
        fmag = (w.sum(-1, keepdim=True) * 2 * img.abs().max()) * scale + 1e-300
        _bound("sampler C%d %dx%d grad_flow" % (C, H, W), gf, fr.grad, fmag, 4 * C + 16)
    return fn, _leaves(img, flow), check


def iou_case(B, H, W, strided, kind="random"):
    g = _gen(2 + H)
    p = torch.rand(B, 4, H, W, generator=g, dtype=D) if strided else torch.rand(B, H, W, generator=g, dtype=D)
    t = (torch.rand(B, H, W, generator=g, dtype=D) > 0.5).to(D)
    if kind == "empty":
        t.zero_()
        (p[:, 3] if strided else p).zero_()
    elif kind == "full":
        t.fill_(1)
    w = torch.rand(B, generator=g, dtype=D)
    td, wd = t.to(DEV), w.to(DEV)

    def fn(x):
        x.grad = None
        loss = loss_utils.neg_iou_loss(x[:, 3] if strided else x, td, avg=False)
        (loss * wd).sum().backward()
        return [loss, x.grad]

    def check(outs):
        loss, gx = outs
        xr = p.clone().requires_grad_(True)
        pa = xr[:, 3] if strided else xr
        ref, I, U = R.iou_ref(pa, t)
        (ref * w).sum().backward()
        _, Im, Um = R.iou_ref(pa.detach(), t, magnitude=True)
        n = H * W // 256 + 64
        # 1 - I/U: |err| <= (dI + |I/U| dU) / U + 2 u, with dI, dU <= gamma_n times the magnitudes
        _bound("iou %s value" % kind, loss, ref, (Im + (I / U).abs() * Um) / U + 2.0, n)
        _close("iou %s grad" % kind, gx, xr.grad, 1e-11, 1e-12)
    return fn, _leaves(p), check


def masked_l1_case(B, H, W, C):
    g = _gen(5 + C)
    rgba = torch.rand(B, 4, H, W, generator=g, dtype=D)
    gt = torch.rand(B, C, H, W, generator=g, dtype=D)
    mgt = (torch.rand(B, H, W, generator=g, dtype=D) > 0.4).to(D)
    w = torch.rand(B, generator=g, dtype=D)
    gtd, md, wd = gt.to(DEV), mgt.to(DEV), w.to(DEV)

    def fn(x):
        x.grad = None
        loss = loss_utils.texture_loss_masks(x[:, :C], gtd, md, x[:, 3], avg=False)   # strided views of the render
        (loss * wd).sum().backward()
        return [loss, x.grad]

    def check(outs):
        loss, gx = outs
        r = rgba.clone().requires_grad_(True)
        ref = R.masked_l1_ref(r[:, :C], gt, mgt, r[:, 3])
        (ref * w).sum().backward()
        mag = R.masked_l1_ref(rgba[:, :C], gt, mgt, rgba[:, 3], magnitude=True)
        _bound("masked_l1 C%d value" % C, loss, ref, mag, C * H * W // 256 + 64)
        _close("masked_l1 C%d grad" % C, gx, r.grad, 1e-14, 1e-15)
    return fn, _leaves(rgba), check


def loss_head_case(B, H):
    g = _gen(6 + B)
    rgba = torch.rand(B, 4, H, H, generator=g, dtype=D)
    gt = torch.rand(B, 3, H, H, generator=g, dtype=D)
    mgt = (torch.rand(B, H, H, generator=g, dtype=D) > 0.4).to(D)
    gtd, md = gt.to(DEV), mgt.to(DEV)

    def fn(x):
        x.grad = None
        loss, per_image = ops.mask_texture_loss(x, gtd, md, 2.5, 3.0)
        (loss * 1.7).backward()
        return [loss, per_image, x.grad]

    def check(outs):
        loss, per_image, gx = outs
        r = rgba.clone().requires_grad_(True)
        ref, per = R.loss_head_ref(r, gt, mgt, 2.5, 3.0)
        (ref * 1.7).backward()
        _close("loss_head value", loss, ref)
        _close("loss_head per_image", per_image, per)
        _close("loss_head grad", gx, r.grad, 1e-11, 1e-12)
    return fn, _leaves(rgba), check


def chamfer_case(B, N, M, Dm, dup=False):
    g = _gen(3 + N)
    a = torch.rand(B, N, Dm, generator=g, dtype=D) - 0.5
    b = torch.rand(B, M, Dm, generator=g, dtype=D) - 0.5
    if dup:
        b[:, 1::2] = b[:, 0::2][:, :b[:, 1::2].shape[1]]   # duplicate points: ties resolved to the lower index
    w1, w2 = torch.rand(B, N, generator=g, dtype=D), torch.rand(B, M, generator=g, dtype=D)
    w1d, w2d = w1.to(DEV), w2.to(DEV)

    def fn(x, y):
        x.grad = y.grad = None
        o = chamfer_python.distChamfer(x, y)
        ((o[0] * w1d).sum() + (o[1] * w2d).sum()).backward()
        return [o[0], o[1], o[2], o[3], x.grad, y.grad]

    def check(outs):
        d1, d2, i1, i2, ga, gb = outs
        _, _, r1, r2 = R.chamfer_ref(a, b)
        assert bool(R.near_tie(a, b, i1, r1, 2).all()) and bool(R.near_tie(b, a, i2, r2, 2).all())
        ar, br = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
        e1, e2, _, _ = R.chamfer_ref(ar, br, i1.long(), i2.long())   # the kernel's (near-tie) choices
        ((e1 * w1).sum() + (e2 * w2).sum()).backward()
        m1, m2, _, _ = R.chamfer_ref(a.abs(), b.abs(), i1.long(), i2.long(), magnitude=True)
        _bound("chamfer d_ab", d1, e1, m1, 2 * Dm + 4)
        _bound("chamfer d_ba", d2, e2, m2, 2 * Dm + 4)
        _close("chamfer grad_a", ga, ar.grad, 1e-11, 1e-12)
        _close("chamfer grad_b", gb, br.grad, 1e-11, 1e-12)
    return fn, _leaves(a, b), check


def texcycle_case(B, F, T, P, source):
    g = _gen(4 + F)
    flow = torch.rand(B, F, T, T, 2, generator=g, dtype=D) * 2 - 1
    prob = torch.rand(B, F, 2, generator=g, dtype=D) * 2 - 1
    ids = torch.randint(-1, F // 2, (B, P), generator=g).to(D)   # -1 = background, upper half never visible
    ids[0, :3] = torch.tensor([F + 3.0, -F - 2.0, 2.0 ** 23], dtype=D)   # ids naming no face mark nothing
    vis = R.visible_ref(ids, F)
    probd, idsd, visd = prob.to(DEV), ids.to(DEV), vis.to(torch.uint8).to(DEV)

    def fn(x):
        x.grad = None
        if source == "visible":
            loss, _ = loss_utils.TexCycle()(x, probd, None, visible=visd)
        else:
            loss, _ = loss_utils.TexCycle()(x, probd, idsd if source == "plane64" else idsd.float())
        loss.backward()
        return [loss, x.grad]

    def check(outs):
        loss, gx = outs
        fr = flow.clone().requires_grad_(True)
        ref = R.texcycle_ref(fr.reshape(B, F, T * T, 2), prob, vis)
        ref.backward()
        mag = R.texcycle_ref(flow.reshape(B, F, T * T, 2), prob, vis, magnitude=True)
        _bound("texcycle %s value" % source, loss, ref, mag, B * F // 256 + T * T + 64)
        _close("texcycle %s grad" % source, gx, fr.grad, 1e-12, 1e-13)
    return fn, _leaves(flow), check


def _mesh(kind, B):
    v, f = R.spiked_uv_sphere(9, 13, 7)
    rng = np.random.default_rng(7)
    verts = torch.from_numpy(v[None] * rng.uniform(0.8, 1.2, size=(B, v.shape[0], 3))).to(D)
    faces = torch.from_numpy(f)
    w = torch.from_numpy(rng.uniform(0.5, 1.5, size=(B,)))
    mod = (sr.LaplacianLoss(torch.from_numpy(v), faces) if kind == "laplacian" else sr.FlattenLoss(faces)).to(DEV)
    wd = w.to(DEV)

    def fn(x):
        x.grad = None
        loss = mod(x)
        (loss * wd).sum().backward()
        return [loss, x.grad]

    def check(outs):
        loss, gx = outs
        xr = verts.clone().requires_grad_(True)
        if kind == "laplacian":
            rp, col, coef = mod.csr_rowptr.cpu(), mod.csr_col.cpu(), mod.csr_coef.cpu()
            ref, _ = R.laplacian_ref(xr, rp, col, coef)
            (ref * w).sum().backward()
            xm = verts.abs().clone().requires_grad_(True)
            mag, _ = R.laplacian_ref(xm, rp, col, coef, magnitude=True)
            (mag * w).sum().backward()
            deg = int(torch.diff(rp.long()).max())
            _bound("laplacian value", loss, ref, mag, 2 * deg + v.shape[0] // 256 + 64)
            _bound("laplacian grad", gx, xr.grad, xm.grad, 4 * deg + 64)
        else:
            edges = mod.edge_table.cpu()
            ref = R.flatten_ref(xr, edges)
            (ref * w).sum().backward()
            lb, gb = R.flatten_error_bound(verts, edges, 1e-6, w, edges.shape[0] // 128 + 16, R.U64)
            _within("flatten value", loss, ref, lb)
            _within("flatten grad", gx, xr.grad, gb)
    return fn, _leaves(verts), check


def corr_case(shared):
    rng = np.random.default_rng(17)
    B, IS = 6, 64
    v, f = synth.icosphere(3)
    V = v.shape[0]
    parts = [torch.from_numpy(p) for p in synth.part_vertex_sets(rng, V, sizes=(20, 40, 20, 40))]
    parts[1] = torch.cat((parts[1], parts[0][:5]))   # vertices listed in two parts
    pts = [torch.from_numpy(p).to(DEV, D) for p in synth.part_points(rng, B)]
    m = loss_utils.CorrLossChamfer(None, IS, part_vertices=parts)
    m.weights = [1, 1, 0.5, 0.25]
    base = torch.from_numpy(synth.bird_like(v, rng, B)).to(D)
    cams0 = torch.from_numpy(synth.cameras(rng, B)).to(D)
    lw = torch.linspace(0.5, 1.5, B, device=DEV, dtype=D)

    def fn(leaf, cams):
        leaf.grad = cams.grad = None
        verts = leaf[None].expand(B, -1, -1) if shared else leaf
        loss = m(pts[0], pts[1], pts[2], pts[3], verts, cams, avg=False)
        (loss * lw).sum().backward()
        return [loss, leaf.grad, cams.grad]

    def check(outs):
        # the reference composition (projection, distChamfer per part, weighted mean) in double torch on the CPU
        leaf, cams = base[0] if shared else base, cams0
        lr, cr = leaf.clone().requires_grad_(True), cams.clone().requires_grad_(True)
        verts = lr[None].expand(B, -1, -1) if shared else lr
        idx = torch.cat([p.long() for p in parts])
        v2d = LO.orthographic_proj_withz(verts[:, idx], cr)[:, :, :2]
        terms, start = [], 0
        for p, t, wgt in zip(parts, pts, m.weights):
            d, _, _, _ = LO.dist_chamfer(v2d[:, start:start + len(p)], t.cpu())
            terms.append(d * wgt)
            start += len(p)
        ref = torch.cat(terms, 1).mean(1)
        (ref * lw.cpu()).sum().backward()
        _close("corr value", outs[0], ref, 1e-11, 1e-12)
        _close("corr grad_verts", outs[1], lr.grad, 1e-10, 1e-11)
        _close("corr grad_cams", outs[2], cr.grad, 1e-10, 1e-11)
    return fn, _leaves(base[0] if shared else base, cams0), check


CASES = {
    "sampler_c1_1x7": lambda: sampler_case(1, 1, 7),
    "sampler_c2_6x1": lambda: sampler_case(2, 6, 1),
    "sampler_c3_17x23": lambda: sampler_case(3, 17, 23),
    "sampler_c4_17x23": lambda: sampler_case(4, 17, 23),
    "iou_odd_strided": lambda: iou_case(3, 37, 41, True),
    "iou_2048_plus_1": lambda: iou_case(2, 1, 2049, False),
    "iou_empty": lambda: iou_case(2, 64, 64, True, "empty"),
    "iou_full": lambda: iou_case(2, 64, 65, False, "full"),
    "masked_l1_c1": lambda: masked_l1_case(3, 37, 41, 1),
    "masked_l1_c3": lambda: masked_l1_case(2, 128, 129, 3),
    "loss_head_b1": lambda: loss_head_case(1, 45),
    "loss_head_b33": lambda: loss_head_case(33, 64),
    "chamfer_d2": lambda: chamfer_case(3, 1000, 333, 2),
    "chamfer_d3_dup": lambda: chamfer_case(2, 33, 70, 3, dup=True),
    "chamfer_large": lambda: chamfer_case(1, 20000, 642, 3),
    "texcycle_plane64": lambda: texcycle_case(3, 300, 3, 37 * 41, "plane64"),
    "texcycle_plane32": lambda: texcycle_case(3, 300, 3, 37 * 41, "plane32"),
    "texcycle_visible": lambda: texcycle_case(3, 300, 3, 37 * 41, "visible"),
    "laplacian": lambda: _mesh("laplacian", 5),
    "flatten": lambda: _mesh("flatten", 5),
    "corr_shared": lambda: corr_case(True),
    "corr_per_render": lambda: corr_case(False),
}


def _host(outs):
    return [None if o is None else o.detach().cpu() for o in outs]


def _run(fn, leaves, stream=None):
    with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream()):
        outs = fn(*leaves)
    torch.cuda.synchronize()
    return _host(outs)


def _assert_equal(a, b, what):
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        assert x.dtype == y.dtype and torch.equal(x, y), "%s: output %d differs bitwise" % (what, k)


def _graph_replays(fn, leaves, ref):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):   # warm-up outside the capture (module caches, allocator)
            fn(*leaves)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = fn(*leaves)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        _assert_equal(ref, _host(outs), "graph replay")


@pytest.fixture
def flag_restored():
    prev = torch.are_deterministic_algorithms_enabled()
    yield
    torch.use_deterministic_algorithms(prev)


@pytest.mark.parametrize("name", list(CASES))
def test_against_reference_and_reproducible(flag_restored, name):
    fn, leaves, check = CASES[name]()
    torch.use_deterministic_algorithms(False)
    ref = _run(fn, leaves)
    for o in ref:
        assert o.dtype in (torch.float64, torch.int32), o.dtype
    check(ref)
    _assert_equal(ref, _run(fn, leaves), "run")
    torch.use_deterministic_algorithms(True)
    _assert_equal(ref, _run(fn, leaves), "deterministic flag")
    torch.use_deterministic_algorithms(False)
    results = [None] * 3

    def work(i):
        st = torch.cuda.Stream(device=DEV)
        with torch.cuda.stream(st):
            mine = [l.detach().clone().requires_grad_(True) for l in leaves]
        st.synchronize()
        results[i] = _run(fn, mine, st)

    ts = [threading.Thread(target=work, args=(i,)) for i in range(3)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for r in results:
        _assert_equal(ref, r, "thread")
    _graph_replays(fn, leaves, ref)


def test_sampler_matches_grid_sample_on_gpu():
    """The forward against torch's own CUDA grid_sample in double.  On dyadic coordinates (x = -1 + m / 1024, whose pixel
    coordinate ((x + 1) / 2) * (W - 1) is exact in any evaluation order) the two may differ only in how the four corner
    terms are rounded and summed: within gamma_8 of the sample's magnitude, a few ulp.  A wrong coordinate map (the other
    align_corners convention, a half-pixel shift) is off by a large fraction of a texel there.  On random coordinates the
    pixel coordinate itself is rounded (u * |ix|), and each weight may move by that much between two evaluations."""
    for C, H, W in ((1, 1, 7), (3, 17, 23), (4, 64, 33)):
        g = _gen(C + H)
        img = (torch.rand(2, C, H, W, generator=g, dtype=D) * 2 - 1).to(DEV)
        dyadic = (torch.randint(-200, 2249, (2, 3001, 2), generator=g).to(D) / 1024 - 1).to(DEV)
        rand = (torch.rand(2, 3001, 2, generator=g, dtype=D) * 2.4 - 1.2).to(DEV)
        for kind, flow, n in (("dyadic", dyadic, 8), ("random", rand, 8 + 4 * max(H, W))):
            ours = ops.bilinear_sample(img, flow)
            ref = TF.grid_sample(img, flow[:, :, None], align_corners=True)[..., 0].permute(0, 2, 1)
            mag = TF.grid_sample(img.abs(), flow[:, :, None], align_corners=True)[..., 0].permute(0, 2, 1)
            _bound("grid_sample cuda C%d %s" % (C, kind), ours, ref, mag, n)


# -------------------------------------------------------------------------------------------------
# gradcheck
# -------------------------------------------------------------------------------------------------
def _gc(fn, *inputs):
    assert torch.autograd.gradcheck(fn, inputs, eps=1e-6, atol=1e-7, rtol=1e-5, nondet_tol=0.0)


def test_gradcheck_ops():
    g = _gen(11)
    r = lambda *s: (torch.rand(*s, generator=g, dtype=D)).to(DEV).requires_grad_(True)   # noqa: E731
    img = r(2, 3, 5, 6)
    flow = (torch.rand(2, 17, 2, generator=g, dtype=D) * 1.8 - 0.9 + 1e-3).to(DEV).requires_grad_(True)
    _gc(lambda a, b: ops.bilinear_sample(a, b), img, flow)
    t = (torch.rand(2, 5, 7, generator=g, dtype=D) > 0.5).to(D).to(DEV)
    _gc(lambda p: ops.neg_iou_per_image(p, t), r(2, 5, 7))
    rgba, gt = r(2, 4, 5, 7), torch.rand(2, 3, 5, 7, generator=g, dtype=D).to(DEV)
    _gc(lambda x: ops.masked_l1_per_image(x[:, :3], gt, t, x[:, 3]), rgba)
    _gc(lambda x: ops.mask_texture_loss(x, gt, t, 2.0, 0.5)[0], rgba)
    a, b = r(2, 9, 3), r(2, 11, 3)
    _gc(lambda x, y: ops.dist_chamfer(x, y)[:2], a, b)
    fl, pr = r(2, 7, 4, 2), torch.rand(2, 7, 2, generator=g, dtype=D).to(DEV)
    vis = (torch.arange(14, device=DEV).view(2, 7) % 3 != 0).to(torch.uint8)
    _gc(lambda x: ops.tex_cycle(x, pr, None, vis), fl)
    v, f = synth.icosphere(1)
    x0 = torch.from_numpy(v).to(DEV, D)
    x = (x0[None] * (1 + 0.1 * torch.rand(2, v.shape[0], 3, generator=g, dtype=D).to(DEV))).requires_grad_(True)
    faces = torch.from_numpy(f.astype(np.int64))
    lap, flat = sr.LaplacianLoss(torch.from_numpy(v), faces).to(DEV), sr.FlattenLoss(faces).to(DEV)
    _gc(lap, x)
    _gc(flat, x)
    rng = np.random.default_rng(3)
    parts = [torch.from_numpy(p) for p in synth.part_vertex_sets(rng, v.shape[0], sizes=(5, 6, 4, 3))]
    pts = [torch.from_numpy(p[:, :7]).to(DEV, D) for p in synth.part_points(rng, 2)]
    corr = loss_utils.CorrLossChamfer(None, 32, part_vertices=parts)
    cams = torch.from_numpy(synth.cameras(rng, 2)).to(DEV, D).requires_grad_(True)
    _gc(lambda xx, cc: corr(pts[0], pts[1], pts[2], pts[3], xx, cc, avg=False), x, cams)


# -------------------------------------------------------------------------------------------------
# dtype rule
# -------------------------------------------------------------------------------------------------
def test_mixed_dtypes_follow_the_rule():
    g = _gen(12)
    img32 = torch.rand(2, 3, 9, 8, generator=g).to(DEV).requires_grad_(True)
    flow64 = (torch.rand(2, 50, 2, generator=g, dtype=D) * 2 - 1).to(DEV).requires_grad_(True)
    out = ops.bilinear_sample(img32, flow64)
    assert out.dtype == D
    out.sum().backward()
    assert img32.grad.dtype == torch.float32 and flow64.grad.dtype == D
    ref = ops.bilinear_sample(img32.detach().double(), flow64.detach())   # same values as an all-float64 call
    assert torch.equal(out.detach(), ref)
    p32 = torch.rand(2, 4, 6, 7, generator=g).to(DEV).requires_grad_(True)
    m64 = (torch.rand(2, 6, 7, generator=g, dtype=D) > 0.5).to(D).to(DEV)
    loss = ops.neg_iou_per_image(p32[:, 3], m64)
    assert loss.dtype == D
    loss.sum().backward()
    assert p32.grad.dtype == torch.float32
    a32, b64 = torch.rand(1, 20, 3, generator=g).to(DEV).requires_grad_(True), torch.rand(1, 9, 3, dtype=D).to(DEV)
    d1, d2, _, _ = ops.dist_chamfer(a32, b64)
    assert d1.dtype == D and d2.dtype == D
    (d1.sum() + d2.sum()).backward()
    assert a32.grad.dtype == torch.float32
    fl32 = torch.rand(2, 5, 4, 2, generator=g).to(DEV).requires_grad_(True)
    ids64 = torch.randint(-1, 5, (2, 30), generator=g).to(DEV, D)
    loss = ops.tex_cycle(fl32, torch.rand(2, 5, 2).to(DEV), ids64)
    assert loss.dtype == D
    loss.backward()
    assert fl32.grad.dtype == torch.float32


def test_half_inputs_stay_float32():
    g = _gen(13)
    img = torch.rand(2, 3, 9, 8, generator=g).to(DEV).half().requires_grad_(True)
    flow = (torch.rand(2, 50, 2, generator=g) * 2 - 1).to(DEV).half()
    assert ops.bilinear_sample(img, flow).dtype == torch.float32
    p = torch.rand(2, 6, 7, generator=g).to(DEV).half()
    assert ops.neg_iou_per_image(p, (p > 0.5).half()).dtype == torch.float32
    a = torch.rand(1, 20, 3, generator=g).to(DEV).half()
    assert ops.dist_chamfer(a, a)[0].dtype == torch.float32


def test_float32_bytes_unchanged_by_a_float64_call():
    g = _gen(14)
    rgba = torch.rand(3, 4, 37, 41, generator=g).to(DEV)
    gt = torch.rand(3, 3, 37, 41, generator=g).to(DEV)
    m = (torch.rand(3, 37, 41, generator=g) > 0.5).float().to(DEV)
    a, b = torch.rand(2, 300, 3, generator=g).to(DEV), torch.rand(2, 77, 3, generator=g).to(DEV)

    def run(dtype):
        x, xa = rgba.to(dtype).clone().requires_grad_(True), a.to(dtype).clone().requires_grad_(True)
        loss, per = ops.mask_texture_loss(x, gt.to(dtype), m.to(dtype))
        d1, d2, i1, i2 = ops.dist_chamfer(xa, b.to(dtype))
        (loss + d1.sum() + d2.sum()).backward()
        torch.cuda.synchronize()
        return _host([loss, per, d1, d2, i1, i2, x.grad, xa.grad])

    before = run(torch.float32)
    assert run(D)[0].dtype == D
    _assert_equal(before, run(torch.float32), "float32 after float64")
    assert before[0].dtype == torch.float32 and before[6].dtype == torch.float32


# -------------------------------------------------------------------------------------------------
# end to end: the train_s2-shaped loss step (test_deterministic_losses_gpu's composition) with float64 leaves
# -------------------------------------------------------------------------------------------------
def make_step(B, H, IS, subdiv, T, seed, dtype):
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(subdiv)
    V, F = v.shape[0], f.shape[0]
    to = lambda a: torch.from_numpy(np.asarray(a)).to(DEV, dtype)   # noqa: E731
    fs = torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1).to(DEV)
    imgs, masks = to(synth.smooth_images(rng, B, IS)), to(synth.ellipse_masks(rng, B, IS))
    dts = to(np.stack([synth.dt_barrier(m) for m in masks.float().cpu().numpy()]))[:, None]
    part_segs = to(rng.uniform(0, 1, size=(B, 5, IS, IS)).astype(np.float32))   # float32 values in either precision
    part = rng.integers(0, 5, size=(F, T * T))
    one_hot = torch.zeros(1, F, T * T, 5)
    one_hot.scatter_(3, torch.from_numpy(part)[None, :, :, None], 1.0)
    part_vertices = [torch.from_numpy(p) for p in synth.part_vertex_sets(rng, V, sizes=(20, 40, 20, 40))]
    head, belly, neck, back = [to(p) for p in synth.part_points(rng, B)]
    rep = lambda t: t.unsqueeze(1).repeat(1, H, 1, 1).view(-1, t.size(1), t.size(2))   # noqa: E731
    mask_fn = loss_utils.MultiMaskLoss(IS, "softmax", H).to(DEV)
    tex_fn = loss_utils.MultiTextureLoss(B, H, IS, "softmax", "l1", "smr").to(DEV)
    part_fn = loss_utils.part_matching_loss(None, None, 0, im_size=IS, batch_size=B, tex_size=T, stex_one_hot=one_hot).to(DEV)
    corr_fn = loss_utils.CorrLossChamfer(None, IS, part_vertices=part_vertices)
    fcpu = torch.from_numpy(f.astype(np.int64))
    lap_fn, flat_fn = sr.LaplacianLoss(torch.from_numpy(v), fcpu).to(DEV), sr.FlattenLoss(fcpu).to(DEV)
    leaves = [to(v.astype(np.float32)), to(0.05 * (synth.bird_like(v, rng, B) - v[None])),
              to(np.stack([synth.cameras(rng, H) for _ in range(B)])), to(rng.normal(size=(B, H)).astype(np.float32)),
              to(synth.texture_flow(rng, B, F, T))]
    leaves = [t.requires_grad_(True) for t in leaves]   # mean shape, deformation, cameras, camera logits, texture flow

    def step(mean_shape, delta, cams, logits, flow):
        for t in (mean_shape, delta, cams, logits, flow):
            t.grad = None
        pred_vs = mean_shape[None] + delta
        probs = torch.softmax(logits, 1)
        proj_cam = cams[:, 0].detach()
        mask_loss, mask_all = mask_fn(pred_vs, fs, cams, probs, masks)
        tri = lap_fn(pred_vs).mean()
        flat = flat_fn(pred_vs).mean()
        tex = geom_utils.sample_textures(flow, imgs).contiguous().view(B, F, T * T, 3)
        tl, tdt, tcyc, _ = tex_fn(pred_vs.detach(), fs, cams.detach(), probs.detach(), proj_cam, imgs, masks, mask_all,
                                  tex, flow, dts)
        pl, _ = part_fn(pred_vs, fs, proj_cam, part_segs)
        ms_rep = mean_shape[None].expand(B, -1, -1).unsqueeze(1).repeat(1, H, 1, 1).view(-1, V, 3)
        corr = corr_fn(rep(head), rep(belly), rep(back), rep(neck), ms_rep, cams.view(-1, 7), avg=False)
        corr = (corr.view(B, H) * probs).sum(1).mean()
        losses = [mask_loss, tri, flat, tl, tdt, tcyc, pl, corr]
        total = mask_loss.mean() + 0.1 * tri + 0.005 * flat + 3.0 * tl.mean() + 3.0 * tdt.mean() + tcyc.mean() \
            + 0.1 * pl.mean() + corr
        total.backward()
        return [total] + [l.detach() for l in losses] + [t.grad for t in (mean_shape, delta, cams, logits, flow)]
    return step, leaves


def test_whole_step_float64(flag_restored):
    step, leaves = make_step(2, 8, 32, 2, 3, 21, D)
    ref = _run(step, leaves)
    for k, o in enumerate(ref):
        assert o.dtype == D, "step output %d is %s" % (k, o.dtype)
        assert bool(torch.isfinite(o).all()), "step output %d not finite" % k
    _assert_equal(ref, _run(step, leaves), "step run")
    torch.use_deterministic_algorithms(True)
    _assert_equal(ref, _run(step, leaves), "step deterministic flag")


def test_gradcheck_multi_texture_loss():
    """MultiTextureLoss with respect to the texture flow and the camera probabilities, everything in double."""
    rng = np.random.default_rng(5)
    B, H, IS, T = 1, 2, 16, 2
    v, f = synth.icosphere(1)
    F = f.shape[0]
    to = lambda a: torch.from_numpy(np.asarray(a)).to(DEV, D)   # noqa: E731
    vs, fs = to(synth.bird_like(v, rng, B)), torch.from_numpy(f.astype(np.int64))[None].to(DEV)
    cams = to(np.stack([synth.cameras(rng, H) for _ in range(B)]))
    imgs, masks = to(synth.smooth_images(rng, B, IS)), to(synth.ellipse_masks(rng, B, IS))
    dts = to(np.stack([synth.dt_barrier(m) for m in masks.float().cpu().numpy()]))[:, None]
    masks_pred = to(rng.uniform(0, 1, size=(B * H, IS, IS)))
    m = loss_utils.MultiTextureLoss(B, H, IS, "softmax", "l1", "smr").to(DEV)
    flow = to(synth.texture_flow(rng, B, F, T)).requires_grad_(True)
    probs = torch.softmax(to(rng.normal(size=(B, H))), 1).requires_grad_(True)

    def fn(fl, pr):
        tx = geom_utils.sample_textures(fl, imgs).contiguous().view(B, F, T * T, 3)
        tl, tdt, tcyc, _ = m(vs, fs, cams, pr, cams[:, 0], imgs, masks, masks_pred, tx, fl, dts)
        return 3.0 * tl + 3.0 * tdt + tcyc

    assert fn(flow, probs).dtype == D
    _gc(fn, flow, probs)
