"""Deterministic mode of the loss kernels (torch.use_deterministic_algorithms(True), include/umr_b200.h): every new entry
point's outputs and gradients are bitwise equal across runs, host threads on side streams and CUDA-graph replay, and agree
with the default path and the CPU oracles under the gates of test_losses_gpu / test_mesh_ops_gpu; the train_s2-shaped
loss step (at test_train_step_gpu's scene shape and tools/train_step_bench.py's default shape) is bitwise reproducible;
with the flag off every op launches what it launched before the mode existed."""
import os

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # the generic SoftRenderer chain's matmul (README)

import threading  # noqa: E402

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

import losses as LO  # noqa: E402  oracle/losses.py (test infrastructure)
import mesh_oracle as MO  # noqa: E402  oracle/mesh_oracle.py
from umr_b200 import _lib, ops, synth  # noqa: E402
from umr_b200 import soft_renderer as sr  # noqa: E402
from umr_b200.nnutils import chamfer_python, geom_utils, loss_utils  # noqa: E402
from util import rel_report  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture
def det():
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(old)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _leaves(*ts):
    return [t.to(DEV, torch.float32).requires_grad_(True) for t in ts]


# -------------------------------------------------------------------------------------------------
# one case per entry point and shape: fn(*leaves) -> outputs (values, then leaf gradients); oracle() -> CPU references;
# tols: (rtol, atol) per output, the gates test_losses_gpu / test_mesh_ops_gpu use for the same quantity
# -------------------------------------------------------------------------------------------------
def iou_case(B, H, W, strided):
    g = _gen(2)
    p = torch.rand(B, 4, H, W, generator=g) if strided else torch.rand(B, H, W, generator=g)
    t = (torch.rand(B, H, W, generator=g) > 0.5).float()
    w = torch.rand(B, generator=g)
    td, wd = t.to(DEV), w.to(DEV)

    def fn(x):
        x.grad = None
        loss = loss_utils.neg_iou_loss(x[:, 3] if strided else x, td, avg=False)   # [:, 3]: the strided alpha plane
        (loss * wd).sum().backward()
        return [loss, x.grad]

    def oracle():
        xr = p.clone().requires_grad_(True)
        ref = LO.neg_iou_loss(xr[:, 3] if strided else xr, t, avg=False)
        (ref * w).sum().backward()
        return [ref, xr.grad]
    return fn, _leaves(p), oracle, [(1e-4, 1e-6), (1e-4, 1e-10)]


def masked_l1_case(B, H, W, C):
    g = _gen(5)
    rgba = torch.rand(B, 4, H, W, generator=g)
    gt = torch.rand(B, C, H, W, generator=g)
    mgt = (torch.rand(B, H, W, generator=g) > 0.4).float()
    w = torch.rand(B, generator=g)
    gtd, md, wd = gt.to(DEV), mgt.to(DEV), w.to(DEV)

    def fn(x):
        x.grad = None
        loss = loss_utils.texture_loss_masks(x[:, :C], gtd, md, x[:, 3], avg=False)   # strided views of the render
        (loss * wd).sum().backward()
        return [loss, x.grad]

    def oracle():
        r = rgba.clone().requires_grad_(True)
        ref = LO.texture_loss_masks(r[:, :C], gt, mgt, r[:, 3], avg=False)
        (ref * w).sum().backward()
        return [ref, r.grad]
    return fn, _leaves(rgba), oracle, [(1e-4, 1e-6), (1e-4, 1e-9)]


def loss_head_case(B, H):
    g = _gen(6)
    rgba = torch.rand(B, 4, H, H, generator=g)
    gt = torch.rand(B, 3, H, H, generator=g)
    mgt = (torch.rand(B, H, H, generator=g) > 0.4).float()
    gtd, md = gt.to(DEV), mgt.to(DEV)

    def fn(x):
        x.grad = None
        loss, per_image = ops.mask_texture_loss(x, gtd, md, 2.5, 3.0)
        (loss * 1.7).backward()
        return [loss, per_image, x.grad]

    def oracle():
        r = rgba.clone().requires_grad_(True)
        iou = LO.neg_iou_loss(r[:, 3], mgt, avg=False)
        l1 = LO.texture_loss_masks(r[:, :3], gt, mgt, r[:, 3], avg=False)
        ref = 2.5 * iou.mean() + 3.0 * l1.mean()
        (ref * 1.7).backward()
        return [ref, torch.stack((iou, l1), 1).detach(), r.grad]
    return fn, _leaves(rgba), oracle, [(1e-5, 1e-7), (1e-4, 1e-6), (1e-4, 1e-9)]


def texcycle_case(B, F, T, P, from_plane):
    g = _gen(4)
    flow = torch.rand(B, F, T, T, 2, generator=g) * 2 - 1
    prob = torch.rand(B, F, 2, generator=g) * 2 - 1
    ids = torch.randint(-1, F // 2, (B, P), generator=g).float()   # -1 = background, upper half never visible
    ids[-1] = 5.0                                                   # one sample without background
    vis = torch.zeros(B, F, dtype=torch.uint8)
    vis.scatter_(1, ids.long() % F, 1)                              # what the plane marks (-1 -> face F-1)
    probd, idsd, visd = prob.to(DEV), ids.to(DEV), vis.to(DEV)

    def fn(x):
        x.grad = None
        if from_plane:
            loss, _ = loss_utils.TexCycle()(x, probd, idsd)
        else:
            loss, _ = loss_utils.TexCycle()(x, probd, None, visible=visd)
        loss.backward()
        return [loss, x.grad]

    def oracle():
        fr = flow.clone().requires_grad_(True)
        ref, _ = LO.tex_cycle(fr, prob, ids)
        ref.backward()
        return [ref, fr.grad]
    return fn, _leaves(flow), oracle, [(1e-4, 1e-6), (1e-4, 1e-9)]


def _mesh_case(kind, subdiv, B, open_mesh=False):
    rng = np.random.default_rng(subdiv)
    v, f = synth.icosphere(subdiv)
    if open_mesh:
        f = f[v[f].mean(1)[:, 2] > 0]
    verts = torch.from_numpy(synth.bird_like(v, rng, B))
    faces = torch.from_numpy(f.astype(np.int64))
    w = torch.from_numpy(rng.uniform(0.5, 1.5, size=(B,)).astype(np.float32))
    mod = (sr.LaplacianLoss(torch.from_numpy(v), faces) if kind == "laplacian" else sr.FlattenLoss(faces)).to(DEV)
    wd = w.to(DEV)
    ref_fn = MO.laplacian_loss if kind == "laplacian" else MO.flatten_loss

    def fn(x):
        x.grad = None
        loss = mod(x)
        (loss * wd).sum().backward()
        return [loss, x.grad]

    def oracle():
        xr = verts.clone().requires_grad_(True)
        ref = ref_fn(xr, f)
        (ref * w).sum().backward()
        return [ref, xr.grad]
    # oracle/mesh_oracle.flatten_edges pairs the faces of a closed mesh only: an open mesh is checked against the default path
    return fn, _leaves(verts), None if open_mesh else oracle, [(2e-5, 1e-6), (1e-4, "scaled")]


def chamfer_case(B, N, M, D, one_nearest):
    g = _gen(3)
    a = torch.rand(B, N, D, generator=g) - 0.5
    if one_nearest:   # every point of b nearest to a[:, 0]: the default backward's scatter piles all M terms on one point
        a[:, 1:] += torch.sign(a[:, 1:]) * 0.2   # every other point of a at least 0.2 from the origin in each coordinate
        a[:, 0] = 0.0
        b = 1e-3 * (torch.rand(B, M, D, generator=g) - 0.5)
    else:
        b = torch.rand(B, M, D, generator=g) - 0.5
    w1, w2 = torch.rand(B, N, generator=g), torch.rand(B, M, generator=g)
    w1d, w2d = w1.to(DEV), w2.to(DEV)

    def fn(x, y):
        x.grad = y.grad = None
        o = chamfer_python.distChamfer(x, y)
        ((o[0] * w1d).sum() + (o[1] * w2d).sum()).backward()
        return [o[0], o[1], o[2], o[3], x.grad, y.grad]

    def oracle():
        ar, br = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
        r = LO.dist_chamfer(ar, br)
        ((r[0] * w1).sum() + (r[1] * w2).sum()).backward()
        return [r[0], r[1], None, None, ar.grad, br.grad]   # argmins: compared with the default path only
    fn.one_nearest = one_nearest
    return fn, _leaves(a, b), oracle, [(1e-4, 1e-6), (1e-4, 1e-6), None, None, (1e-4, 1e-5), (1e-4, 1e-4)]


def corr_case(shared):
    rng = np.random.default_rng(17)
    B, IS = 6, 64
    v, f = synth.icosphere(3)
    V = v.shape[0]
    parts = [torch.from_numpy(p) for p in synth.part_vertex_sets(rng, V, sizes=(20, 40, 20, 40))]
    parts[1] = torch.cat((parts[1], parts[0][:5]))   # vertices listed in two parts
    pts = [torch.from_numpy(p).to(DEV) for p in synth.part_points(rng, B)]
    m = loss_utils.CorrLossChamfer(None, IS, part_vertices=parts)
    m.weights = [1, 1, 0.5, 0.25]
    base = torch.from_numpy(synth.bird_like(v, rng, B))
    cams0 = torch.from_numpy(synth.cameras(rng, B))
    lw = torch.linspace(0.5, 1.5, B, device=DEV)

    def fn(leaf, cams):
        leaf.grad = cams.grad = None
        verts = leaf[None].expand(B, -1, -1) if shared else leaf   # expanded: vertices_batch_stride = 0
        loss = m(pts[0], pts[1], pts[2], pts[3], verts, cams, avg=False)
        (loss * lw).sum().backward()
        return [loss, leaf.grad, cams.grad]
    return fn, _leaves(base[0] if shared else base, cams0), None, [(1e-5, 1e-7), (1e-4, "scaled"), (1e-4, "scaled5")]


CASES = {
    "iou_c2": lambda: iou_case(16, 256, 256, False),
    "iou_c3_alpha_plane": lambda: iou_case(256, 512, 512, True),
    "iou_below_one_tile": lambda: iou_case(3, 37, 41, True),
    "iou_b1_2048": lambda: iou_case(1, 2048, 2048, False),
    "masked_l1_c2": lambda: masked_l1_case(16, 256, 256, 3),
    "masked_l1_below_one_tile_c1": lambda: masked_l1_case(3, 37, 41, 1),
    "masked_l1_b1_2048": lambda: masked_l1_case(1, 2048, 2048, 3),
    "loss_head_c2": lambda: loss_head_case(16, 256),
    "loss_head_below_one_tile": lambda: loss_head_case(2, 37),
    "loss_head_b1_2048": lambda: loss_head_case(1, 2048),
    "texcycle_plane": lambda: texcycle_case(16, 1280, 6, 64 * 64, True),
    "texcycle_visible": lambda: texcycle_case(16, 1280, 6, 64 * 64, False),
    "texcycle_small_plane": lambda: texcycle_case(3, 64, 6, 32 * 32, True),
    "laplacian_ico3": lambda: _mesh_case("laplacian", 3, 16),
    "laplacian_ico1": lambda: _mesh_case("laplacian", 1, 1),
    "flatten_ico3": lambda: _mesh_case("flatten", 3, 16),
    "flatten_open": lambda: _mesh_case("flatten", 2, 3, open_mesh=True),
    "chamfer_d2": lambda: chamfer_case(3, 80, 30, 2, False),
    "chamfer_d3": lambda: chamfer_case(2, 33, 7, 3, False),
    "chamfer_d2_one_nearest": lambda: chamfer_case(2, 50, 2000, 2, True),
    "chamfer_d3_one_nearest": lambda: chamfer_case(2, 40, 700, 3, True),
    "corr_shared_vertices": lambda: corr_case(True),
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
        assert torch.equal(x, y), "%s: output %d differs bitwise" % (what, k)


def _assert_close(got, ref, tols, what):
    msgs, ok = [], True
    for k, (x, r, tol) in enumerate(zip(got, ref, tols)):
        if r is None or tol is None:
            continue
        x, r = x.numpy(), r.detach().cpu().numpy()
        rtol, atol = tol
        if atol == "scaled":
            atol = 2e-5 * float(np.abs(r).max())
        elif atol == "scaled5":
            atol = 1e-5 * float(np.abs(r).max())
        o, m = rel_report("%s[%d]" % (what, k), x, r, rtol, atol)
        ok &= o
        msgs.append(m)
    assert ok, "\n".join(msgs)


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


@pytest.mark.parametrize("name", list(CASES))
def test_entry_point(det, name):
    fn, leaves, oracle, tols = CASES[name]()
    ref = _run(fn, leaves)
    for _ in range(2):
        _assert_equal(ref, _run(fn, leaves), "run")
    results = [None] * 4

    def work(i):
        torch.use_deterministic_algorithms(True)
        st = torch.cuda.Stream(device=DEV)
        with torch.cuda.stream(st):
            mine = [l.detach().clone().requires_grad_(True) for l in leaves]
        st.synchronize()
        results[i] = _run(fn, mine, st)

    ts = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for r in results:
        _assert_equal(ref, r, "thread")
    _graph_replays(fn, leaves, ref)
    torch.use_deterministic_algorithms(False)
    default = _run(fn, leaves)
    torch.use_deterministic_algorithms(True)
    _assert_close(ref, default, tols, name + " vs default")
    if name.startswith("chamfer"):   # forward planes, argmins included, are the default kernels' bits
        for k in range(4):
            assert torch.equal(ref[k], default[k])
        if getattr(fn, "one_nearest", False):
            assert bool((ref[3] == 0).all())
    if oracle is not None:
        _assert_close(ref, _host(oracle()), tols, name + " vs oracle")
    for k, o in enumerate(ref):
        assert bool(torch.isfinite(o.float()).all()), "%s output %d not finite" % (name, k)


# -------------------------------------------------------------------------------------------------
# non-finite inputs
# -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["default", "deterministic"])
def test_nan_input_gives_nan_loss(mode):
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(mode == "deterministic")
    try:
        g = _gen(9)
        B, H = 3, 64
        rgba = torch.rand(B, 4, H, H, generator=g).to(DEV)
        rgba[1, 3, 10, 20] = float("nan")
        gt = torch.rand(B, 3, H, H, generator=g).to(DEV)
        m = (torch.rand(B, H, H, generator=g) > 0.5).float().to(DEV)
        iou = loss_utils.neg_iou_loss(rgba[:, 3], m, avg=False)
        l1 = loss_utils.texture_loss_masks(rgba[:, :3], gt, m, rgba[:, 3], avg=False)
        head, per_image = ops.mask_texture_loss(rgba, gt, m)
        for per in (iou, l1, per_image[:, 0], per_image[:, 1]):
            assert torch.isnan(per[1]) and bool(torch.isfinite(per[[0, 2]]).all())
        assert torch.isnan(head)
        flow = torch.rand(2, 16, 4, 2, generator=g).to(DEV)
        flow[1, 3, 2, 0] = float("nan")
        vis = torch.ones(2, 16, dtype=torch.uint8, device=DEV)
        assert torch.isnan(ops.tex_cycle(flow, torch.zeros(2, 16, 2, device=DEV), None, vis))
        v, f = synth.icosphere(1)
        x = torch.from_numpy(np.stack([v, v]).astype(np.float32)).to(DEV)
        x[1, 4, 0] = float("nan")
        faces = torch.from_numpy(f.astype(np.int64))
        for mod in (sr.LaplacianLoss(torch.from_numpy(v), faces), sr.FlattenLoss(faces)):
            loss = mod.to(DEV)(x)
            assert torch.isnan(loss[1]) and torch.isfinite(loss[0])
    finally:
        torch.use_deterministic_algorithms(old)


# -------------------------------------------------------------------------------------------------
# the train_s2-shaped loss step (tools/train_step_bench.py's step; test_train_step_gpu's scene)
# -------------------------------------------------------------------------------------------------
def make_step(B, H, IS, subdiv, T, seed):
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(subdiv)
    V, F = v.shape[0], f.shape[0]
    fs = torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1).to(DEV)
    imgs = torch.from_numpy(synth.smooth_images(rng, B, IS)).to(DEV)
    masks = torch.from_numpy(synth.ellipse_masks(rng, B, IS)).to(DEV)
    dts = torch.from_numpy(np.stack([synth.dt_barrier(m) for m in masks.cpu().numpy()]))[:, None].to(DEV)
    part_segs = torch.from_numpy(rng.uniform(0, 1, size=(B, 5, IS, IS)).astype(np.float32)).to(DEV)
    part = rng.integers(0, 5, size=(F, T * T))
    one_hot = torch.zeros(1, F, T * T, 5)
    one_hot.scatter_(3, torch.from_numpy(part)[None, :, :, None], 1.0)
    part_vertices = [torch.from_numpy(p) for p in synth.part_vertex_sets(rng, V, sizes=(20, 40, 20, 40))]
    head, belly, neck, back = [torch.from_numpy(p).to(DEV) for p in synth.part_points(rng, B)]
    rep = lambda t: t.unsqueeze(1).repeat(1, H, 1, 1).view(-1, t.size(1), t.size(2))
    mask_fn = loss_utils.MultiMaskLoss(IS, "softmax", H).to(DEV)
    tex_fn = loss_utils.MultiTextureLoss(B, H, IS, "softmax", "l1", "smr").to(DEV)
    part_fn = loss_utils.part_matching_loss(None, None, 0, im_size=IS, batch_size=B, tex_size=T, stex_one_hot=one_hot).to(DEV)
    corr_fn = loss_utils.CorrLossChamfer(None, IS, part_vertices=part_vertices)
    fcpu = torch.from_numpy(f.astype(np.int64))
    lap_fn = sr.LaplacianLoss(torch.from_numpy(v), fcpu).to(DEV)
    flat_fn = sr.FlattenLoss(fcpu).to(DEV)
    leaves = [torch.from_numpy(v.astype(np.float32)),
              0.05 * torch.from_numpy(synth.bird_like(v, rng, B) - v[None]),
              torch.from_numpy(np.stack([synth.cameras(rng, H) for _ in range(B)])),
              torch.from_numpy(rng.normal(size=(B, H)).astype(np.float32)),
              torch.from_numpy(synth.texture_flow(rng, B, F, T))]
    leaves = _leaves(*leaves)   # mean shape, deformation, cameras, camera logits, texture flow

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
        total = mask_loss.mean() + 0.1 * tri + 0.005 * flat + 3.0 * tl.mean() + 3.0 * tdt.mean() + tcyc.mean() \
            + 0.1 * pl.mean() + corr
        total.backward()
        return [total] + [t.grad for t in (mean_shape, delta, cams, logits, flow)]
    return step, leaves


STEPS = {"train_step_scene_shape": (2, 8, 32, 2, 3, 21), "bench_default": (16, 8, 256, 3, 6, 0)}


@pytest.mark.parametrize("name", list(STEPS))
def test_whole_step_bitwise_reproducible(det, name):
    step, leaves = make_step(*STEPS[name])
    ref = _run(step, leaves)
    for _ in range(2):
        _assert_equal(ref, _run(step, leaves), "step run")
    results = [None] * 4

    def work(i):
        torch.use_deterministic_algorithms(True)
        st = torch.cuda.Stream(device=DEV)
        with torch.cuda.stream(st):
            mine = [l.detach().clone().requires_grad_(True) for l in leaves]
        st.synchronize()
        results[i] = _run(step, mine, st)

    ts = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for r in results:
        _assert_equal(ref, r, "step thread")
    torch.use_deterministic_algorithms(False)
    default = _run(step, leaves)
    torch.use_deterministic_algorithms(True)
    assert all(bool(torch.isfinite(t).all()) for t in ref)
    for k, (x, r) in enumerate(zip(ref, default)):   # test_train_step_gpu's part-matching gate (the widest it uses)
        ok, msg = rel_report("step output %d" % k, x.numpy(), r.numpy(), 2e-4, 2e-5 * float(r.abs().max()) + 1e-9)
        print(msg)
        assert ok, msg


# -------------------------------------------------------------------------------------------------
# launch counts per call: unchanged with the flag off, fixed with it on
# -------------------------------------------------------------------------------------------------
def _launches(fn):
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.umr_launch_count()
    out = fn()
    return lib.umr_launch_count() - n0, out


@pytest.mark.parametrize("mode", ["default", "deterministic"])
def test_launch_counts(mode):
    dflt = mode == "default"
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(not dflt)
    try:
        g = _gen(10)
        B, H = 2, 48
        rgba = torch.rand(B, 4, H, H, generator=g).to(DEV).requires_grad_(True)
        gt = torch.rand(B, 3, H, H, generator=g).to(DEV)
        m = (torch.rand(B, H, H, generator=g) > 0.5).float().to(DEV)
        # (forward, backward) launches of each op: today's counts with the flag off
        want = {"iou": (2, 1) if dflt else (2, 1), "masked_l1": (1, 1) if dflt else (2, 1),
                "loss_head": (2, 1) if dflt else (3, 1), "texcycle_plane": (2, 1) if dflt else (3, 1),
                "texcycle_visible": (1, 1) if dflt else (2, 1), "laplacian": (1, 1) if dflt else (2, 1),
                "flatten": (1, 1) if dflt else (2, 2), "chamfer": (2, 2), "corr": (1, 1) if dflt else (1, 2)}
        flow = torch.rand(B, 16, 4, 2, generator=g).to(DEV).requires_grad_(True)
        prob = torch.rand(B, 16, 2, generator=g).to(DEV)
        ids = torch.randint(-1, 16, (B, 64), generator=g).float().to(DEV)
        vis = torch.ones(B, 16, dtype=torch.uint8, device=DEV)
        v, f = synth.icosphere(2)
        x = torch.from_numpy(synth.bird_like(v, np.random.default_rng(0), B)).to(DEV).requires_grad_(True)
        faces = torch.from_numpy(f.astype(np.int64))
        lap, flat = sr.LaplacianLoss(torch.from_numpy(v), faces).to(DEV), sr.FlattenLoss(faces).to(DEV)
        a = torch.rand(B, 30, 2, generator=g).to(DEV).requires_grad_(True)
        b = torch.rand(B, 20, 2, generator=g).to(DEV).requires_grad_(True)
        rng = np.random.default_rng(1)
        parts = [torch.from_numpy(p) for p in synth.part_vertex_sets(rng, v.shape[0], sizes=(5, 6, 7, 8))]
        corr = loss_utils.CorrLossChamfer(None, 32, part_vertices=parts)
        pts = [torch.from_numpy(p).to(DEV) for p in synth.part_points(rng, B)]
        cams = torch.from_numpy(synth.cameras(rng, B)).to(DEV).requires_grad_(True)
        corr(pts[0], pts[1], pts[2], pts[3], x, cams, avg=False)   # fills the module's index cache
        ops_ = {
            "iou": lambda: loss_utils.neg_iou_loss(rgba[:, 3], m, avg=False).sum(),
            "masked_l1": lambda: loss_utils.texture_loss_masks(rgba[:, :3], gt, m, rgba[:, 3], avg=False).sum(),
            "loss_head": lambda: ops.mask_texture_loss(rgba, gt, m)[0],
            "texcycle_plane": lambda: ops.tex_cycle(flow, prob, ids),
            "texcycle_visible": lambda: ops.tex_cycle(flow, prob, None, vis),
            "laplacian": lambda: lap(x).sum(),
            "flatten": lambda: flat(x).sum(),
            "chamfer": lambda: sum(o.sum() for o in chamfer_python.distChamfer(a, b)[:2]),
            "corr": lambda: corr(pts[0], pts[1], pts[2], pts[3], x, cams, avg=False).sum(),
        }
        for name, op in ops_.items():
            nf, loss = _launches(op)
            nb, _ = _launches(loss.backward)
            assert (nf, nb) == want[name], (name, mode, nf, nb)
    finally:
        torch.use_deterministic_algorithms(old)
