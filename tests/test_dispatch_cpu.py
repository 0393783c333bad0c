"""Which kernels the autograd bindings of ops.py and raster.py call, without a GPU.

A fake library stands in for libumr_b200.so: it converts every argument with the ctypes argument types of
`_lib.EXPORTS` (so a wrong count or type fails as it would on the real library), records the call and returns 0, or a
byte count for the `*_bytes*` queries.  The tensors are CPU tensors that claim to be CUDA ones.  The library writes
nothing, so these tests check dispatch, never values: for every public entry in float32, deterministic float32,
float64, mixed float32/float64 and half inputs, the sequence of symbols called (forward then backward), which pointer
arguments are NULL, the output dtypes and that each gradient has its input's dtype."""
import contextlib
import ctypes
import re
import types

import pytest
import torch

from umr_b200 import _lib, ops, raster
from umr_b200.soft_renderer.losses import FlattenLoss

MODES = ("f32", "det", "f64", "mixed", "half")


class FakeLib(object):
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name not in _lib.EXPORTS:
            raise AttributeError(name)
        argtypes = _lib.EXPORTS[name][1]

        def call(*args):
            assert len(args) == len(argtypes), "%s takes %d arguments, got %d" % (name, len(argtypes), len(args))
            for t, a in zip(argtypes, args):
                t.from_param(a)   # TypeError on a mismatch, as ctypes raises it
            self.calls.append((name, args))
            return 64 if "_bytes" in name else 0
        return call


def _mask(args):
    """'1' / '0' per pointer argument (non-NULL / NULL); for the raster parameter block, whether it names a pair buffer."""
    out = ""
    for a in args:
        if isinstance(a, ctypes.c_void_p):
            out += "1" if a.value else "0"
        elif isinstance(getattr(a, "_obj", None), _lib.UmrRasterParams):
            out += "P" if a._obj.pair_buffer else "p"
    return out


def trace(fake):
    return ["%s:%s" % (name, _mask(args)) for name, args in fake.calls]


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(torch.cuda, "device", lambda device: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: types.SimpleNamespace(cuda_stream=0))
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(raster, "PAIR_ADAPTIVE", False)
    monkeypatch.setattr(raster, "_PAIR_MAX_GB", "1")
    return lib


def _dtypes(mode):
    """dtype of the k-th floating-point input: mixed makes the first float32 and the others float64."""
    one = {"f32": torch.float32, "det": torch.float32, "f64": torch.float64, "half": torch.float16}.get(mode)
    return lambda k: one if one is not None else (torch.float32 if k == 0 else torch.float64)


def _rand(shape, dtype, grad=False, seed=[0]):
    seed[0] += 1
    g = torch.Generator().manual_seed(seed[0])
    return torch.rand(shape, generator=g).to(dtype).requires_grad_(grad)


_TET = torch.tensor([[0, 1, 2], [0, 2, 3], [0, 3, 1], [1, 3, 2]])


# Each entry: dt -> (outputs, scalar to differentiate, leaf inputs with a gradient)
def _sample(dt):
    img, flow = _rand((2, 3, 4, 5), dt(0), True), _rand((2, 6, 2), dt(1), True)
    out = ops.bilinear_sample(img, flow)
    return [out], out.sum(), [img, flow]


def _iou(dt):
    p, t = _rand((2, 4, 4), dt(0), True), _rand((2, 4, 4), dt(1))
    out = ops.neg_iou_per_image(p, t)
    return [out], out.sum(), [p]


def _masked_l1(dt):
    p, g = _rand((2, 3, 4, 4), dt(0), True), _rand((2, 3, 4, 4), dt(1))
    mg, mp = _rand((2, 4, 4), dt(1)), _rand((2, 4, 4), dt(0), True)
    out = ops.masked_l1_per_image(p, g, mg, mp)
    return [out], out.sum(), [p, mp]


def _loss_head(dt):
    x, g, m = _rand((2, 4, 4, 4), dt(0), True), _rand((2, 3, 4, 4), dt(1)), _rand((2, 4, 4), dt(1))
    loss, per_image = ops.mask_texture_loss(x, g, m, 0.5, 2.0)
    return [loss, per_image], loss, [x]


def _chamfer(dt):
    a, b = _rand((2, 5, 3), dt(0), True), _rand((2, 6, 3), dt(1), True)
    d_ab, d_ba, i_ab, i_ba = ops.dist_chamfer(a, b)
    return [d_ab, d_ba], d_ab.sum() + d_ba.sum(), [a, b]


def _texcycle(dt, visible):
    flow, prob = _rand((2, 3, 4, 2), dt(0), True), _rand((2, 3, 2), dt(1))
    if visible:
        out = ops.tex_cycle(flow, prob, None, torch.tensor([[1, 0, 1], [1, 1, 0]], dtype=torch.uint8))
    else:
        out = ops.tex_cycle(flow, prob, torch.tensor([[-1, 0, 2, 2], [1, -1, 0, 0]]).to(dt(1)))
    return [out], out, [flow]


def _laplacian(dt):
    x = _rand((2, 4, 3), dt(0), True)
    cdt = torch.float32 if dt(1) == torch.float16 else dt(1)   # the module's coefficient buffers: float32, or widened
    rowptr = torch.tensor([0, 3, 6, 9, 12], dtype=torch.int32)
    col = torch.tensor([1, 2, 3, 0, 2, 3, 0, 1, 3, 0, 1, 2], dtype=torch.int32)
    coef = torch.full((12,), -1.0 / 3).to(cdt)
    out = ops.LaplacianFunction.apply(x, rowptr, col, coef, coef.clone())
    return [out], out.sum(), [x]


def _flatten(dt, prebuilt):
    v = _rand((2, 4, 3), dt(0), True)
    m = FlattenLoss(_TET)
    table = (m.vert_rowptr, m.vert_incidence) if prebuilt else ()
    out = ops.FlattenFunction.apply(v, m.edge_table, 1e-6, *table)
    return [out], out.sum(), [v]


def _corr(dt, shared):
    B, V = 2, 6
    verts, cams = _rand((1 if shared else B, V, 3), dt(0), True), _rand((B, 7), dt(1), True)
    sel = torch.tensor([0, 2, 3, 5, 1, 4], dtype=torch.int32)
    targets = [_rand((B, m, 2), dt(1)) for m in (2, 3, 1, 2)]
    loss, vert2d = ops.corr_chamfer(verts, cams, sel, targets, (2, 3, 5, 6), (1.0, 0.5, 0.25, 2.0))
    return [loss, vert2d], loss.sum() + vert2d.sum(), [verts, cams]


def _raster(dt, channels=3, geom=True, tex=True, **kw):
    B, F = 2, 3
    fv = _rand((B, F, 3, 3), dt(0), geom)
    tx = _rand((B, F, 4, channels), dt(1), tex)
    images, p2f, aggrs = raster.soft_rasterize(fv, tx, 8, **kw)
    return [images, p2f, aggrs], images.sum(), [t for t in (fv, tx) if t.requires_grad]


ENTRIES = {
    "sample": _sample,
    "iou": _iou,
    "masked_l1": _masked_l1,
    "loss_head": _loss_head,
    "chamfer": _chamfer,
    "texcycle_plane": lambda dt: _texcycle(dt, False),
    "texcycle_visible": lambda dt: _texcycle(dt, True),
    "laplacian": _laplacian,
    "flatten_built_here": lambda dt: _flatten(dt, False),
    "flatten_prebuilt": lambda dt: _flatten(dt, True),
    "corr_shared": lambda dt: _corr(dt, True),
    "corr_per_render": lambda dt: _corr(dt, False),
    "raster_softmax": lambda dt: _raster(dt),
    "raster_generic": lambda dt: _raster(dt, dist_func="barycentric", aggr_func_alpha="sum"),
    "raster_hard": lambda dt: _raster(dt, aggr_func_rgb="hard"),
    "raster_part_map": lambda dt: _raster(dt, channels=4, tex=False, background_color=(0, 0, 0, 1)),
    "raster_vertex_part_map": lambda dt: _raster(dt, channels=4, tex=False, texture_type="vertex"),
    "raster_aa": lambda dt: _raster(dt, anti_aliasing=True),
    "raster_texture_only": lambda dt: _raster(dt, geom=False),
    "raster_generic_texture_only": lambda dt: _raster(dt, geom=False, dist_func="barycentric"),
}

# name -> {space-separated modes: the calls of a forward + backward, each as `symbol:mask` (mask: `_mask`), or the
# ValueError the forward raises}
EXPECTED = {
    'chamfer': {
        'f32 half': ['umr_chamfer_forward:1111110', 'umr_chamfer_backward:111111110'],
        'det': ['umr_chamfer_forward:1111110', 'umr_chamfer_backward_deterministic:111111110'],
        'f64 mixed': ['umr_chamfer_forward_f64:1111110', 'umr_chamfer_backward_f64:111111110'],
    },
    'corr_per_render': {
        'f32 half': ['umr_corr_chamfer_forward:1111110', 'umr_corr_chamfer_backward:1111111110'],
        'det': [
            'umr_corr_chamfer_forward:1111110', 'umr_corr_chamfer_workspace_bytes_deterministic:',
            'umr_corr_chamfer_backward_deterministic:1111111111110'
        ],
        'f64 mixed': [
            'umr_corr_chamfer_forward_f64:1111110', 'umr_corr_chamfer_workspace_bytes_f64:',
            'umr_corr_chamfer_backward_f64:1111111111110'
        ],
    },
    'corr_shared': {
        'f32 half': ['umr_corr_chamfer_forward:1111110', 'umr_corr_chamfer_backward:1111111110'],
        'det': [
            'umr_corr_chamfer_forward:1111110', 'umr_corr_chamfer_workspace_bytes_deterministic:',
            'umr_corr_chamfer_backward_deterministic:1111111111110'
        ],
        'f64 mixed': [
            'umr_corr_chamfer_forward_f64:1111110', 'umr_corr_chamfer_workspace_bytes_f64:',
            'umr_corr_chamfer_backward_f64:1111111111110'
        ],
    },
    'flatten_built_here': {
        'f32 mixed half': ['umr_flatten_forward:1110', 'umr_flatten_backward:11110'],
        'det': [
            'umr_flatten_forward_workspace_bytes_deterministic:', 'umr_flatten_forward_deterministic:11110',
            'umr_flatten_backward_workspace_bytes_deterministic:', 'umr_flatten_backward_deterministic:11111110'
        ],
        'f64': [
            'umr_flatten_forward_workspace_bytes_f64:', 'umr_flatten_forward_f64:11110',
            'umr_flatten_backward_workspace_bytes_f64:', 'umr_flatten_backward_f64:11111110'
        ],
    },
    'flatten_prebuilt': {
        'f32 mixed half': ['umr_flatten_forward:1110', 'umr_flatten_backward:11110'],
        'det': [
            'umr_flatten_forward_workspace_bytes_deterministic:', 'umr_flatten_forward_deterministic:11110',
            'umr_flatten_backward_workspace_bytes_deterministic:', 'umr_flatten_backward_deterministic:11111110'
        ],
        'f64': [
            'umr_flatten_forward_workspace_bytes_f64:', 'umr_flatten_forward_f64:11110',
            'umr_flatten_backward_workspace_bytes_f64:', 'umr_flatten_backward_f64:11111110'
        ],
    },
    'iou': {
        'f32 half': ['umr_iou_forward:111110', 'umr_iou_backward:111110'],
        'det': [
            'umr_iou_workspace_bytes_deterministic:', 'umr_iou_forward_deterministic:1111110',
            'umr_iou_backward:111110'
        ],
        'f64 mixed': ['umr_iou_workspace_bytes_f64:', 'umr_iou_forward_f64:1111110', 'umr_iou_backward_f64:111110'],
    },
    'laplacian': {
        'f32 half': ['umr_laplacian_forward:1111110', 'umr_laplacian_backward:1111110'],
        'det': [
            'umr_laplacian_workspace_bytes_deterministic:', 'umr_laplacian_forward_deterministic:11111110',
            'umr_laplacian_backward:1111110'
        ],
        'f64 mixed': [
            'umr_laplacian_workspace_bytes_f64:', 'umr_laplacian_forward_f64:11111110',
            'umr_laplacian_backward_f64:1111110'
        ],
    },
    'loss_head': {
        'f32 half': ['umr_loss_head_forward:1111110', 'umr_loss_head_backward:1111110'],
        'det': [
            'umr_loss_head_workspace_bytes_deterministic:', 'umr_loss_head_forward_deterministic:11111110',
            'umr_loss_head_backward:1111110'
        ],
        'f64 mixed': [
            'umr_loss_head_workspace_bytes_f64:', 'umr_loss_head_forward_f64:11111110',
            'umr_loss_head_backward_f64:1111110'
        ],
    },
    'masked_l1': {
        'f32 half': ['umr_masked_l1_forward:111110', 'umr_masked_l1_backward:11111110'],
        'det': [
            'umr_masked_l1_workspace_bytes_deterministic:', 'umr_masked_l1_forward_deterministic:1111110',
            'umr_masked_l1_backward:11111110'
        ],
        'f64 mixed': [
            'umr_masked_l1_workspace_bytes_f64:', 'umr_masked_l1_forward_f64:1111110',
            'umr_masked_l1_backward_f64:11111110'
        ],
    },
    'raster_aa': {
        'f32 mixed half': [
            'umr_raster_workspace_bytes:', 'umr_raster_pair_buffer_bytes:', 'umr_raster_forward:111111P10',
            'umr_raster_workspace_bytes:', 'umr_raster_backward:1111111P10'
        ],
        'det': [
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_forward_deterministic:111111p10',
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_backward_deterministic:1111111p10'
        ],
        'f64': [
            'umr_raster_workspace_bytes_f64:', 'umr_raster_forward_f64:111111p10', 'umr_raster_workspace_bytes_f64:',
            'umr_raster_backward_f64:1111111p10'
        ],
    },
    'raster_generic': {
        'f32 mixed half': [
            'umr_raster_workspace_bytes:', 'umr_raster_forward:111011p10', 'umr_raster_workspace_bytes:',
            'umr_raster_backward:1111111p10'
        ],
        'det': [
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_forward_deterministic:111011p10',
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_backward_deterministic:1111111p10'
        ],
        'f64': [
            'umr_raster_workspace_bytes_f64:', 'umr_raster_forward_f64:111011p10', 'umr_raster_workspace_bytes_f64:',
            'umr_raster_backward_f64:1111111p10'
        ],
    },
    'raster_generic_texture_only': {
        'f32 mixed half': [
            'umr_raster_workspace_bytes:', 'umr_raster_forward:111011p10', 'umr_raster_workspace_bytes:',
            'umr_raster_backward:1111111p10'
        ],
        'det': [
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_forward_deterministic:111011p10',
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_backward_deterministic:1111101p10'
        ],
        'f64': [
            'umr_raster_workspace_bytes_f64:', 'umr_raster_forward_f64:111011p10', 'umr_raster_workspace_bytes_f64:',
            'umr_raster_backward_f64:1111101p10'
        ],
    },
    'raster_hard': {
        'f32 mixed half': [
            'umr_raster_workspace_bytes:', 'umr_raster_pair_buffer_bytes:', 'umr_raster_forward:111011P10',
            'umr_raster_workspace_bytes:', 'umr_raster_backward:1111111P10'
        ],
        'det': [
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_forward_deterministic:111011p10',
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_backward_deterministic:1111111p10'
        ],
        'f64': [
            'umr_raster_workspace_bytes_f64:', 'umr_raster_forward_f64:111011p10', 'umr_raster_workspace_bytes_f64:',
            'umr_raster_backward_f64:1111111p10'
        ],
    },
    'raster_part_map': {
        'f32 mixed half': [
            'umr_raster_workspace_bytes:', 'umr_raster_pair_buffer_bytes:', 'umr_raster_forward:111011P10',
            'umr_raster_workspace_bytes:', 'umr_raster_backward:1111110P10'
        ],
        'det': [
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_forward_deterministic:111011p10',
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_backward_deterministic:1111110p10'
        ],
        'f64': 'float64 rasterisation takes 3 colour channels, got 4 (part-map textures are float32 only)',
    },
    'raster_vertex_part_map': {
        'f32 mixed half det': 'vertex textures take 3 colour channels, got 4 (4-channel part maps are surface textures only)',
        'f64': 'float64 rasterisation takes 3 colour channels, got 4 (part-map textures are float32 only)',
    },
    'raster_softmax': {
        'f32 mixed half': [
            'umr_raster_workspace_bytes:', 'umr_raster_pair_buffer_bytes:', 'umr_raster_forward:111011P10',
            'umr_raster_workspace_bytes:', 'umr_raster_backward:1111111P10'
        ],
        'det': [
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_forward_deterministic:111011p10',
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_backward_deterministic:1111111p10'
        ],
        'f64': [
            'umr_raster_workspace_bytes_f64:', 'umr_raster_forward_f64:111011p10', 'umr_raster_workspace_bytes_f64:',
            'umr_raster_backward_f64:1111111p10'
        ],
    },
    'raster_texture_only': {
        'f32 mixed half': [
            'umr_raster_workspace_bytes:', 'umr_raster_pair_buffer_bytes:', 'umr_raster_forward:111011P10',
            'umr_raster_workspace_bytes:', 'umr_raster_backward:1111101P10'
        ],
        'det': [
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_forward_deterministic:111011p10',
            'umr_raster_workspace_bytes_deterministic:', 'umr_raster_backward_deterministic:1111101p10'
        ],
        'f64': [
            'umr_raster_workspace_bytes_f64:', 'umr_raster_forward_f64:111011p10', 'umr_raster_workspace_bytes_f64:',
            'umr_raster_backward_f64:1111101p10'
        ],
    },
    'sample': {
        'f32 half': ['umr_bilinear_sample_forward:1110', 'umr_bilinear_sample_backward:111110'],
        'det': [
            'umr_bilinear_sample_forward:1110', 'umr_bilinear_sample_cells:110',
            'umr_bilinear_sample_backward_deterministic:11111110'
        ],
        'f64 mixed': [
            'umr_bilinear_sample_forward_f64:1110', 'umr_bilinear_sample_cells_f64:110',
            'umr_bilinear_sample_backward_f64:11111110'
        ],
    },
    'texcycle_plane': {
        'f32 half': ['umr_texcycle_forward:111110', 'umr_texcycle_backward:111110'],
        'det': [
            'umr_texcycle_workspace_bytes_deterministic:', 'umr_texcycle_forward_deterministic:1111110',
            'umr_texcycle_backward:111110'
        ],
        'f64 mixed': [
            'umr_texcycle_workspace_bytes_f64:', 'umr_texcycle_forward_f64:1111110', 'umr_texcycle_backward_f64:111110'
        ],
    },
    'texcycle_visible': {
        'f32 half': ['umr_texcycle_forward:110110', 'umr_texcycle_backward:111110'],
        'det': [
            'umr_texcycle_workspace_bytes_deterministic:', 'umr_texcycle_forward_deterministic:1101110',
            'umr_texcycle_backward:111110'
        ],
        'f64 mixed': [
            'umr_texcycle_workspace_bytes_f64:', 'umr_texcycle_forward_f64:1101110', 'umr_texcycle_backward_f64:111110'
        ],
    },
}


def run_entry(name, mode):
    """(outputs, leaves) of one forward + backward of `name` in `mode`; the calls land on the installed fake."""
    det = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(mode == "det")
    try:
        outs, loss, leaves = ENTRIES[name](_dtypes(mode))
        loss.backward()
    finally:
        torch.use_deterministic_algorithms(det)
    return outs, leaves


def _odd_offset(t):
    """A contiguous view of `t` one element into a fresh buffer: aligned to the element, never to an (x, y) pair."""
    buf = torch.zeros(t.numel() + 1, dtype=t.dtype)
    v = buf[1:].view(t.shape)
    v.copy_(t.detach())
    assert v.data_ptr() % (2 * v.element_size()) != 0
    return v.requires_grad_(t.requires_grad)


# symbol prefix -> the positions of its (x, y)-pair pointer arguments (include/umr_b200.h)
PAIR_ARGS = {"umr_bilinear_sample_forward": (1,), "umr_bilinear_sample_cells": (0,), "umr_bilinear_sample_backward": (1, 3),
             "umr_texcycle_forward": (0, 1), "umr_texcycle_backward": (0, 1, 4)}


@pytest.mark.parametrize("mode", ["f32", "det", "f64", "mixed"])
@pytest.mark.parametrize("op", ["sample", "texcycle"])
def test_odd_offset_pairs_reach_the_library_aligned(fake, op, mode):
    """Contiguous flow / prob views at an odd element offset: every pair pointer the library receives, forward and
    backward, is a multiple of 2 * sizeof(element), and an input already aligned in the compute dtype is passed in place."""
    dt = _dtypes(mode)
    det = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(mode == "det")
    try:
        if op == "sample":
            img, flow = _rand((2, 3, 4, 5), dt(0), True), _odd_offset(_rand((2, 6, 2), dt(1), True))
            aligned = _rand((2, 6, 2), dt(1), True)
            ops.bilinear_sample(img, flow).sum().backward()
            ops.bilinear_sample(img, aligned).sum().backward()
        else:
            flow, prob = _odd_offset(_rand((2, 3, 4, 2), dt(0), True)), _odd_offset(_rand((2, 3, 2), dt(1)))
            vis = torch.tensor([[1, 0, 1], [1, 1, 0]], dtype=torch.uint8)
            aligned = _rand((2, 3, 4, 2), dt(0), True)
            ops.tex_cycle(flow, prob, None, vis).backward()
            ops.tex_cycle(aligned, prob, None, vis).backward()
    finally:
        torch.use_deterministic_algorithms(det)
    assert flow.grad is not None and flow.grad.dtype == flow.dtype
    seen = 0
    for name, args in fake.calls:
        pos = [p for prefix, p in PAIR_ARGS.items() if name.startswith(prefix)]
        if not pos:
            continue
        size = 8 if name.endswith("_f64") else 4
        for k in pos[0]:
            assert args[k].value % (2 * size) == 0, "%s: argument %d at %#x" % (name, k, args[k].value)
            seen += 1
    assert seen >= (6 if op == "sample" else 10)
    # the second call's flow reaches the library in place when it already has the compute dtype
    forwards = [args for name, args in fake.calls if name.startswith(("umr_bilinear_sample_forward", "umr_texcycle_forward"))]
    if aligned.dtype == (torch.float64 if mode in ("f64", "mixed") else torch.float32):
        assert forwards[-1][1 if op == "sample" else 0].value == aligned.data_ptr()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", sorted(ENTRIES))
def test_dispatch(fake, name, mode):
    want = [w for modes, w in EXPECTED[name].items() if mode in modes.split()]
    assert len(want) == 1
    want = want[0]
    if isinstance(want, str):   # an error message
        with pytest.raises(ValueError, match=re.escape(want)):
            run_entry(name, mode)
        assert fake.calls == []
        return
    outs, leaves = run_entry(name, mode)
    assert trace(fake) == want
    f64 = any(s.split(":")[0].endswith("_f64") for s in want)
    for o in outs:
        assert o.dtype == (torch.float64 if f64 else torch.float32)
    assert leaves
    for t in leaves:
        assert t.grad is not None and t.grad.dtype == t.dtype
