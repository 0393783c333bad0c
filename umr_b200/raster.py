"""torch.autograd binding of the sm_90a soft rasteriser (C ABI: include/umr_b200.h).

Host-side mirror of the reference's autograd Function
`external/SoftRas/soft_renderer/functional/soft_rasterize.py:9-125` -- same arguments, same
returned triple -- except that everything the reference did on the host around its kernels is
fused into ours: no CPU-side buffer fills / H2D copies (soft_rasterize.py:47-62), no `grid`
tensor, in-kernel p2f normalisation (:73) and, optionally, the 2x2 anti-aliasing average pool of
`rasterizer.py:52-53` (`anti_aliasing=True`).

There is NO CPU path: CPU tensors raise (the reference intends the same, soft_rasterize.py:117-118).
"""
import ctypes
import math
import os

import torch

from . import _lib

FUNC_DIST = {"hard": 0, "barycentric": 1, "euclidean": 2}
FUNC_RGB = {"hard": 0, "softmax": 1}
FUNC_ALPHA = {"hard": 0, "sum": 1, "prod": 2}
FUNC_SAMPLE = {"surface": 0, "vertex": 1}


# --- optional live kernel timing (bench.py): the C ABI records a cudaEvent pair around the main raster
# kernel of every forward / backward call while a sink is installed ------------------------------
_profile_sink = None


class _EventPair(object):
    """Two cudaEvents owned by this object: destroyed by the finaliser, so a sink that is dropped without
    collect_profile() (exception, set_profile_sink(None) and forget) leaks nothing."""

    __slots__ = ("start", "stop")

    def __init__(self):
        lib = _lib.load()
        self.start, self.stop = ctypes.c_void_p(), ctypes.c_void_p()
        _lib.check(lib.umr_event_create(ctypes.byref(self.start)), "umr_event_create")
        try:
            _lib.check(lib.umr_event_create(ctypes.byref(self.stop)), "umr_event_create")
        except Exception:
            lib.umr_event_destroy(self.start)
            self.start = ctypes.c_void_p()
            raise

    def elapsed_ms(self):
        ms = ctypes.c_float()
        _lib.check(_lib.load().umr_event_elapsed_ms(self.start, self.stop, ctypes.byref(ms)), "umr_event_elapsed_ms")
        return float(ms.value)

    def __del__(self):
        try:
            lib = _lib.load()
            for e in (self.start, self.stop):
                if e is not None and e.value:
                    lib.umr_event_destroy(e)
        except Exception:  # interpreter shutdown
            pass


def set_profile_sink(sink):
    """sink: a list that receives (kind, _EventPair) per raster call, or None to stop."""
    global _profile_sink
    _profile_sink = sink


def _attach_events(params, kind):
    if _profile_sink is None:
        return
    ev = _EventPair()
    params.ev_kernel_start, params.ev_kernel_stop = ev.start.value, ev.stop.value
    _profile_sink.append((kind, ev))


def collect_profile(sink):
    """Elapsed milliseconds of every recorded kernel, grouped by kind; empties the sink (the events are
    destroyed with their _EventPair objects)."""
    out = {"fwd": [], "bwd": []}
    for kind, ev in sink or []:
        out[kind].append(ev.elapsed_ms())
    if sink is not None:
        del sink[:]
    return out


# --- pair buffer (saved (pixel, face) records streamed by the backward; include/umr_b200.h) -------------
# Budget in candidate pairs per raster pixel (measured: 2.7 at F=1280, 4.8 at F=5120, SURVEY.md App. C) and an
# upper bound on one render's buffer; tiles that do not fit are recomputed by the backward (same results).
PAIR_CAND_PER_PIXEL = float(os.environ.get("UMR_PAIR_CAND_PER_PIXEL", "8.0"))
FORWARD_TILE = int(os.environ.get("UMR_FORWARD_TILE", "0"))  # 0 auto | 16 | 32 (UmrRasterParams.tile_mode; tests force both)
# The bound is UMR_PAIR_MAX_GB, else a quarter of the device's memory (20 GB on an 80 GB H100): a train step keeps two
# renders alive until its backward (mask and texture branches), and those two then hold at most half of the card.
_PAIR_MAX_GB = os.environ.get("UMR_PAIR_MAX_GB")
_pair_max = {}  # device index -> bytes


def pair_max_bytes(device=None):
    if _PAIR_MAX_GB is not None:
        return int(float(_PAIR_MAX_GB) * (1 << 30))
    dev = torch.device("cuda" if device is None else device)
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    if idx not in _pair_max:
        _pair_max[idx] = torch.cuda.get_device_properties(idx).total_memory // 4
    return _pair_max[idx]


def pair_buffer_bytes(B, image_size, anti_aliasing, cand_per_pixel=None, blocks_per_image=None, device=None):
    lib = _lib.load()
    S = int(image_size) * (2 if anti_aliasing else 1)
    cpp = PAIR_CAND_PER_PIXEL if cand_per_pixel is None else cand_per_pixel
    tiles = B * ((S + 15) // 16) ** 2
    if blocks_per_image is not None:
        blocks = int(B * blocks_per_image * PAIR_HEADROOM) + 2 * tiles + 64
    else:
        blocks = int(B * S * S * cpp / 32.0) + 2 * tiles + 64
    nbytes = lib.umr_raster_pair_buffer_bytes(B, int(image_size), 1 if anti_aliasing else 0, blocks)
    return min(int(nbytes), pair_max_bytes(device))


# Adaptive sizing: after every forward the buffer's own counters (blocks the render WANTED, tiles left unsaved) are copied
# to pinned memory asynchronously; a later call with the same (raster size, face count) sizes its buffer from the largest
# need seen per image (x PAIR_HEADROOM) instead of the fixed budget -- 0.8 GB instead of 1.7 GB at C2.  A render that
# needs more than that just recomputes some tiles in its backward (same results) and the next one grows.  Nothing here
# synchronises; inside CUDA-graph capture the read-back is skipped.
PAIR_HEADROOM = float(os.environ.get("UMR_PAIR_HEADROOM", "1.35"))
PAIR_ADAPTIVE = os.environ.get("UMR_PAIR_ADAPTIVE", "1") != "0"
_pair_need = {}      # (S, F, tile_mode) -> blocks per image
_pair_pending = []   # (key, B, pinned int32[2], event)


def _pair_poll():
    keep = []
    for key, B, host, ev in _pair_pending:
        if ev.query():
            need = float(host[0]) / max(B, 1)
            _pair_need[key] = max(_pair_need.get(key, 0.0), need)
        else:
            keep.append((key, B, host, ev))
    _pair_pending[:] = keep


def _pair_record(key, B, pairs):
    if not PAIR_ADAPTIVE or torch.cuda.is_current_stream_capturing() or len(_pair_pending) > 64:
        return
    host = torch.empty(2, dtype=torch.int32, pin_memory=True)
    host.copy_(pairs[:8].view(torch.int32), non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    _pair_pending.append((key, B, host, ev))


def _stream_ptr(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def make_params(B, F, T2, image_size, anti_aliasing, background_color, near, far, fill_back, eps,
                sigma_val, dist_func, dist_eps, gamma_val, aggr_func_rgb, aggr_func_alpha, texture_type):
    p = _lib.UmrRasterParams()
    p.batch_size, p.num_faces, p.texture_size = B, F, T2
    p.image_size, p.anti_aliasing = int(image_size), 1 if anti_aliasing else 0
    p.near_plane, p.far_plane, p.eps = float(near), float(far), float(eps)
    p.sigma_val, p.gamma_val = float(sigma_val), float(gamma_val)
    p.dist_eps = float(math.log(1.0 / dist_eps - 1.0))  # soft_rasterize.py:35
    p.func_id_dist = FUNC_DIST[dist_func]
    p.func_id_rgb = FUNC_RGB[aggr_func_rgb]
    p.func_id_alpha = FUNC_ALPHA[aggr_func_alpha]
    p.texture_sample_type = FUNC_SAMPLE[texture_type]
    p.double_side = 1 if fill_back else 0
    for k in range(3):
        p.background_color[k] = float(background_color[k])
    return p


# --- float64 path (umr_raster_forward_f64 / umr_raster_backward_f64, DESIGN.md §9): float64 face vertices select it, as the
# reference's kernels dispatch on `faces.type()`.  Everything is float64 (textures and incoming gradients are converted),
# there is no pair buffer, and the kernels are bitwise reproducible, so torch.use_deterministic_algorithms changes nothing.
def _forward_f64(ctx, face_vertices, textures, image_size, background_color, near, far, fill_back, eps, sigma_val,
                 dist_func, dist_eps, gamma_val, aggr_func_rgb, aggr_func_alpha, texture_type, anti_aliasing):
    lib = _lib.load()
    dev = face_vertices.device
    B, F = face_vertices.shape[:2]
    fv = face_vertices.detach().reshape(B, F, 9).contiguous()
    Bt = textures.shape[0]
    if Bt != B and (Bt <= 0 or B % Bt != 0):
        raise ValueError("textures batch %d does not divide face_vertices batch %d" % (Bt, B))
    group = B // Bt
    tex = textures.detach().contiguous().double()
    if int(tex.shape[-1]) != 3:
        raise ValueError("float64 rasterisation takes 3 colour channels, got %d (part-map textures are float32 only)"
                         % int(tex.shape[-1]))
    S = int(image_size) * (2 if anti_aliasing else 1)
    params = make_params(B, F, tex.shape[2], image_size, anti_aliasing, background_color, near, far, fill_back, eps,
                         sigma_val, dist_func, dist_eps, gamma_val, aggr_func_rgb, aggr_func_alpha, texture_type)
    params.shared_textures = group if group > 1 else 0
    params.color_channels = 3
    need_bwd = face_vertices.requires_grad or textures.requires_grad
    _attach_events(params, "fwd")
    with torch.cuda.device(dev):
        images = torch.empty(B, 4, image_size, image_size, device=dev, dtype=torch.float64)
        colors_hi = images
        if anti_aliasing:
            colors_hi = torch.empty(B, 4, S, S, device=dev, dtype=torch.float64) if need_bwd else None
        aggrs = torch.empty(B, 2, S, S, device=dev, dtype=torch.float64)
        p2f = torch.empty(B, F, 2, device=dev, dtype=torch.float64)
        ws = torch.empty(lib.umr_raster_workspace_bytes_f64(B, F, int(image_size), params.anti_aliasing), device=dev,
                         dtype=torch.uint8)
        rc = lib.umr_raster_forward_f64(_ptr(fv), _ptr(tex), _ptr(images), _ptr(colors_hi) if anti_aliasing else _ptr(None),
                                        _ptr(aggrs), _ptr(p2f), ctypes.byref(params), _ptr(ws), _stream_ptr(dev))
    _lib.check(rc, "umr_raster_forward_f64")
    params.ev_kernel_start = params.ev_kernel_stop = None
    ctx.params = params
    ctx.in_shape = tuple(face_vertices.shape)
    ctx.tex_needs_grad = textures.requires_grad
    ctx.geom_needs_grad = face_vertices.requires_grad
    ctx.tex_dtype = textures.dtype
    if need_bwd:
        ctx.save_for_backward(fv, tex, colors_hi, aggrs)
    ctx.mark_non_differentiable(p2f, aggrs)
    return images, p2f, aggrs


def _backward_f64(ctx, grad_images):
    lib = _lib.load()
    fv, tex, colors_hi, aggrs = ctx.saved_tensors
    dev = fv.device
    B, F = fv.shape[:2]
    g = grad_images.contiguous().double()
    _attach_events(ctx.params, "bwd")
    with torch.cuda.device(dev):
        grad_faces = torch.empty_like(fv) if ctx.geom_needs_grad else None
        grad_tex = torch.empty_like(tex) if ctx.tex_needs_grad else None
        ws = torch.empty(lib.umr_raster_workspace_bytes_f64(B, F, ctx.params.image_size, ctx.params.anti_aliasing),
                         device=dev, dtype=torch.uint8)
        rc = lib.umr_raster_backward_f64(_ptr(fv), _ptr(tex), _ptr(colors_hi), _ptr(aggrs), _ptr(g), _ptr(grad_faces),
                                         _ptr(grad_tex), ctypes.byref(ctx.params), _ptr(ws), _stream_ptr(dev))
    _lib.check(rc, "umr_raster_backward_f64")
    ctx.params.ev_kernel_start = ctx.params.ev_kernel_stop = None
    if grad_tex is not None:
        grad_tex = grad_tex.to(ctx.tex_dtype)  # textures of another dtype were converted on the way in
    return (None if grad_faces is None else grad_faces.view(ctx.in_shape), grad_tex) + (None,) * 14


class SoftRasterizeFunction(torch.autograd.Function):
    """forward(face_vertices[B,F,3,3|9], textures[B,F,T2,3], ...) ->
    (images[B,4,is,is], p2f_info[B,F,2], aggrs_info[B,2,S,S]),  S = is * (2 if anti_aliasing else 1).
    float64 face_vertices render in double precision and return float64; every other dtype renders in float32."""

    @staticmethod
    def forward(ctx, face_vertices, textures, image_size=256, background_color=(0, 0, 0), near=1,
                far=100, fill_back=True, eps=1e-3, sigma_val=1e-5, dist_func="euclidean",
                dist_eps=1e-4, gamma_val=1e-4, aggr_func_rgb="softmax", aggr_func_alpha="prod",
                texture_type="surface", anti_aliasing=False):
        if not face_vertices.is_cuda or not textures.is_cuda:
            raise TypeError("Rasterize module supports only cuda Tensors")  # soft_rasterize.py:117-118
        ctx.f64 = face_vertices.dtype == torch.float64
        if ctx.f64:
            return _forward_f64(ctx, face_vertices, textures, image_size, background_color, near, far, fill_back, eps,
                                sigma_val, dist_func, dist_eps, gamma_val, aggr_func_rgb, aggr_func_alpha, texture_type,
                                anti_aliasing)
        lib = _lib.load()
        dev = face_vertices.device
        B, F = face_vertices.shape[:2]
        fv = face_vertices.detach().reshape(B, F, 9).contiguous().float()
        # a [1,F,T2,3] texture with B > 1 is a batch-SHARED parameter: the kernels read the one copy for every image and
        # accumulate its gradient directly (the reference materialises repeat(B,...) copies, loss_utils.py:305)
        # fewer textures than renders: every B / Bt consecutive renders share one texture -- Bt == 1: a batch-shared
        # parameter; Bt == B / 8: the 8 camera hypotheses of each sample (the reference materialises repeat(...) copies,
        # loss_utils.py:305).  The kernels index textures[b // group] and accumulate the group's gradient directly.
        Bt = textures.shape[0]
        if Bt != B and (Bt <= 0 or B % Bt != 0):
            raise ValueError("textures batch %d does not divide face_vertices batch %d" % (Bt, B))
        group = B // Bt
        tex = textures.detach().contiguous().float()
        T2 = tex.shape[2]
        # colour channels: 3, or 4 for the one-render part maps of part_matching_loss (SURVEY.md §8f-2); images then
        # carry NC + 1 planes (colours + alpha)
        NC = int(tex.shape[-1]) if texture_type == "surface" else 3
        if NC not in (3, 4):
            raise ValueError("textures must have 3 (or, surface textures only, 4) colour channels, got %d" % NC)
        S = int(image_size) * (2 if anti_aliasing else 1)
        params = make_params(B, F, T2, image_size, anti_aliasing, background_color, near, far, fill_back,
                             eps, sigma_val, dist_func, dist_eps, gamma_val, aggr_func_rgb,
                             aggr_func_alpha, texture_type)
        params.shared_textures = group if group > 1 else 0
        params.tile_mode = FORWARD_TILE
        params.color_channels = NC
        if NC == 4:
            params.background_extra = float(background_color[3]) if len(background_color) > 3 else 0.0
            if textures.requires_grad:
                raise ValueError("4-channel (part-map) textures are constants: no texture gradient is built")
        need_bwd = face_vertices.requires_grad or textures.requires_grad
        generic = dist_func != "euclidean" or aggr_func_alpha != "prod" or texture_type != "surface"
        # torch.use_deterministic_algorithms(True): bitwise-reproducible kernels (include/umr_b200.h), read once here so the
        # backward runs in the mode of its forward
        det = torch.are_deterministic_algorithms_enabled()
        _attach_events(params, "fwd")
        with torch.cuda.device(dev):
            images = torch.empty(B, NC + 1, image_size, image_size, device=dev, dtype=torch.float32)
            if anti_aliasing:
                colors_hi = torch.empty(B, NC + 1, S, S, device=dev, dtype=torch.float32) if need_bwd else None
            else:
                colors_hi = images
            aggrs = torch.empty(B, 2, S, S, device=dev, dtype=torch.float32)
            p2f = torch.empty(B, F, 2, device=dev, dtype=torch.float32)
            ws_bytes = lib.umr_raster_workspace_bytes_deterministic if det else lib.umr_raster_workspace_bytes
            ws = torch.empty(ws_bytes(B, F, int(image_size), params.anti_aliasing), device=dev, dtype=torch.uint8)
            pairs = None
            pair_key = (S, F, FORWARD_TILE)
            if need_bwd and not generic and not det and PAIR_CAND_PER_PIXEL > 0:
                capturing = torch.cuda.is_current_stream_capturing()
                if PAIR_ADAPTIVE and not capturing:
                    _pair_poll()
                need = _pair_need.get(pair_key) if (PAIR_ADAPTIVE and PAIR_CAND_PER_PIXEL >= 1.0) else None
                pairs = torch.empty(pair_buffer_bytes(B, image_size, anti_aliasing, blocks_per_image=need, device=dev), device=dev,
                                    dtype=torch.uint8)
                params.pair_buffer, params.pair_buffer_bytes = pairs.data_ptr(), pairs.numel()
            fwd = lib.umr_raster_forward_deterministic if det else lib.umr_raster_forward
            rc = fwd(_ptr(fv), _ptr(tex), _ptr(images),
                                        _ptr(colors_hi) if anti_aliasing else _ptr(None),
                                        _ptr(aggrs), _ptr(p2f), ctypes.byref(params), _ptr(ws),
                                        _stream_ptr(dev))
        _lib.check(rc, "umr_raster_forward_deterministic" if det else "umr_raster_forward")
        if pairs is not None:
            _pair_record(pair_key, B, pairs)
        params.ev_kernel_start = params.ev_kernel_stop = None
        ctx.params = params
        ctx.in_shape = tuple(face_vertices.shape)
        ctx.tex_needs_grad = textures.requires_grad
        ctx.geom_needs_grad = face_vertices.requires_grad
        ctx.has_pairs = pairs is not None
        ctx.det = det
        if need_bwd:
            if pairs is not None:
                ctx.save_for_backward(fv, tex, colors_hi, aggrs, pairs)
            else:
                ctx.save_for_backward(fv, tex, colors_hi, aggrs)
        ctx.mark_non_differentiable(p2f, aggrs)
        return images, p2f, aggrs

    @staticmethod
    def backward(ctx, grad_images, grad_p2f=None, grad_aggrs=None):
        if ctx.f64:
            return _backward_f64(ctx, grad_images)
        lib = _lib.load()
        if ctx.has_pairs:
            fv, tex, colors_hi, aggrs, pairs = ctx.saved_tensors
            assert ctx.params.pair_buffer == pairs.data_ptr()
        else:
            fv, tex, colors_hi, aggrs = ctx.saved_tensors
        dev = fv.device
        B, F = fv.shape[:2]
        g = grad_images.contiguous().float()
        _attach_events(ctx.params, "bwd")
        with torch.cuda.device(dev):
            # detached geometry (UMR's texture branch, train_s2.py:248): texture-only backward, no vertex arithmetic
            tex_only = ctx.tex_needs_grad and not ctx.geom_needs_grad and (ctx.has_pairs or ctx.det)
            grad_faces = None if tex_only else torch.empty_like(fv)
            grad_tex = torch.empty_like(tex) if ctx.tex_needs_grad else None
            ws_bytes = lib.umr_raster_workspace_bytes_deterministic if ctx.det else lib.umr_raster_workspace_bytes
            ws = torch.empty(ws_bytes(B, F, ctx.params.image_size, ctx.params.anti_aliasing), device=dev, dtype=torch.uint8)
            bwd = lib.umr_raster_backward_deterministic if ctx.det else lib.umr_raster_backward
            rc = bwd(_ptr(fv), _ptr(tex), _ptr(colors_hi), _ptr(aggrs), _ptr(g),
                                         _ptr(grad_faces), _ptr(grad_tex), ctypes.byref(ctx.params),
                                         _ptr(ws), _stream_ptr(dev))
        _lib.check(rc, "umr_raster_backward_deterministic" if ctx.det else "umr_raster_backward")
        ctx.params.ev_kernel_start = ctx.params.ev_kernel_stop = None
        return (None if grad_faces is None else grad_faces.view(ctx.in_shape), grad_tex) + (None,) * 14


def soft_rasterize(face_vertices, textures, image_size=256, background_color=(0, 0, 0), near=1, far=100,
                   fill_back=True, eps=1e-3, sigma_val=1e-5, dist_func="euclidean", dist_eps=1e-4,
                   gamma_val=1e-4, aggr_func_rgb="softmax", aggr_func_alpha="prod", texture_type="surface",
                   anti_aliasing=False):
    """Drop-in for `soft_renderer.functional.soft_rasterize` (soft_rasterize.py:111-125), plus the
    optional fused `anti_aliasing` pool (then `image_size` is the OUTPUT size and the raster runs at 2x)."""
    return SoftRasterizeFunction.apply(face_vertices, textures, image_size, background_color, near, far,
                                       fill_back, eps, sigma_val, dist_func, dist_eps, gamma_val,
                                       aggr_func_rgb, aggr_func_alpha, texture_type, anti_aliasing)


def visibility(face_vertices, image_size=256, near=1, far=100, fill_back=True, eps=1e-3, sigma_val=1e-5,
               dist_eps=1e-4, gamma_val=1e-4, anti_aliasing=False, want_faces=False):
    """The hard z-buffer's winner per raster pixel and nothing else: returns aggrs_info [B,2,S,S] = (depth_min,
    float(face_index_min)), bit-identical to `soft_rasterize(..., aggr_func_rgb="hard")[2]` (euclidean / prod / surface
    configuration), without the distance / sigmoid / alpha / colour arithmetic and without image planes.  It is all the
    reference keeps of the hard render in MultiTextureLoss (nnutils/loss_utils.py:327-329).  No gradient (the reference
    detaches its inputs there).

    want_faces=True returns instead the [B,F] uint8 "face wins at least one pixel" bytes TexCycle derives from the plane
    (a background pixel marks face F-1, like the reference's negative index) and writes no plane at all."""
    if not face_vertices.is_cuda:
        raise TypeError("Rasterize module supports only cuda Tensors")  # soft_rasterize.py:117-118
    lib = _lib.load()
    dev = face_vertices.device
    B, F = face_vertices.shape[:2]
    fv = face_vertices.detach().reshape(B, F, 9).contiguous().float()
    S = int(image_size) * (2 if anti_aliasing else 1)
    params = make_params(B, F, 1, image_size, anti_aliasing, (0, 0, 0), near, far, fill_back, eps, sigma_val, "euclidean",
                         dist_eps, gamma_val, "hard", "prod", "surface")
    _attach_events(params, "fwd")
    with torch.cuda.device(dev):
        aggrs = None if want_faces else torch.empty(B, 2, S, S, device=dev, dtype=torch.float32)
        faces = torch.empty(B, F, device=dev, dtype=torch.uint8) if want_faces else None
        ws = torch.empty(lib.umr_raster_workspace_bytes(B, F, int(image_size), params.anti_aliasing), device=dev,
                         dtype=torch.uint8)
        rc = lib.umr_raster_visibility(_ptr(fv), _ptr(aggrs), _ptr(faces), ctypes.byref(params), _ptr(ws), _stream_ptr(dev))
    _lib.check(rc, "umr_raster_visibility")
    params.ev_kernel_start = params.ev_kernel_stop = None
    return faces if want_faces else aggrs
