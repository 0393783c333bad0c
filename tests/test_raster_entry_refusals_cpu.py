"""Return codes of the 13 raster C entry points for every input they refuse (no GPU).

Each entry point runs its parameter checks, its buffer checks and its mode refusals before any device work, in a fixed
order.  `expected()` restates that order for each family; every case below is refused by it, so no call reaches the
device and the fake buffer addresses are never touched.  A case the library accepted would, without a GPU, come back as
a CUDA error and fail the comparison."""
import ctypes

import pytest

from umr_b200 import _lib, raster

OK, UNSUPPORTED, BAD_ARG, TOO_LARGE = 0, -1, -2, -3
MAX_FACES = 16777216
MAX_RASTER = 65535 * 16  # raster side limit of the deterministic float32 and the float64 entry points

FAKE = 256                # non-NULL and 256-byte aligned
ODD = 256 + 2             # not 4-byte aligned
WS_ODD = 256 + 16         # 4-byte aligned, not 256-byte aligned (the workspace)

# name -> (family, deterministic, pointer arguments before the params block)
ENTRY_POINTS = {
    "umr_raster_forward": ("forward", False, ("fv", "tex", "images", "soft", "aggrs", "p2f")),
    "umr_raster_forward_deterministic": ("forward", True, ("fv", "tex", "images", "soft", "aggrs", "p2f")),
    "umr_raster_forward_f64": ("forward_f64", True, ("fv", "tex", "images", "soft", "aggrs", "p2f")),
    "umr_raster_visibility": ("visibility", False, ("fv", "aggrs", "vis")),
    "umr_raster_backward": ("backward", False, ("fv", "tex", "soft", "aggrs", "gimg", "gf", "gt")),
    "umr_raster_backward_deterministic": ("backward", True, ("fv", "tex", "soft", "aggrs", "gimg", "gf", "gt")),
    "umr_raster_backward_split": ("split", False, ("fv", "tex", "soft", "aggrs", "gimg", "gf", "gt")),
    "umr_raster_backward_split_deterministic": ("split", True, ("fv", "tex", "soft", "aggrs", "gimg", "gf", "gt")),
    "umr_raster_backward_f64": ("backward_f64", True, ("fv", "tex", "soft", "aggrs", "gimg", "gf", "gt")),
    "umr_raster_forward_silhouette": ("sil_forward", False, ("fv", "alpha", "alpha_hi")),
    "umr_raster_forward_silhouette_deterministic": ("sil_forward", True, ("fv", "alpha", "alpha_hi")),
    "umr_raster_backward_silhouette": ("sil_backward", False, ("fv", "alpha_hi", "galpha", "gf")),
    "umr_raster_backward_silhouette_deterministic": ("sil_backward", True, ("fv", "alpha_hi", "galpha", "gf")),
}


def _params(**kw):
    cfg = dict(B=2, F=4, T2=4, image_size=8, anti_aliasing=False, background_color=(0, 0, 0), near=1, far=100,
               fill_back=True, eps=1e-3, sigma_val=1e-5, dist_func="euclidean", dist_eps=1e-4, gamma_val=1e-4,
               aggr_func_rgb="softmax", aggr_func_alpha="prod", texture_type="surface")
    cfg.update(kw)
    return raster.make_params(**cfg)


def _with(**fields):
    p = _params()
    for k, v in fields.items():
        setattr(p, k, v)
    return p


HUGE = dict(image_size=MAX_RASTER + 1)          # raster side past the limit, without anti-aliasing
HUGE_AA = dict(image_size=MAX_RASTER // 2 + 1, anti_aliasing=1)
GENERIC = {"dist hard": dict(func_id_dist=0), "dist barycentric": dict(func_id_dist=1), "alpha hard": dict(func_id_alpha=0),
           "alpha sum": dict(func_id_alpha=1), "vertex textures": dict(texture_sample_type=1, texture_size=3)}

# every single invalid field of the parameter checks, the mode refusals, and the combinations that pin their order
PARAMS = {
    "valid": {},
    "batch_size 0": dict(batch_size=0),
    "batch_size -1": dict(batch_size=-1),
    "num_faces 0": dict(num_faces=0),
    "texture_size 0": dict(texture_size=0),
    "image_size 0": dict(image_size=0),
    "image_size -8": dict(image_size=-8),
    "num_faces past the limit": dict(num_faces=MAX_FACES + 1),
    "batch_size 65536": dict(batch_size=65536),
    "func_id_dist -1": dict(func_id_dist=-1),
    "func_id_dist 3": dict(func_id_dist=3),
    "func_id_alpha -1": dict(func_id_alpha=-1),
    "func_id_alpha 3": dict(func_id_alpha=3),
    "texture_sample_type -1": dict(texture_sample_type=-1),
    "texture_sample_type 2": dict(texture_sample_type=2),
    "vertex textures with texture_size 4": dict(texture_sample_type=1, texture_size=4),
    "shared_textures 3 of batch 2": dict(shared_textures=3),
    "shared_textures 2": dict(shared_textures=2),
    "func_id_rgb -1": dict(func_id_rgb=-1),
    "func_id_rgb 2": dict(func_id_rgb=2),
    "hard colours": dict(func_id_rgb=0),
    "color_channels -1": dict(color_channels=-1),
    "color_channels 1": dict(color_channels=1),
    "color_channels 2": dict(color_channels=2),
    "color_channels 3": dict(color_channels=3),
    "color_channels 4": dict(color_channels=4),
    "color_channels 5": dict(color_channels=5),
    "color_channels 4, hard colours": dict(color_channels=4, func_id_rgb=0),
    "raster past the limit": HUGE,
    "raster past the limit (anti-aliasing)": HUGE_AA,
    # precedence: the float64 limit comes before the mode-id checks, the deterministic float32 one after all of them
    "raster past the limit, func_id_dist 7": dict(HUGE, func_id_dist=7),
    "raster past the limit, func_id_rgb 7": dict(HUGE, func_id_rgb=7),
    "raster past the limit, vertex textures with texture_size 4": dict(HUGE, texture_sample_type=1, texture_size=4),
    "raster past the limit, color_channels 5": dict(HUGE, color_channels=5),
    "raster past the limit, color_channels 4": dict(HUGE, color_channels=4),
    "raster past the limit, batch_size 65536": dict(HUGE, batch_size=65536),
    "raster past the limit, dist barycentric": dict(HUGE, func_id_dist=1),
}
for _name, _kw in GENERIC.items():
    PARAMS[_name] = _kw
    PARAMS[_name + ", color_channels 4"] = dict(_kw, color_channels=4)


def _generic(p):
    return p.func_id_dist != 2 or p.func_id_alpha != 2 or p.texture_sample_type != 0


def _raster_side(p):
    return p.image_size * (2 if p.anti_aliasing else 1)


def _check_params(p, f64):
    if p is None:
        return BAD_ARG
    if p.batch_size <= 0 or p.num_faces <= 0 or p.texture_size <= 0 or p.image_size <= 0:
        return BAD_ARG
    if p.num_faces > MAX_FACES or p.batch_size > 65535:
        return TOO_LARGE
    if f64 and _raster_side(p) > MAX_RASTER:
        return TOO_LARGE
    if not (0 <= p.func_id_dist <= 2 and 0 <= p.func_id_alpha <= 2 and 0 <= p.texture_sample_type <= 1):
        return UNSUPPORTED
    if p.texture_sample_type == 1 and p.texture_size != 3:
        return BAD_ARG
    if p.shared_textures > 1 and p.batch_size % p.shared_textures != 0:
        return BAD_ARG
    if p.func_id_rgb not in (0, 1):
        return UNSUPPORTED
    if p.color_channels not in ((0, 3) if f64 else (0, 3, 4)):
        return BAD_ARG
    if p.color_channels == 4 and (_generic(p) or p.func_id_rgb != 1):
        return UNSUPPORTED
    return OK


def expected(family, det, p, a):
    """The code the entry point returns before any device work, or None when it accepts the call."""
    f64 = family.endswith("_f64")
    rc = _check_params(p, f64)
    if rc:
        return rc
    too_large = det and not f64 and _raster_side(p) > MAX_RASTER
    ws_bad = a["ws"] is None or a["ws"] % 256 != 0
    if family in ("forward", "forward_f64"):
        if too_large:
            return TOO_LARGE
        if any(a[k] is None for k in ("fv", "tex", "images", "aggrs")) or ws_bad:
            return BAD_ARG
        return None
    if family == "visibility":
        if a["fv"] is None or (a["aggrs"] is None and a["vis"] is None) or ws_bad:
            return BAD_ARG
        return UNSUPPORTED if _generic(p) else None
    if family in ("backward", "split", "backward_f64"):
        if family == "split" and (a["gf"] is None or a["gt"] is None or _generic(p) or p.color_channels == 4):
            return BAD_ARG
        if too_large:
            return TOO_LARGE
        if any(a[k] is None for k in ("fv", "tex", "soft", "aggrs", "gimg")) or (a["gf"] is None and a["gt"] is None):
            return BAD_ARG
        if ws_bad:
            return BAD_ARG
        if f64:
            return None
        if p.color_channels == 4 and a["gt"] is not None:
            return UNSUPPORTED  # part maps take no texture gradient
        if not det and a["gf"] is None and _generic(p):
            return UNSUPPORTED  # the texture-only backward exists for UMR's configuration only
        return None
    # silhouette
    if _generic(p) or p.color_channels == 4:
        return BAD_ARG
    if too_large:
        return TOO_LARGE
    names = ENTRY_POINTS["umr_raster_forward_silhouette" if family == "sil_forward" else "umr_raster_backward_silhouette"][2]
    required = ("fv", "alpha") if family == "sil_forward" else names
    if any(a[k] is None for k in required) or ws_bad:
        return BAD_ARG
    if any(a[k] is not None and a[k] % 4 != 0 for k in names):
        return BAD_ARG
    return None


def _buffer_cases(family, names):
    """All buffers valid, then each one NULL, each one misaligned, and the pairs that matter together."""
    base = dict({k: FAKE for k in names}, ws=FAKE)
    cases = [base]
    for k in list(names) + ["ws"]:
        cases.append(dict(base, **{k: None}))
        cases.append(dict(base, **{k: WS_ODD if k == "ws" else ODD}))
    if family == "visibility":
        cases.append(dict(base, aggrs=None, vis=None))
    if family in ("backward", "split", "backward_f64"):
        cases.append(dict(base, gf=None, gt=None))
        cases.append(dict(base, gf=None, ws=WS_ODD))
        cases.append(dict(base, fv=None, gf=None))
    return cases


def _call(lib, name, p, a):
    names = ENTRY_POINTS[name][2]
    return getattr(lib, name)(*[a[k] for k in names], ctypes.byref(p) if p is not None else None, a["ws"], None)


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


@pytest.mark.parametrize("name", sorted(ENTRY_POINTS))
def test_null_params_block(lib, name):
    family, det, names = ENTRY_POINTS[name]
    for a in _buffer_cases(family, names):
        assert _call(lib, name, None, a) == BAD_ARG, a


@pytest.mark.parametrize("case", sorted(PARAMS))
@pytest.mark.parametrize("name", sorted(ENTRY_POINTS))
def test_refusals(lib, name, case):
    family, det, names = ENTRY_POINTS[name]
    p = _with(**PARAMS[case])
    refused = 0
    for a in _buffer_cases(family, names):
        want = expected(family, det, p, a)
        if want is None:
            continue  # accepted: it would go on to the device
        assert _call(lib, name, p, a) == want, (case, a)
        refused += 1
    assert refused > 0


def test_precedence_examples(lib):
    """The orders the families differ in, stated directly."""
    bufs = lambda name: dict({k: FAKE for k in ENTRY_POINTS[name][2]}, ws=FAKE)
    # float64 checks its raster limit before the mode ids; float32 checks the mode ids first
    p = _with(**PARAMS["raster past the limit, func_id_dist 7"])
    assert _call(lib, "umr_raster_forward_f64", p, bufs("umr_raster_forward_f64")) == TOO_LARGE
    assert _call(lib, "umr_raster_backward_f64", p, bufs("umr_raster_backward_f64")) == TOO_LARGE
    for name in ("umr_raster_forward_deterministic", "umr_raster_backward_deterministic", "umr_raster_forward"):
        assert _call(lib, name, p, bufs(name)) == UNSUPPORTED
    # the deterministic float32 limit comes after all of the parameter checks, and before the buffers
    p = _with(**PARAMS["raster past the limit, color_channels 5"])
    assert _call(lib, "umr_raster_forward_deterministic", p, bufs("umr_raster_forward_deterministic")) == BAD_ARG
    assert _call(lib, "umr_raster_forward_f64", p, bufs("umr_raster_forward_f64")) == TOO_LARGE
    p = _with(**HUGE)
    assert _call(lib, "umr_raster_backward_deterministic", p, dict(bufs("umr_raster_backward"), fv=None)) == TOO_LARGE
    assert _call(lib, "umr_raster_backward", p, dict(bufs("umr_raster_backward"), fv=None)) == BAD_ARG
    # the split refusal comes before the deterministic limit
    assert _call(lib, "umr_raster_backward_split_deterministic", p, dict(bufs("umr_raster_backward"), gf=None)) == BAD_ARG
    assert _call(lib, "umr_raster_backward_deterministic", p, dict(bufs("umr_raster_backward"), gf=None)) == TOO_LARGE
    # generic modes: the silhouette and split entry points answer BAD_ARG, the visibility render UNSUPPORTED
    p = _with(func_id_dist=1)
    for name in ("umr_raster_forward_silhouette", "umr_raster_backward_silhouette_deterministic",
                 "umr_raster_backward_split"):
        assert _call(lib, name, p, bufs(name)) == BAD_ARG
    assert _call(lib, "umr_raster_visibility", p, bufs("umr_raster_visibility")) == UNSUPPORTED
    assert _call(lib, "umr_raster_visibility", p, dict(bufs("umr_raster_visibility"), fv=None)) == BAD_ARG


@pytest.mark.parametrize("case", sorted(GENERIC))
def test_generic_texture_only_backward_is_refused(lib, case):
    """A texture-only backward in a generic mode is refused before any device work (the streamed kernels that take it
    exist for UMR's configuration only); the deterministic and float64 backwards take it."""
    p = _with(**GENERIC[case])
    a = dict({k: FAKE for k in ENTRY_POINTS["umr_raster_backward"][2]}, ws=FAKE, gf=None)
    assert _call(lib, "umr_raster_backward", p, a) == UNSUPPORTED
    assert expected("backward", True, p, a) is None and expected("backward_f64", True, p, a) is None
