"""The NMR renderer kernels (csrc/nmr.cu) across their accepted input range, against the CPU oracle (oracle/nmr.py).

Forward planes (face index, raster depth, rgb, alpha, depth) are compared bit-exact (NaN equals NaN only), through the
C ABI so that pointer offsets and NULL outputs are the test's choice.  Every input sits between guard values (NaN, or
an out-of-range index), every output is prefilled with a NaN payload (or INT_MIN) inside guards: a stray read shows as
a difference from the oracle, a stray write as a changed guard, an unwritten element as a left-over prefill.  Each case
asserts, and prints, a count of the feature it targets.

The texture gradient (default and deterministic entry points) is held to a derived bound: each of the n terms landing
on a texel is (l * w) * g, two roundings (the / 4 of the pool is exact), and the n terms are summed in some order, so
|got - ref| <= gamma_{n+2} * sum |l w g| with gamma_k = k u / (1 - k u), u = 2^-24.  Each case prints its largest
error / bound ratio.  The scenes are in tests/nmr_scenes.py; tests/test_nmr_range_cpu.py checks the oracle on them."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

import nmr as oracle
import nmr_scenes as sc
from umr_b200 import _lib
from umr_b200.raster import _stream_ptr

pytestmark = pytest.mark.gpu
f32 = np.float32
EYE = sc.EYE
DEV = torch.device("cuda:0")
GUARD = 64                                       # guard elements (256 bytes) either side of every buffer
IN_F, IN_I = 0x7fc00000, 2 ** 31 - 1             # input guards: NaN, an index outside [0, V)
OUT_F, OUT_I = 0x7fd1e5e5, -2 ** 31              # output prefill: a NaN payload the kernels never produce, INT_MIN
U = 2.0 ** -24
LIGHT0 = dict(Ia=0.5, Id=0.5, ca=(1, 1, 1), cd=(1, 1, 1), direction=(0, 1, 0))


@pytest.fixture(params=[False, True], ids=["default", "deterministic"])
def det(request):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(request.param)
    yield request.param
    torch.use_deterministic_algorithms(prev)


class Buf:
    """n 4-byte elements at element offset GUARD + off of a device buffer filled with `fill` bits."""

    def __init__(self, n, fill, off=0, data=None):
        self.n, self.fill, self.o = n, fill, GUARD + off
        self.buf = torch.full((n + 2 * GUARD + off,), fill, dtype=torch.int32, device=DEV)
        if data is not None:
            self.buf[self.o:self.o + n] = torch.from_numpy(np.ascontiguousarray(data).view(np.int32).ravel()).to(DEV)

    def ptr(self):
        return ctypes.c_void_p(self.buf.data_ptr() + 4 * self.o)

    def body(self):
        return self.buf[self.o:self.o + self.n]

    def check(self, name, output):
        assert (self.buf[:self.o] == self.fill).all() and (self.buf[self.o + self.n:] == self.fill).all(), \
            "%s: a guard element changed" % name
        if output:
            left = int((self.body() == self.fill).sum())
            assert left == 0, "%s: %d elements not written" % (name, left)


def params(B, V, F, T, IS, aa=True, fill_back=True, G=1, eye=EYE, near=0.1, far=100.0, bg=(0, 0, 0), **light):
    lt = dict(LIGHT0, **light)
    p = _lib.UmrNmrParams()
    p.batch_size, p.num_vertices, p.num_faces, p.texture_res = B, V, F, T
    p.image_size, p.anti_aliasing, p.fill_back, p.shared_textures = IS, int(aa), int(fill_back), G
    p.eye_z, p.near_plane, p.far_plane = eye, near, far
    p.light_intensity_ambient, p.light_intensity_directional = lt["Ia"], lt["Id"]
    p.light_color_ambient[:], p.light_color_directional[:], p.light_direction[:] = lt["ca"], lt["cd"], lt["direction"]
    p.background_color[:] = bg
    return p


def forward(verts, faces, tex, IS, outs=("rgb", "alpha", "depth"), offsets=(), host=True, **kw):
    """umr_nmr_forward on guarded buffers.  `outs`: the non-NULL outputs; `offsets`: outputs placed 4 bytes off their
    16-byte alignment.  Returns the planes (numpy, or device int32 bit views with host=False) and a backward(g, det,
    off) closure."""
    lib = _lib.load()
    B, V = verts.shape[:2]
    F = faces.shape[1]
    T = 0 if tex is None else tex.shape[2]
    G = 1 if tex is None else B // tex.shape[0]   # (a G in kw is for the oracle)
    p = params(B, V, F, T, IS, G=G, **{k: x for k, x in kw.items() if k != "G"})
    S = IS * (2 if p.anti_aliasing else 1)
    ins = {"vertices": Buf(verts.size, IN_F, data=np.asarray(verts, f32)),
           "faces": Buf(faces.size, IN_I, data=np.asarray(faces, np.int32))}
    if tex is not None:
        ins["textures"] = Buf(tex.size, IN_F, data=np.asarray(tex, f32))
    ws = torch.empty(lib.umr_nmr_workspace_bytes(B, F, p.fill_back), device=DEV, dtype=torch.uint8)
    o = {"face_index": Buf(B * S * S, OUT_I), "raster_depth": Buf(B * S * S, OUT_F)}
    for n, size in (("rgb", B * 3 * IS * IS), ("alpha", B * IS * IS), ("depth", B * IS * IS)):
        if n in outs and (n != "rgb" or tex is not None):
            o[n] = Buf(size, OUT_F, off=1 if n in offsets else 0)
    nul = ctypes.c_void_p(0)
    rc = lib.umr_nmr_forward(ins["vertices"].ptr(), ins["faces"].ptr(),
                             ins["textures"].ptr() if tex is not None else nul,
                             o["face_index"].ptr(), o["raster_depth"].ptr(),
                             *[o[n].ptr() if n in o else nul for n in ("rgb", "alpha", "depth")],
                             ctypes.byref(p), ctypes.c_void_p(ws.data_ptr()), _stream_ptr(DEV))
    _lib.check(rc, "umr_nmr_forward")
    torch.cuda.synchronize()
    for n, b in ins.items():
        b.check(n, False)
        assert torch.equal(b.body(), torch.from_numpy(np.ascontiguousarray({"vertices": verts, "faces": faces,
                                                                             "textures": tex}[n]).view(np.int32).ravel()).to(DEV))
    for n, b in o.items():
        b.check(n, True)
    shapes = {"face_index": (B, S, S), "raster_depth": (B, S, S), "rgb": (B, 3, IS, IS), "alpha": (B, IS, IS),
              "depth": (B, IS, IS)}
    if host:
        got = {n: b.body().cpu().numpy().view(np.int32 if n == "face_index" else f32).reshape(shapes[n])
               for n, b in o.items()}
    else:
        got = {n: b.body().view(shapes[n]) for n, b in o.items()}

    def backward(grad_rgb, det, off=0):
        g = Buf(grad_rgb.size, IN_F, data=np.asarray(grad_rgb, f32))
        gt = Buf(tex.size, OUT_F, off=off)   # the call zero-fills it
        fn = lib.umr_nmr_backward_textures_deterministic if det else lib.umr_nmr_backward_textures
        rc = fn(ins["vertices"].ptr(), ins["faces"].ptr(), o["face_index"].ptr(), g.ptr(), gt.ptr(), ctypes.byref(p),
                ctypes.c_void_p(ws.data_ptr()), _stream_ptr(DEV))
        _lib.check(rc, "umr_nmr_backward_textures")
        torch.cuda.synchronize()
        g.check("grad_rgb", False)
        o["face_index"].check("face_index", True)
        gt.check("grad_textures", True)
        return gt.body().cpu().numpy().view(f32).reshape(tex.shape)
    return got, backward


def okw(IS, aa=True, fill_back=True, G=1, eye=EYE, near=0.1, far=100.0, bg=(0, 0, 0), **light):
    lt = dict(LIGHT0, **light)
    return dict(image_size=IS, anti_aliasing=aa, fill_back=fill_back, eye_z=eye, near=near, far=far,
                light_intensity_ambient=lt["Ia"], light_intensity_directional=lt["Id"], light_color_ambient=lt["ca"],
                light_color_directional=lt["cd"], light_direction=lt["direction"], background_color=bg,
                shared_textures=G)


_ZB = {}


def reference(key, verts, faces, tex, IS, **kw):
    """oracle.render with the z-buffer cached per (scene key, z-buffer settings)."""
    k = okw(IS, **kw)
    zk = (key, IS, k["anti_aliasing"], k["fill_back"], k["eye_z"], k["near"], k["far"])
    if zk not in _ZB:
        _ZB[zk] = oracle.zbuffer(verts, faces, IS, k["anti_aliasing"], k["fill_back"], k["eye_z"], k["near"], k["far"])
    return oracle.render(verts, faces, tex, zbuf=_ZB[zk], **k)


def assert_planes_equal(got, ref, names=("face_index", "raster_depth", "rgb", "alpha", "depth")):
    for n in names:
        if n not in ref or n not in got:
            continue
        a, b = got[n], ref[n]
        assert a.shape == b.shape, (n, a.shape, b.shape)
        bad = ~((a == b) | (np.isnan(a) & np.isnan(b)) if a.dtype.kind == "f" else (a == b))
        assert not bad.any(), "%s differs at %d of %d elements, first %s: got %r, oracle %r" % (
            n, bad.sum(), bad.size, np.argwhere(bad)[0], a[tuple(np.argwhere(bad)[0])], b[tuple(np.argwhere(bad)[0])])


def textures(B, F, T, seed=0, lo=0.0, hi=1.0):
    return np.random.default_rng(seed).uniform(lo, hi, size=(B, F, T, T, T, 3)).astype(f32)


def check_scene(key, verts, faces, tex, IS, what, count, **kw):
    got, bwd = forward(verts, faces, tex, IS, **kw)
    ref = reference(key, verts, faces, tex, IS, **kw)
    assert_planes_equal(got, ref)
    print("%-44s %s = %d" % (key if isinstance(key, str) else "/".join(map(str, key)), what, count))
    assert count > 0
    return got, ref, bwd


# ---------------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("IS", [1, 2, 3, 5, 63, 65, 127, 129])
@pytest.mark.parametrize("aa", [False, True])
def test_image_sizes(IS, aa):
    """Odd sizes run k_nmr_shade<1>; S = 1, 2 and partial 64x64 bins."""
    verts, faces = sc.mesh(B=2, seed=1, soup=6, scale=1.0)
    tex = textures(2, faces.shape[1], 3, seed=IS)
    got, ref, _ = check_scene(("sizes", IS, aa), verts, faces, tex, IS, "covered raster pixels",
                              int((reference(("sizes", IS, aa), verts, faces, None, IS, aa=aa)["face_index"] >= 0).sum()),
                              aa=aa, bg=(0.2, 0.4, 0.6))
    if IS >= 63:
        assert (got["face_index"] >= faces.shape[1]).any()


def test_misaligned_and_null_outputs():
    """Each output 4 bytes off its alignment (the scalar shading path at is = 64), and every subset of NULL outputs."""
    verts, faces = sc.mesh(B=2, seed=2, soup=6)
    tex = textures(2, faces.shape[1], 4, seed=3)
    for off in ("rgb", "alpha", "depth"):
        check_scene("align64", verts, faces, tex, 64, "misaligned %s, vector path off" % off, 1, offsets=(off,))
    for r in range(4):
        for outs in itertools.combinations(("rgb", "alpha", "depth"), r):
            got, _, _ = check_scene("align64", verts, faces, tex, 64, "outputs %s" % (outs,), 1, outs=outs)
            assert set(got) == {"face_index", "raster_depth"} | set(outs)


@pytest.mark.parametrize("eye", [EYE, -1.0, -100.0])
def test_near_and_far_planes_cut_faces(eye):
    verts, faces = sc.clipped(B=2)
    tex = textures(2, faces.shape[1], 3, seed=4)
    dz = eye - EYE   # keep the scene at the same depths relative to the eye
    verts = verts.copy()
    verts[..., 2] += f32(dz)
    for near, far in ((0.1, 100.0), (4.5, 9.0), (-3.0, 6.0), (7.0, 7.5)):
        st = sc.pixel_stats(verts, faces, 32, True, True, eye, near, far)
        check_scene(("clip", eye, near, far), verts, faces, tex, 32, "pixels clipped (near %d, far %d)"
                    % (st["near"], st["far"]), st["near"] + st["far"], eye=eye, near=near, far=far)
    # some vertex behind the eye plane (z - eye <= 0)
    assert (verts[..., 2] - f32(eye) <= 0).any()


@pytest.mark.parametrize("plane", ["near", "far"])
def test_a_plane_at_the_exact_depth_excludes_it(plane):
    """near (far) set to the exact float depth of many covered pixels: those pixels lose that face."""
    verts, faces = sc.grid(64, n=8, step=6)
    cv, cf = sc.clipped()
    verts, faces = sc.append(verts, faces, cv[0], cf[0])
    ref0 = reference("exact", verts, faces, None, 32)
    vals, cnt = np.unique(ref0["raster_depth"][ref0["face_index"] >= 0], return_counts=True)
    z = float(vals[np.argmax(cnt)])
    at = (ref0["raster_depth"] == f32(z)) & (ref0["face_index"] >= 0)
    kw = dict(near=z, far=100.0) if plane == "near" else dict(near=0.1, far=z)
    got, ref, _ = check_scene(("exact", plane), verts, faces, textures(1, faces.shape[1], 2), 32,
                              "pixels at depth %r excluded" % z, int(at.sum()), **kw)
    assert not ((got["face_index"] == ref0["face_index"]) & at).any()


def test_depth_ties():
    """Exact (zp, face) ties: a flat grid with shared edges through pixel centres, faces duplicated at higher indices
    (as they are and rotated), zero-area faces whose two copies both pass the back-face test."""
    gv, gf = sc.grid(64, n=8, step=6)
    st = sc.pixel_stats(gv, gf, 32, True, True)
    tex = textures(1, gf.shape[1], 3, seed=5)
    check_scene("grid", gv, gf, tex, 32, "tie pixels", st["ties"])
    mv, mf = sc.mesh(B=2, seed=6, soup=8)
    dv, df = sc.duplicates(mv, mf, k=mf.shape[1])
    st = sc.pixel_stats(dv, df, 32, True, True)
    got, _, _ = check_scene("dup", dv, df, textures(2, df.shape[1], 3, seed=6), 32, "tie pixels", st["ties"])
    F0, F = mf.shape[1], df.shape[1]
    fi = got["face_index"]
    assert not ((fi >= 0) & (fi % F >= F0) & (fi % F < 2 * F0)).any()   # an unrotated duplicate never wins its tie
    zv, zf = sc.zero_area(64)
    nz = zf.shape[1]
    zv, zf = sc.append(mv[:1], mf[:1], zv[0], zf[0])
    both = sum(sum(sc.whole_image_copies(zv, zf[:, j:j + 1], True)) == 2 for j in range(F0, F0 + nz))
    assert both >= 5   # the exactly collinear faces: neither copy is culled as back-facing
    check_scene("zero", zv, zf, textures(1, zf.shape[1], 3, seed=7), 32, "zero-area faces with both copies tested", both)


def test_signed_zero_depths():
    """eye_z = +0 and near < 0: depths +0 and -0 meet.  NMR's '<' does not order them, so the lower face index wins,
    with its own zero's sign in the raster depth."""
    v, f = sc.signed_zero()
    st = sc.pixel_stats(v, f, 16, False, False, eye_z=0.0, near=-1.0)
    got, ref, _ = check_scene("signed_zero", v, f, None, 16, "zero-depth tie pixels", st["ties"], aa=False,
                              fill_back=False, eye=0.0, near=-1.0)
    assert np.array_equal(np.signbit(got["raster_depth"]), np.signbit(ref["raster_depth"]))
    assert set(np.unique(got["face_index"])) == {-1, 0, 2}


def _segment_in_view(p, q):
    """Parameters [t0, t1] of the part of p + t (q - p) inside [-1, 1]^2 (Liang-Barsky), or None."""
    t0, t1 = 0.0, 1.0
    d = q - p
    for k in range(2):
        for s, lim in ((-1, -1.0), (1, 1.0)):
            num, den = s * (lim - p[k]), s * d[k]
            if den == 0:
                if num < 0:
                    return None
                continue
            t = num / den
            if den > 0:
                t1 = min(t1, t)
            else:
                t0 = max(t0, t)
    return (t0, t1) if t0 <= t1 else None


def _crops(verts, faces, S, h=16, per_edge=10):
    """Even-aligned raster windows (c0, c1, r0, r1) around every on-screen vertex and along every edge."""
    pts = []
    for tri in verts[0, faces[0]].astype(np.float64):
        for k in range(3):
            p, q = tri[k, :2], tri[(k + 1) % 3, :2]
            seg = _segment_in_view(p, q)
            if seg is None:
                continue
            for t in np.linspace(seg[0], seg[1], per_edge):
                pts.append(p + t * (q - p))
    out = set()
    for x, y in pts:
        cx, cy = 0.5 * (x * S + S - 1), 0.5 * (y * S + S - 1)
        c0 = int(np.clip(np.floor(cx) - h, 0, S - 2 * h)) // 2 * 2
        r0 = int(np.clip(np.floor(cy) - h, 0, S - 2 * h)) // 2 * 2
        out.add((c0, c0 + 2 * h - 1, r0, r0 + 2 * h - 1))
    return sorted(out)


@pytest.mark.parametrize("IS", [256, 2048, 8192])
def test_pixel_box_edges(IS):
    """Faces either side of the sine threshold, coordinates just under 1e6 and at 1e6, vertices on pixel centres, at
    S = 512, 4096 and 16384 (silhouettes and depth), compared on windows around every vertex and along every edge."""
    S = 2 * IS
    v, f = sc.thin(S)
    whole, boxed = sc.whole_image_copies(v, f, True)
    assert whole > 0 and boxed > 0
    if S <= 512:
        check_scene(("thin", S), v, f, None, IS, "whole-image copies (boxed %d)" % boxed, whole)
        return
    got, _ = forward(v, f, None, IS, outs=("alpha", "depth"), host=False)
    crops = _crops(v, f, S)
    for c0, c1, r0, r1 in crops:
        zb = oracle.zbuffer(v, f, IS, True, True, EYE, window=(c0, c1, r0, r1))
        g = {"face_index": got["face_index"][:, r0:r1 + 1, c0:c1 + 1].cpu().numpy(),
             "raster_depth": got["raster_depth"][:, r0:r1 + 1, c0:c1 + 1].cpu().numpy().view(f32)}
        ro0, ro1 = (S - 1 - r1) // 2, (S - 1 - r0) // 2
        g["alpha"] = got["alpha"][:, ro0:ro1 + 1, c0 // 2:c1 // 2 + 1].cpu().numpy().view(f32)
        g["depth"] = got["depth"][:, ro0:ro1 + 1, c0 // 2:c1 // 2 + 1].cpu().numpy().view(f32)
        ref = {"face_index": zb[0], "raster_depth": zb[1],
               "alpha": oracle.flip_pool((zb[0] >= 0).astype(f32)[:, None], True)[:, 0],
               "depth": oracle.flip_pool(zb[1][:, None], True)[:, 0]}
        assert_planes_equal(g, ref)
    print("thin S=%-5d whole-image copies = %d, boxed %d, windows compared = %d" % (S, whole, boxed, len(crops)))


def test_invalid_faces_and_coordinates():
    verts, faces, F0 = sc.invalid(B=2)
    F = faces.shape[1]
    tex = textures(2, F, 3, seed=8)
    got, ref = forward(verts, faces, tex, 32)[0], reference("invalid", verts, faces, tex, 32)
    assert_planes_equal(got, ref)
    clean, _ = forward(verts, faces[:, :F0], tex[:, :F0], 32)
    fi = got["face_index"]
    mapped = np.where(fi >= F, fi - F + F0, fi)                     # back copies renumbered for the clean scene
    drawn = (fi >= 0) & ((fi % F) >= F0)                             # the invalid faces that are drawn (+inf z)
    assert set(np.unique(fi[drawn] % F)) <= {F0 + 7}
    same = ~drawn
    assert np.array_equal(mapped[same], clean["face_index"][same])
    assert np.array_equal(got["raster_depth"][same].view(np.int32), clean["raster_depth"][same].view(np.int32))
    print("invalid: %d faces, %d raster pixels won by the +inf-z face, neighbours unchanged" % (F - F0, drawn.sum()))
    assert drawn.sum() > 0


def test_batch_grid_limit():
    """B = 65535 (the z-buffer's gridDim.z) at is = 1, a different face list and geometry per item (period 7)."""
    B, P = 65535, 7
    rng = np.random.default_rng(9)
    pv = rng.uniform(-1.5, 1.5, size=(P, 6, 3)).astype(f32)
    pv[..., 2] = rng.uniform(3, 6, size=(P, 6))
    pf = np.stack([[np.roll([0, 1, 2], p % 3), rng.permutation([3, 4, 5])] for p in range(P)]).astype(np.int32)
    for aa in (False, True):
        ref = oracle.render(pv, pf, None, **okw(1, aa=aa))
        got, _ = forward(np.tile(pv, (B // P + 1, 1, 1))[:B], np.tile(pf, (B // P + 1, 1, 1))[:B], None, 1, aa=aa)
        idx = np.arange(B) % P
        assert_planes_equal(got, {k: x[idx] for k, x in ref.items()})
        print("B=%d aa=%d: distinct per-item face-index patterns = %d" % (B, aa, len({tuple(r.ravel()) for r in ref["face_index"]})))


def test_per_item_face_lists_and_many_faces():
    # per-item faces and vertex usage
    rng = np.random.default_rng(10)
    v, f = sc.mesh(B=3, seed=10, soup=6)
    f = np.stack([f[b, rng.permutation(f.shape[1])] for b in range(3)])   # each item its own face order
    f[1, :20] = f[1, :20, ::-1]                                             # item 1: some faces turned round
    perm = rng.permutation(v.shape[1])                                      # item 2: its vertices stored permuted
    v[2] = v[2, perm]
    f[2] = np.argsort(perm)[f[2]]
    f[0, -6:] = f[0, :6]                                                    # item 0: repeated faces, unused vertices
    check_scene("per_item", v, f, textures(3, f.shape[1], 3, seed=10), 48, "items with distinct face lists",
                len({f[b].tobytes() for b in range(3)}))
    # F = 70000 with fill_back: Fc = 140000 > 2^17, face indices past 16 bits win
    F = 70000
    c = rng.uniform(-1, 1, size=(F, 2))
    ang = rng.uniform(0, 2 * np.pi, size=(F, 1)) + np.array([0, 2.1, 4.2])
    r = rng.uniform(0.01, 0.05, size=(F, 1))
    xy = c[:, None] + r[..., None] * np.stack([np.cos(ang), np.sin(ang)], -1)
    vv = np.concatenate([xy, rng.uniform(3, 7, size=(F, 3, 1))], -1).reshape(1, 3 * F, 3).astype(f32)
    ff = np.arange(3 * F).reshape(1, F, 3).astype(np.int32)
    ff[0, ::2] = ff[0, ::2, ::-1]   # half back-facing: their copies F + f win
    got, _, _ = check_scene("many", vv, ff, textures(1, F, 2, seed=11), 64, "pixels won by copies >= 65536", 0 + int(
        (reference("many", vv, ff, None, 64)["face_index"] >= 65536).sum()))
    assert (got["face_index"] >= F).any()


@pytest.mark.parametrize("T", [2, 5, 17, 101])
def test_texture_resolutions(T):
    n, step, S = 2, 12, 64
    gv, gf = sc.grid(S, n=n, step=step)   # a handful of faces; vertices on pixel centres sample the clamped texels
    tex = textures(1, gf.shape[1], T, seed=T)
    i0 = (S - n * step) // 2
    ii = i0 + step * np.arange(n + 1)
    fi = reference(("tex", T), gv, gf, None, 32)["face_index"][0]
    check_scene(("tex", T), gv, gf, tex, 32, "vertex pixels (tif at (T-1) - 1e-3)", int((fi[np.ix_(ii, ii)] >= 0).sum()))


LIGHTS = [dict(Ia=0.0, Id=0.7, direction=(0.3, 1, -1)), dict(Ia=0.6, Id=0.0), dict(Ia=0.0, Id=0.0),
          dict(Ia=-0.4, Id=1.5, cd=(2.0, 1.0, 3.0), direction=(3.0, -2.0, 5.0)),
          dict(Ia=1.2, Id=-0.8, ca=(1.5, 0.2, 4.0), direction=(0, 0, -7.0))]


@pytest.mark.parametrize("li", range(len(LIGHTS)))
def test_light_background_and_shared_textures(li):
    """Ia / Id = 0 (the term not added), negative intensities, unnormalised directions, colours > 1, a non-zero
    background pooled at silhouettes, and G = 2 shared textures over different geometry per render."""
    v, f = sc.mesh(B=4, seed=12, soup=6)
    tex = textures(2, f.shape[1], 4, seed=13, lo=-0.5, hi=2.0)
    a = reference(("light", li), v, f, None, 32)["alpha"]
    got, ref, _ = check_scene(("light", li), v, f, tex, 32, "silhouette pixels with background mixed in",
                              int(((a > 0) & (a < 1)).sum()), G=2, bg=(0.3, -0.5, 2.0), **LIGHTS[li])
    assert not np.array_equal(got["rgb"][0::2], got["rgb"][1::2])   # shared texture, different geometry


# ---------------------------------------------------------------------------------------------------------------------
# texture gradient
# ---------------------------------------------------------------------------------------------------------------------
GRAD_CASES = {
    "T2": lambda: (sc.mesh(B=2, seed=20, soup=8), 2, 32, dict()),
    "T101": lambda: (sc.grid(64, n=2, step=12), 101, 32, dict()),
    "is65": lambda: (sc.mesh(B=2, seed=21, soup=8), 3, 65, dict()),
    "G2": lambda: (sc.mesh(B=4, seed=22, soup=8), 3, 32, dict(G=2)),
    "noaa": lambda: (sc.mesh(B=2, seed=23, soup=8), 3, 32, dict(aa=False)),
    "thin": lambda: (_turn_half(*sc.thin(128)), 3, 64, dict()),
    "clipped": lambda: (_turn_half(*sc.clipped(B=2)), 3, 32, dict(near=4.5, far=9.0)),
}


def _turn_half(v, f):
    """Every other face with its vertex order reversed, so that fill_back copies win pixels."""
    f = f.copy()
    f[:, ::2] = f[:, ::2, ::-1]
    return v, f


@pytest.mark.parametrize("name", sorted(GRAD_CASES))
@pytest.mark.parametrize("off", [0, 1])
def test_texture_gradient_within_the_summation_bound(name, off, det):
    (v, f), T, IS, kw = GRAD_CASES[name]()
    G = kw.pop("G", 1)
    B, F = f.shape[:2]
    rng = np.random.default_rng(30 + T)
    tex = textures(B // G, F, T, seed=31)
    light = dict(Ia=0.6, Id=0.5, ca=(1, 0.9, 0.8), cd=(0.5, 1, 1), direction=(0.2, 1, -1))
    got, bwd = forward(v, f, tex, IS, **kw, **light)
    ref = reference(("grad", name), v, f, tex, IS, G=G, **kw, **light)
    assert_planes_equal(got, ref)
    g = rng.normal(size=(B, 3, IS, IS)).astype(f32)
    g[:, :, ::3] = 0.0                                   # exact zeros on some pixels
    g[:, 1, 1::3] = 0.0
    gk = bwd(g, det, off)
    zb = (got["face_index"], got["raster_depth"])
    aa = kw.get("aa", True)
    gr, mag, n = oracle.grad_textures(g, v, f, tex.shape, zb, anti_aliasing=aa, fill_back=True, eye_z=EYE,
                                      shared_textures=G, magnitude=True, counts=True, **light)
    k = (n + 2)[..., None].astype(np.float64)
    bound = k * U / (1 - k * U) * mag
    err = np.abs(gk.astype(np.float64) - gr)
    ratio = float((err / np.maximum(bound, 1e-300)).max())
    print("grad %-8s off=%d %-13s max err/bound = %.3e (max n %d)" % (name, off, "deterministic" if det else "default",
                                                                      ratio, n.max()))
    assert np.isfinite(gk).all()
    assert (err <= bound).all(), "%d texels outside the bound, worst ratio %.3g" % ((err > bound).sum(), ratio)
    assert (mag > 0).any()
    if n.max() > 1:
        assert ((mag > 0) & (np.abs(gr) < 0.5 * mag)).any()   # mixed signs cancel somewhere
    if name not in ("T101",):
        assert (zb[0] >= F).any() and np.abs(gr[:, np.unique(zb[0][zb[0] >= F] - F) % F]).max() > 0   # back copies
    if det:
        assert np.array_equal(gk.view(np.int32), bwd(g, det, off).view(np.int32))


# ---------------------------------------------------------------------------------------------------------------------
# module level
# ---------------------------------------------------------------------------------------------------------------------
def test_renderer_module_against_the_oracle():
    from umr_b200.neural_renderer import Renderer
    v, f = sc.mesh(B=2, seed=40, soup=6)
    T, IS = 3, 32
    tex = textures(2, f.shape[1], T, seed=41)
    light = dict(light_intensity_ambient=0.7, light_intensity_directional=0.3, light_direction=[0.5, 1, -1],
                 light_color_ambient=[1, 0.8, 0.6], light_color_directional=[0.9, 1, 1.2])
    r = Renderer(image_size=IS, anti_aliasing=True, camera_mode="look_at", perspective=False,
                 background_color=[0.1, 0.2, 0.3], **light)
    r.eye = [0, 0, EYE]
    vt, ft, tt = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV), torch.from_numpy(tex).to(DEV)
    ref = oracle.render(v, f, tex, image_size=IS, anti_aliasing=True, fill_back=True, eye_z=EYE, near=0.1, far=100.0,
                        light_intensity_ambient=0.7, light_intensity_directional=0.3, light_color_ambient=(1, 0.8, 0.6),
                        light_color_directional=(0.9, 1, 1.2), light_direction=(0.5, 1, -1),
                        background_color=(0.1, 0.2, 0.3))
    with torch.no_grad():
        rgb, depth, alpha = r.render(vt, ft, tt)
        outs = {"rgb": rgb, "depth": depth, "alpha": alpha, "d": r.render_depth(vt, ft), "s": r.render_silhouettes(vt, ft),
                "m_rgb": r(vt, ft, tt, mode="rgb"), "m_s": r(vt, ft, mode="silhouettes"), "m_d": r(vt, ft, mode="depth")}
        m_rgb, m_depth, m_alpha = r(vt, ft, tt)
    outs = {k: x.cpu().numpy() for k, x in outs.items()}
    assert_planes_equal({"rgb": outs["rgb"], "depth": outs["depth"], "alpha": outs["alpha"]}, ref)
    for a, b in (("d", "depth"), ("m_d", "depth"), ("s", "alpha"), ("m_s", "alpha"), ("m_rgb", "rgb")):
        assert_planes_equal({b: outs[a]}, ref, names=(b,))
    assert_planes_equal({"rgb": m_rgb.cpu().numpy(), "depth": m_depth.cpu().numpy(), "alpha": m_alpha.cpu().numpy()}, ref)
    # float64 textures render in float32 and get a float64 gradient
    t64 = torch.from_numpy(tex.astype(np.float64)).to(DEV).requires_grad_(True)
    img = r.render_rgb(vt, ft, t64)
    assert img.dtype == torch.float32
    assert np.array_equal(img.detach().cpu().numpy(), ref["rgb"])
    g = np.random.default_rng(42).normal(size=img.shape).astype(f32)
    img.backward(torch.from_numpy(g).to(DEV))
    assert t64.grad.dtype == torch.float64
    gr = oracle.grad_textures(g, v, f, tex.shape, (ref["face_index"], ref["raster_depth"]), anti_aliasing=True,
                              fill_back=True, eye_z=EYE, Ia=0.7, Id=0.3, ca=(1, 0.8, 0.6), cd=(0.9, 1, 1.2),
                              direction=(0.5, 1, -1))
    assert np.abs(gr).max() > 0 and np.allclose(t64.grad.cpu().numpy(), gr, rtol=1e-4, atol=1e-5 * np.abs(gr).max())
