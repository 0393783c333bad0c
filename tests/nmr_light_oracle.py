"""numpy float64 restatement of `neural_renderer.lighting` (DESIGN.md §15), forward and every gradient, with a
first-order running error bound for the kernel's precision.

Each value is an `E`: the float64 value `v` and a bound `e` on how far a computation with unit roundoff `u` (2^-24 for
the float32 kernels, 2^-53 for the float64 ones) that performs the kernels' operations, one rounding each, can land
from it.  Inputs are exact (the kernels read the same numbers).  Sums whose order is not the oracle's are bounded with
gamma_{n-1} * sum|term|, whatever the order.  `ambiguous` marks the faces whose relu or eps branch could go either way
within that bound; tests keep those out of random scenes and build the exact cases on purpose.
"""
import numpy as np

EPS = 1e-5
U32, U64 = 2.0 ** -24, 2.0 ** -53


def eps_for(u):
    """normalize's eps as the kernel holds it: 1e-5f in float32."""
    return float(np.float32(EPS)) if u == U32 else EPS


class E:
    __slots__ = ("v", "e", "u")

    def __init__(self, v, e=None, u=U32):
        self.v = np.asarray(v, np.float64)
        self.e = np.zeros_like(self.v) if e is None else np.asarray(e, np.float64)
        self.u = u

    def _w(self, o):
        return o if isinstance(o, E) else E(o, u=self.u)

    def __add__(self, o):
        o = self._w(o)
        v = self.v + o.v
        return E(v, self.e + o.e + self.u * np.abs(v), self.u)

    def __sub__(self, o):
        o = self._w(o)
        v = self.v - o.v
        return E(v, self.e + o.e + self.u * np.abs(v), self.u)

    def __neg__(self):
        return E(-self.v, self.e, self.u)

    def __mul__(self, o):
        o = self._w(o)
        v = self.v * o.v
        with np.errstate(invalid="ignore"):
            e = np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e + self.u * np.abs(v)
        return E(v, e, self.u)

    def __truediv__(self, o):
        o = self._w(o)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = self.v / o.v
            lo = np.abs(o.v) - o.e
            e = np.where(lo > 0, (self.e + np.abs(v) * o.e) / np.where(lo > 0, lo, 1), np.inf) + self.u * np.abs(v)
        return E(v, e, self.u)

    def __getitem__(self, k):
        return E(self.v[k], self.e[k], self.u)


def sqrt(x):
    with np.errstate(invalid="ignore", divide="ignore"):
        v = np.sqrt(x.v)
        lo = np.sqrt(np.maximum(x.v - x.e, 0))
        e = np.where(x.e > 0, x.e / (v + lo), 0) + x.u * v
    return E(v, e, x.u)


def maximum(x, c):
    """fmax(x, c), c exact: a NaN x gives c, as the kernels' fmax does.  1-Lipschitz, and exact when x cannot exceed
    c."""
    v = np.fmax(x.v, c)
    return E(v, np.where(x.v + x.e <= c, 0, x.e), x.u)


def relu(x):
    with np.errstate(invalid="ignore"):
        v = np.where(x.v < 0, 0.0, x.v)  # NaN stays NaN
        e = np.where(x.v + x.e <= 0, 0, x.e)
    return E(v, e, x.u)


def esum(x, axis):
    """Sum in any order: sum of the terms' bounds plus gamma_{n-1} * sum|term|."""
    n = x.v.shape[axis]
    g = (n - 1) * x.u / (1 - (n - 1) * x.u)
    return E(x.v.sum(axis), x.e.sum(axis) + g * np.abs(x.v).sum(axis), x.u)


def stack(xs, axis):
    return E(np.stack([x.v for x in xs], axis), np.stack([x.e for x in xs], axis), xs[0].u)


def intensity(x, u):
    """An intensity as the kernel holds it: the float32 kernels round it to float."""
    x = float(x)
    return E(x, abs(x - float(np.float32(x))) if u == U32 else 0.0, u)


def _vec(x, B):
    x = np.asarray(x, np.float64)
    return np.broadcast_to(x, (B, 3)) if x.ndim == 1 else x


def light(faces, Ia, Id, ca, cd, direction, u=U32):
    """faces [B,F,3,3] -> dict: light [B,F,3] and the intermediates the gradients chain through (all E)."""
    faces = np.asarray(faces, np.float64)
    B, F = faces.shape[:2]
    v = [[E(faces[:, :, k, d], u=u) for d in range(3)] for k in range(3)]
    ca, cd, dr = (_vec(x, B)[:, None, :] for x in (ca, cd, direction))
    Iae, Ide = intensity(Ia, u), intensity(Id, u)
    d = [E(np.broadcast_to(dr[..., k], (B, F)), u=u) for k in range(3)]
    a = [v[0][k] - v[1][k] for k in range(3)]
    b = [v[2][k] - v[1][k] for k in range(3)]
    c = [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]
    nrm = sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2])
    den = maximum(nrm, eps_for(u))
    n = [ck / den for ck in c]
    nd = (n[0] * d[0] + n[1] * d[1]) + n[2] * d[2]
    cs = relu(nd)
    ls = []
    for ch in range(3):
        lc = E(np.zeros((B, F)), u=u)
        if Ia != 0:
            lc = lc + E(np.broadcast_to(ca[..., ch], (B, F)), u=u) * Iae
        if Id != 0:
            lc = lc + (E(np.broadcast_to(cd[..., ch], (B, F)), u=u) * cs) * Ide
        ls.append(lc)
    with np.errstate(invalid="ignore"):
        amb = (np.abs(nd.v) <= nd.e) & ~((nd.v == 0) & (nd.e == 0))          # relu's side not certain
        amb |= (np.abs(nrm.v - eps_for(u)) <= nrm.e)                              # eps branch not certain
    return {"light": stack(ls, 2), "a": a, "b": b, "nrm": nrm, "den": den, "n": n, "d": d, "cs": cs, "nd": nd,
            "cd": E(np.broadcast_to(cd, (B, F, 3)), u=u), "ambiguous": amb & (Id != 0)}


def forward(faces, textures, Ia=0.5, Id=0.5, ca=(1, 1, 1), cd=(1, 1, 1), direction=(0, 1, 0), u=U32):
    """lit textures [B,F,T,T,T,3] (E) and the light's parts."""
    L = light(faces, Ia, Id, ca, cd, direction, u)
    tex = E(np.asarray(textures, np.float64), u=u)
    lv = L["light"]
    return tex * E(lv.v[:, :, None, None, None, :], lv.e[:, :, None, None, None, :], u), L


def backward(faces, textures, g, Ia=0.5, Id=0.5, ca=(1, 1, 1), cd=(1, 1, 1), direction=(0, 1, 0), u=U32):
    """-> dict of E: grad_textures [B,F,T,T,T,3], grad_faces [B,F,3,3], and per image [B,3] grad_ca, grad_cd, grad_dir
    (sum them over the batch for a [3] argument)."""
    faces = np.asarray(faces, np.float64)
    B, F = faces.shape[:2]
    L = light(faces, Ia, Id, ca, cd, direction, u)
    tex = np.asarray(textures, np.float64).reshape(B, F, -1, 3)
    gg = np.asarray(g, np.float64).reshape(B, F, -1, 3)
    lv = L["light"]
    gt = E(gg, u=u) * E(lv.v[:, :, None, :], lv.e[:, :, None, :], u)
    s = esum(E(tex, u=u) * E(gg, u=u), 2)                     # [B,F,3]
    zero = E(np.zeros((B, F)), u=u)
    Iae, Ide = intensity(Ia, u), intensity(Id, u)
    gca = [s[..., c] * Iae if Ia != 0 else zero for c in range(3)]
    if Id != 0:
        gcd = [(s[..., c] * Ide) * L["cs"] for c in range(3)]
        gcs = zero
        for c in range(3):
            gcs = gcs + (s[..., c] * Ide) * L["cd"][..., c]
        with np.errstate(invalid="ignore"):
            keep = ~(L["cs"].v <= 0)                                   # relu passes where its output is not <= 0
        gnd = E(np.where(keep, gcs.v, 0), np.where(keep, gcs.e, 0), u)
        n, d = L["n"], L["d"]
        gdir = [gnd * n[k] for k in range(3)]
        gn = [gnd * d[k] for k in range(3)]
        t = (gn[0] * n[0] + gn[1] * n[1]) + gn[2] * n[2]
        with np.errstate(invalid="ignore"):
            pas = L["nrm"].v >= eps_for(u)
        gc = []
        for k in range(3):
            full = (gn[k] - t * n[k]) / L["den"]
            part = gn[k] / L["den"]
            gc.append(E(np.where(pas, full.v, part.v), np.where(pas, full.e, part.e), u))
        a, b = L["a"], L["b"]
        ga = [b[1] * gc[2] - b[2] * gc[1], b[2] * gc[0] - b[0] * gc[2], b[0] * gc[1] - b[1] * gc[0]]
        gb = [gc[1] * a[2] - gc[2] * a[1], gc[2] * a[0] - gc[0] * a[2], gc[0] * a[1] - gc[1] * a[0]]
        gv = [ga, [-ga[k] - gb[k] for k in range(3)], gb]
        gfaces = stack([stack(gv[j], 2) for j in range(3)], 2)
    else:
        gcd = [zero] * 3
        gdir = [zero] * 3
        gfaces = E(np.zeros((B, F, 3, 3)), u=u)
    per_face = lambda xs: esum(stack(xs, 2), 1)  # noqa: E731  [B,F,3] -> [B,3], faces summed
    return {"grad_textures": E(gt.v.reshape(np.shape(textures)), gt.e.reshape(np.shape(textures)), u),
            "grad_faces": gfaces, "grad_ca": per_face(gca), "grad_cd": per_face(gcd), "grad_dir": per_face(gdir),
            "ambiguous": L["ambiguous"]}


def batch_sum(x):
    """[B,3] -> [3]: the gradient of a [3] argument that lights every image."""
    return esum(x, 0)
