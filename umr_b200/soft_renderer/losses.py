"""Mesh regularisers UMR takes from SoftRas (reference: SoftRas/losses.py:6-114; call sites
experiments/train_s2.py:138-139, :220-221).  CUDA inputs run hand-written kernels (csrc/mesh_ops.cu, SURVEY.md §8f-4):
the Laplacian is a CSR neighbour gather instead of the reference's dense V x V matmul, the flatten loss one fused
kernel per direction instead of ~40 elementwise launches.  CPU inputs evaluate the reference's formulas in torch."""
import numpy as np
import torch
import torch.nn as nn


class LaplacianLoss(nn.Module):
    """|L x|^2 with the row-normalised graph Laplacian of the template (losses.py:6-37)."""

    def __init__(self, vertex, faces, average=False):
        super().__init__()
        self.nv = vertex.size(0)
        self.nf = faces.size(0)
        self.average = average
        f = faces.detach().cpu().numpy().astype(np.int64)
        lap = np.zeros((self.nv, self.nv), dtype=np.float32)
        for a, b in ((0, 1), (1, 2), (2, 0)):
            lap[f[:, a], f[:, b]] = -1
            lap[f[:, b], f[:, a]] = -1
        idx = np.arange(self.nv)
        lap[idx, idx] = -lap.sum(1)
        lap = lap / lap[idx, idx][:, None]
        self.register_buffer("laplacian", torch.from_numpy(lap))
        # CSR of the off-diagonal entries (values exactly as in the dense matrix) + the transposed entries for backward
        off = lap.copy()
        off[idx, idx] = 0
        rows, cols = np.nonzero(off)
        rowptr = np.zeros(self.nv + 1, np.int32)
        np.add.at(rowptr, rows + 1, 1)
        self.register_buffer("csr_rowptr", torch.from_numpy(np.cumsum(rowptr).astype(np.int32)))
        self.register_buffer("csr_col", torch.from_numpy(cols.astype(np.int32)))
        self.register_buffer("csr_coef", torch.from_numpy(off[rows, cols].astype(np.float32)))
        self.register_buffer("csr_tcoef", torch.from_numpy(off[cols, rows].astype(np.float32)))

    def forward(self, x):
        batch_size = x.size(0)
        if x.is_cuda and x.dim() == 3 and x.size(-1) == 3:
            from .. import ops
            loss = ops.LaplacianFunction.apply(x, self.csr_rowptr, self.csr_col, self.csr_coef, self.csr_tcoef)
            return loss.sum() / batch_size if self.average else loss
        x = torch.matmul(self.laplacian, x)
        x = x.pow(2).sum(tuple(range(1, x.dim())))
        return x.sum() / batch_size if self.average else x


class FlattenLoss(nn.Module):
    """sum over edges of (cos(dihedral) + 1)^2 (losses.py:39-114).  The edge table (v0, v1 = edge,
    v2 / v3 = the opposite corners of its two triangles) is built with a dictionary instead of the
    reference's O(E*F) scan; the loss is symmetric in v2 <-> v3 so the result is the same."""

    def __init__(self, faces, average=False):
        super().__init__()
        self.nf = faces.size(0)
        self.average = average
        f = faces.detach().cpu().numpy().astype(np.int64)
        opp = {}
        for tri in f:
            for k in range(3):
                a, b, c = int(tri[k]), int(tri[(k + 1) % 3]), int(tri[(k + 2) % 3])
                opp.setdefault((min(a, b), max(a, b)), []).append(c)
        edges = sorted(e for e, o in opp.items() if len(o) >= 2)
        v0 = [e[0] for e in edges]
        v1 = [e[1] for e in edges]
        v2 = [opp[e][0] for e in edges]
        v3 = [opp[e][1] for e in edges]
        for name, v in (("v0s", v0), ("v1s", v1), ("v2s", v2), ("v3s", v3)):
            self.register_buffer(name, torch.tensor(v, dtype=torch.long))
        self.register_buffer("edge_table", torch.tensor(list(zip(v0, v1, v2, v3)), dtype=torch.int32).reshape(-1, 4))
        # the edge table transposed (vertex -> ascending edge * 4 + role), for the deterministic backward's per-vertex
        # gather under torch.use_deterministic_algorithms(True); not part of the state dict
        from ..ops import vertex_incidence
        rowptr, inc = vertex_incidence(self.edge_table.numpy(), int(f.max()) + 1 if f.size else 0)
        self.register_buffer("vert_rowptr", torch.from_numpy(rowptr), persistent=False)
        self.register_buffer("vert_incidence", torch.from_numpy(inc), persistent=False)

    @staticmethod
    def _perp(a, b, eps):
        """Length-scaled component of b perpendicular to a, and its length estimate."""
        al2 = a.pow(2).sum(-1)
        bl2 = b.pow(2).sum(-1)
        al1 = (al2 + eps).sqrt()
        bl1 = (bl2 + eps).sqrt()
        ab = (a * b).sum(-1)
        cos = ab / (al1 * bl1 + eps)
        sin = (1 - cos.pow(2) + eps).sqrt()
        c = a * (ab / (al2 + eps))[:, :, None]
        return b - c, bl1 * sin

    def forward(self, vertices, eps=1e-6):
        batch_size = vertices.size(0)
        if vertices.is_cuda and vertices.dim() == 3:
            from .. import ops
            loss = ops.FlattenFunction.apply(vertices, self.edge_table, eps, self.vert_rowptr, self.vert_incidence)
            return loss.sum() / batch_size if self.average else loss
        p0, p1 = vertices[:, self.v0s, :], vertices[:, self.v1s, :]
        p2, p3 = vertices[:, self.v2s, :], vertices[:, self.v3s, :]
        cb1, l1 = self._perp(p1 - p0, p2 - p0, eps)
        cb2, l2 = self._perp(p1 - p0, p3 - p0, eps)
        cos = (cb1 * cb2).sum(-1) / (l1 * l2 + eps)
        loss = (cos + 1).pow(2).sum(tuple(range(1, cos.dim())))
        return loss.sum() / batch_size if self.average else loss
