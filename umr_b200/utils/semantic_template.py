"""The SCOPS semantic template of `experiments/avg_uv.py::compute_uv` (:203-293) on the GPU.

Between its two training stages UMR averages, over the dataset, the SCOPS part probabilities of the k images per batch
nearest an exemplar in UV space, then labels every texel, face and vertex of the template with the part it most often
shows.  `train_s2`'s `part_matching_loss` reads the label image (`semantic_seg.png`) and `CorrLossChamfer` the vertex
lists (`vertices_idx/*_vertices.npy`).  Here the averaging pass is `UVPartAverage` (two kernel launches per batch, no
host synchronisation) and the labelling pass `semantic_template` (three launches and one host synchronisation to size the
part lists); `save_semantic_template` writes the files where those losses read them.  Kernels: csrc/semantic_template.cu;
contract, tie rules and deviations from the reference: DESIGN.md §18.
"""
import ctypes
import math
import os
from collections import namedtuple

import numpy as np
import torch

from .. import _lib, ops
from ..nnutils import loss_utils
from ..raster import _ptr, _stream_ptr

MAX_IMAGES = 1024      # UMR_ST_MAX_IMAGES
MAX_CHANNELS = 32      # UMR_ST_MAX_CHANNELS
PART_NAMES = ("head", "neck", "back", "belly")   # labels 1..4 (avg_uv.py:290-293)

SemanticTemplate = namedtuple("SemanticTemplate", ["label_image", "texel_labels", "face_labels", "vertex_labels",
                                                   "part_vertices", "stex_one_hot"])
SemanticTemplate.__doc__ = """The labelling pass's outputs, all on the input's device.
label_image [H,W] uint8: argmax over channels of avg_prob (`semantic_seg.png`);
texel_labels [F,T2], face_labels [F], vertex_labels [V] int32 (-1: a vertex no face uses);
part_vertices: for each label 1..C-1, the ascending int64 indices of the vertices with that label;
stex_one_hot [1,F,T2,C] float32: what part_matching_loss builds from the label image."""


def _cuda_float(name, t, dim):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TypeError("%s must be a CUDA tensor" % name)
    if t.dtype != torch.float32:
        raise TypeError("%s must be float32, got %s" % (name, t.dtype))
    if t.dim() != dim:
        raise ValueError("%s must have %d dimensions, got shape %s" % (name, dim, tuple(t.shape)))
    return t.detach().contiguous()


def _same_device(**ts):
    if len({t.device for t in ts.values()}) > 1:
        raise ValueError("%s must be on one device, got %s" % (", ".join(ts), ", ".join(str(t.device) for t in ts.values())))


class UVPartAverage(object):
    """The averaging pass (avg_uv.py:203-236): for every batch, the k images whose UV part maps are nearest the
    exemplar's, summed into a dataset-wide accumulator.

    exemplar_uv [C,H,W] float32 CUDA: the exemplar's part probabilities in UV space (`best_uv`, which the caller forms,
    e.g. with ops.bilinear_sample).  1 <= k <= 1024 and C <= 32."""

    def __init__(self, exemplar_uv, k=5):
        self.exemplar = _cuda_float("exemplar_uv", exemplar_uv, 3)
        if isinstance(k, bool) or int(k) != k or not 1 <= k <= MAX_IMAGES:
            raise ValueError("k must be an integer in [1, %d], got %r" % (MAX_IMAGES, k))
        C, H, W = self.exemplar.shape
        if not 1 <= C <= MAX_CHANNELS:
            raise ValueError("exemplar_uv must have 1 to %d channels, got %d" % (MAX_CHANNELS, C))
        self.k = int(k)
        self.acc = torch.zeros_like(self.exemplar)
        self.count = 0

    def add(self, part_segs, uvimage_pred):
        """One batch: part_segs [B,C,S,S] SCOPS probabilities and uvimage_pred [B,2,H,W] the texture-flow UV image,
        float32 on the exemplar's device, k <= B <= 1024.  uv_parts[b] = grid_sample(part_segs[b], uvimage_pred[b])
        (align_corners=True, zeros padding) is never materialised: dist[b] = sum (uv_parts[b] - exemplar)^2, the k
        images first in (dist, index) order are selected, NaN distances last, and their maps, summed in selection
        order, are added to the accumulator.  Two kernel launches, no host synchronisation (CUDA-graph capturable).
        Returns the device tensors (dist [B] float32, selected [k] int32)."""
        segs = _cuda_float("part_segs", part_segs, 4)
        uv = _cuda_float("uvimage_pred", uvimage_pred, 4)
        _same_device(exemplar_uv=self.exemplar, part_segs=segs, uvimage_pred=uv)
        C, H, W = self.exemplar.shape
        B, Cs, S, S2 = segs.shape
        if Cs != C or S != S2:
            raise ValueError("part_segs must be [B,%d,S,S], got %s" % (C, tuple(segs.shape)))
        if tuple(uv.shape) != (B, 2, H, W):
            raise ValueError("uvimage_pred must be [%d,2,%d,%d], got %s" % (B, H, W, tuple(uv.shape)))
        if not self.k <= B <= MAX_IMAGES:
            raise ValueError("part_segs must hold k = %d to %d images, got %d" % (self.k, MAX_IMAGES, B))
        lib = _lib.load()
        dev = segs.device
        with torch.cuda.device(dev):
            ws = torch.empty(lib.umr_st_average_workspace_bytes(B, H, W) // 4, device=dev, dtype=torch.float32)
            dist = torch.empty(B, device=dev, dtype=torch.float32)
            selected = torch.empty(self.k, device=dev, dtype=torch.int32)
            _lib.check(lib.umr_st_average_add(_ptr(segs), _ptr(uv), _ptr(self.exemplar), B, C, S, H, W, self.k, _ptr(ws),
                                              _ptr(dist), _ptr(selected), _ptr(self.acc), _stream_ptr(dev)),
                       "umr_st_average_add")
        self.count += self.k
        return dist, selected

    def mean(self):
        """avg_prob [H,W,C] float32 = accumulator / (number of images added), one IEEE division per element
        (avg_uv.py:227-230).  One kernel launch."""
        if self.count == 0:
            raise ValueError("UVPartAverage.mean: no batch has been added")
        C, H, W = self.acc.shape
        dev = self.acc.device
        with torch.cuda.device(dev):
            avg = torch.empty(H, W, C, device=dev, dtype=torch.float32)
            _lib.check(_lib.load().umr_st_average_mean(_ptr(self.acc), C, H, W, self.count, _ptr(avg), _stream_ptr(dev)),
                       "umr_st_average_mean")
        return avg


def semantic_template(avg_prob, uv_sampler, faces, num_sym_faces, num_vertices=None):
    """The labelling pass (avg_uv.py:254-293).

    avg_prob [H,W,C] float32 and uv_sampler [1,F',T2,2] float32 (the model's `uv_sampler[0].unsqueeze(0)`, T2 = tex_size^2)
    are CUDA tensors, faces [F,3] an integer CUDA tensor with F = F' + num_sym_faces, 1 <= num_sym_faces <= F'.  The
    faces past F' take the samples of the last num_sym_faces ones, as the reference appends them.  num_vertices defaults
    to faces.max() + 1, the reference's vertex range (one more host synchronisation).

    A texel's label is the argmax over channels of avg_prob sampled at it (the first NaN, else the first largest), a
    face's the most frequent of its texels', a vertex's the most frequent of its faces' (ties to the smallest label; a
    vertex no face uses gets -1 and no part).  Returns a SemanticTemplate; part_vertices[p - 1] holds the vertices of
    label p.  Three kernel launches and one host synchronisation, to size the part lists."""
    prob = _cuda_float("avg_prob", avg_prob, 3)
    sampler = _cuda_float("uv_sampler", uv_sampler, 4)
    if not isinstance(faces, torch.Tensor) or not faces.is_cuda:
        raise TypeError("faces must be a CUDA tensor")
    if faces.dtype not in (torch.int32, torch.int64):
        raise TypeError("faces must be int32 or int64, got %s" % faces.dtype)
    _same_device(avg_prob=prob, uv_sampler=sampler, faces=faces)
    H, W, C = prob.shape
    if not 1 <= C <= MAX_CHANNELS:
        raise ValueError("avg_prob must have 1 to %d channels, got %d" % (MAX_CHANNELS, C))
    if sampler.shape[0] != 1 or sampler.shape[3] != 2:
        raise ValueError("uv_sampler must be [1,F',T2,2], got %s" % (tuple(sampler.shape),))
    F_src, T2 = sampler.shape[1:3]
    T = math.isqrt(T2)
    if T * T != T2:
        raise ValueError("uv_sampler must hold tex_size^2 points per face, got %d" % T2)
    if isinstance(num_sym_faces, bool) or int(num_sym_faces) != num_sym_faces or not 1 <= num_sym_faces <= F_src:
        raise ValueError("num_sym_faces must be an integer in [1, %d], got %r" % (F_src, num_sym_faces))
    num_sym_faces = int(num_sym_faces)
    F = F_src + num_sym_faces
    if faces.dim() != 2 or tuple(faces.shape) != (F, 3):
        raise ValueError("faces must be [%d,3] (F' + num_sym_faces), got %s" % (F, tuple(faces.shape)))
    if num_vertices is None:
        num_vertices = int(faces.max()) + 1
    elif isinstance(num_vertices, bool) or int(num_vertices) != num_vertices or num_vertices < 1:
        raise ValueError("num_vertices must be a positive integer, got %r" % (num_vertices,))
    V = int(num_vertices)
    dev = prob.device
    with torch.cuda.device(dev):
        rowptr, corners = ops.device_incidence(faces, V)
        label_image = torch.empty(H, W, device=dev, dtype=torch.uint8)
        texel_labels = torch.empty(F, T2, device=dev, dtype=torch.int32)
        face_labels = torch.empty(F, device=dev, dtype=torch.int32)
        vertex_labels = torch.empty(V, device=dev, dtype=torch.int32)
        _lib.check(_lib.load().umr_st_labels(_ptr(prob), H, W, C, _ptr(sampler), F_src, T2, num_sym_faces, _ptr(rowptr),
                                             _ptr(corners), V, _ptr(label_image), _ptr(texel_labels), _ptr(face_labels),
                                             _ptr(vertex_labels), _stream_ptr(dev)),
                   "umr_st_labels")
        # one stable grouping of the vertex labels (-1 drops out past the last row), and the face range read with it
        part_ptr, by_label = ops.device_incidence(vertex_labels, C)
        lo, hi = torch.aminmax(faces)
        sizes = torch.cat([part_ptr.long(), lo.long().view(1), hi.long().view(1)]).tolist()   # the host synchronisation
    if sizes[-2] < 0 or sizes[-1] >= V:
        raise ValueError("faces must index vertices in [0, %d), got [%d, %d]" % (V, sizes[-2], sizes[-1]))
    part_vertices = [by_label[sizes[p]:sizes[p + 1]].long() for p in range(1, C)]
    stex_one_hot = loss_utils.label_image_one_hot(label_image.float().view(1, 1, H, W), sampler, num_sym_faces, T, C)
    return SemanticTemplate(label_image, texel_labels, face_labels, vertex_labels, part_vertices, stex_one_hot)


def save_semantic_template(directory, avg_prob, template):
    """Write a 5-channel template where train_s2's losses read it: `semantic_prob.npy` (avg_prob [H,W,C] float32) and
    `semantic_seg.png` (the label image) in `directory`, and `vertices_idx/{head,neck,back,belly}_vertices.npy` (int64)
    below it -- the layout `part_matching_loss(scops_path)` and `CorrLossChamfer(scops_path)` open.  The reference writes
    the four vertex lists flat into its output directory (avg_uv.py:290-293) and leaves the move to the user."""
    from PIL import Image
    if len(template.part_vertices) != len(PART_NAMES):
        raise ValueError("save_semantic_template writes the %d SCOPS parts %s, got %d part lists"
                         % (len(PART_NAMES), PART_NAMES, len(template.part_vertices)))
    os.makedirs(os.path.join(directory, "vertices_idx"), exist_ok=True)
    np.save(os.path.join(directory, "semantic_prob.npy"), avg_prob.detach().float().cpu().numpy())
    Image.fromarray(template.label_image.cpu().numpy()).save(os.path.join(directory, "semantic_seg.png"), "PNG")
    for name, verts in zip(PART_NAMES, template.part_vertices):
        np.save(os.path.join(directory, "vertices_idx", "%s_vertices.npy" % name), verts.cpu().numpy().astype(np.int64))
