"""Geometric losses of the reference's nnutils/loss_utils.py on the H100 kernels.

Same names and call signatures as the reference (file:line cited per item).  Differences, all
host-side:
* no files are read in constructors: `CorrLossChamfer` and `part_matching_loss` take the data the
  reference loads from `scops_path` (`vertices_idx/*.npy`, `semantic_seg.png`) as optional tensors,
  falling back to the reference's file layout when a path is given;
* the perceptual (LPIPS) branch of `MultiTextureLoss` is outside the hot path (a dense CNN with
  downloaded weights): `PerceptualTextureLoss` delegates to the REFERENCE's own `perceptual_loss`
  module (reachable under `umr_b200.compat.overlay`) and raises loudly when it is not importable --
  the default stays "perceptual" like the reference (loss_utils.py:279), so the objective never
  changes silently; pass `texture_loss_type="l1"` for the reference's L1 alternative (:289-292);
* `TexCycle` builds its visibility mask with a bitmap kernel instead of a per-sample
  `torch.unique` + host sync (loss_utils.py:174-179).
"""
import os.path as osp

import numpy as np
import torch
import torch.nn as nn

from .. import ops
from . import geom_utils
from .chamfer_python import distChamfer
from .smr import SoftRenderer


# ---------------------------------------------------------------------------------------------
# elementwise / reduction losses
# ---------------------------------------------------------------------------------------------
def neg_iou_loss(predict, target, avg=True):
    """loss_utils.py:41-48.  One fused reduction kernel per call (+ fused backward)."""
    per_image = ops.neg_iou_per_image(predict, target)  # 1 - I/U per image
    if avg:
        # reference: 1 - (I/U).sum() / B  ==  mean(1 - I/U)
        return per_image.sum() / per_image.nelement()
    return per_image


def texture_dt_loss(texture_flow, dist_transf, vis_rend=None, cams=None, verts=None, tex_pred=None):
    """loss_utils.py:50-90: mean of the distance-transform map sampled at the texture-flow
    coordinates (visualisation branch :66-88 not provided)."""
    B, nf, T = texture_flow.size(0), texture_flow.size(1), texture_flow.size(-2)
    d = ops.bilinear_sample(dist_transf, texture_flow.reshape(B, nf * T * T, 2))
    return d.mean()


def texture_loss(img_pred, img_gt, mask_gt):
    """loss_utils.py:93-101."""
    mask_gt = mask_gt.unsqueeze(1)
    return torch.nn.L1Loss()(img_pred * mask_gt, img_gt * mask_gt)


def texture_loss_masks(img_pred, img_gt, mask_gt, mask_pred, avg=True):
    """loss_utils.py:103-116.  CUDA tensors: one fused reduction kernel (+ fused backward) that reads
    the RGB / alpha planes of the render in place; anything else: the reference's torch expression."""
    if img_pred.is_cuda and img_pred.dim() == 4 and img_pred.size(1) in (1, 3):
        per_image = ops.masked_l1_per_image(img_pred, img_gt, mask_gt, mask_pred)
        return per_image.mean() if avg else per_image  # equal image sizes: mean of means == global mean
    mask_gt = mask_gt.unsqueeze(1)
    mask_pred = mask_pred.unsqueeze(1)
    if avg:
        return torch.nn.L1Loss()(img_pred * mask_pred, img_gt * mask_gt)
    loss = torch.nn.L1Loss(reduction="none")(img_pred * mask_pred, img_gt * mask_gt)
    return torch.sum(loss, dim=(1, 2, 3)) / (loss.size(1) * loss.size(2) * loss.size(3))


def mask_texture_loss(images, img_gt, mask_gt, mask_wt=1.0, tex_wt=1.0):
    """Fused form of the two per-render losses the reference always applies to the SAME RGBA render
    (train_s1.py:211-215; loss_utils.py:41-48 and :103-116):
        mask_wt * neg_iou_loss(images[:, 3], mask_gt) + tex_wt * texture_loss_masks(images[:, :3], img_gt, mask_gt, images[:, 3])
    One reduction kernel forward and one kernel backward (csrc/losses.cu `k_losshead_*`).  Not a reference name --
    an addition; the two reference functions above stay available and give the same value."""
    return ops.mask_texture_loss(images, img_gt, mask_gt, mask_wt, tex_wt)[0]


def deform_l2reg(V):
    """loss_utils.py:118-123."""
    V = V.view(-1, V.size(2))
    return torch.mean(torch.norm(V, p=2, dim=1))


def sym_reg(verts):
    """loss_utils.py:125-126."""
    return torch.mean(torch.abs(verts[:, :, 1]))


class edge_regularization(nn.Module):
    """loss_utils.py:26-39."""

    def __init__(self, edges):
        super().__init__()
        self.edges = edges.long()

    def forward(self, pred):
        l2_loss = nn.MSELoss(reduction="mean")
        return l2_loss(pred[:, self.edges[:, 0]], pred[:, self.edges[:, 1]]) * pred.size(-1)


class PerceptualTextureLoss(object):
    """loss_utils.py:128-150.  LPIPS is a dense CNN with downloaded weights -- outside the hot path -- so
    this is a shim around the REFERENCE's own `nnutils/perceptual_loss.py::PerceptualLoss`, found through
    the overlay package (`umr_b200.compat.overlay`) or any importable `perceptual_loss` module.  When none
    is importable the constructor raises: the objective must never silently change to L1."""

    def __init__(self, perceptual_loss=None):
        if perceptual_loss is None:
            perceptual_loss = self._find()()
        self.perceptual_loss = perceptual_loss

    @staticmethod
    def _find():
        import importlib
        import sys
        tried = []
        names = [m[:-len("loss_utils")] + "perceptual_loss" for m in list(sys.modules)
                 if m.endswith(".nnutils.loss_utils") and not m.startswith("umr_b200")]
        for name in names + ["UMR.nnutils.perceptual_loss", "nnutils.perceptual_loss", "perceptual_loss"]:
            try:
                return importlib.import_module(name).PerceptualLoss
            except Exception as e:  # ImportError, missing LPIPS weights, ...
                tried.append("%s (%s: %s)" % (name, type(e).__name__, e))
        raise NotImplementedError(
            "texture_loss_type='perceptual' needs the reference's LPIPS module (nnutils/perceptual_loss.py + its "
            "weights), which is outside the H100 hot path and was not importable: %s.  Install umr_b200.compat."
            "overlay(<reference root>) or pass texture_loss_type='l1'." % "; ".join(tried))

    def __call__(self, img_pred, img_gt, mask_gt, mask_pred=None, avg=True):
        mask_gt = mask_gt.unsqueeze(1)
        if mask_pred is not None:
            dist = self.perceptual_loss(img_pred * mask_pred.unsqueeze(1), img_gt * mask_gt)
        else:
            dist = self.perceptual_loss(img_pred * mask_gt, img_gt * mask_gt)
        return dist.mean() if avg else dist


def entropy_loss(A):
    """loss_utils.py:184-192: mean row entropy of a K x N probability matrix."""
    return torch.mean(-torch.sum(A * torch.log(A), 1))


class TexCycle(nn.Module):
    """loss_utils.py:152-182: pull the mean texture flow of every VISIBLE face towards the
    renderer's pixel->face affinity `prob`."""

    def __init__(self, im_size=256, nf=1280, eps=1e-12):
        super().__init__()

    def forward(self, flow, prob, aggr_info, visible=None):
        """`visible` (extension): the [B,F] uint8 face-visibility bytes of `SoftRenderer.visible_faces`, used instead of
        scanning `aggr_info` (which may then be None)."""
        nb, nf = flow.size(0), flow.size(1)
        flow_grid = flow.reshape(nb, nf, -1, 2)
        if visible is not None:
            loss = ops.tex_cycle(flow_grid, prob, None, visible)
        else:
            loss = ops.tex_cycle(flow_grid, prob, aggr_info.reshape(nb, -1))
        # second output is for visualisation only in the reference (:181-182)
        avg_flow_vis = flow_grid[0, 0:10].mean(dim=1)
        return loss, avg_flow_vis


# ---------------------------------------------------------------------------------------------
# chamfer correspondence
# ---------------------------------------------------------------------------------------------
class CorrLossChamfer(nn.Module):
    """loss_utils.py:194-248.  `part_vertices` = (head, belly, neck, back) index tensors replaces the
    four `vertices_idx/*.npy` files the reference loads from `scops_path` (:197-209)."""

    def __init__(self, scops_path, image_size, part_vertices=None):
        super().__init__()
        if part_vertices is None:
            part_vertices = [torch.from_numpy(np.load(osp.join(scops_path, "vertices_idx/%s_vertices.npy" % n))).long()
                             for n in ("head", "belly", "neck", "back")]
        self.head_vertices, self.belly_vertices, self.neck_vertices, self.back_vertices = [
            torch.as_tensor(p).long() for p in part_vertices]
        self.head_num, self.belly_num = len(self.head_vertices), len(self.belly_vertices)
        self.neck_num, self.back_num = len(self.neck_vertices), len(self.back_vertices)
        self.renderer = SoftRenderer(image_size)
        self.weights = [1, 1, 0, 0]
        nums = [self.head_num]
        nums.append(nums[0] + self.belly_num)
        nums.append(nums[1] + self.neck_num)
        nums.append(nums[2] + self.back_num)
        self.nums = nums

    def _index_on(self, device):
        """Concatenated part-vertex indices on `device`, uploaded once (the reference indexes with CPU tensors on every
        call, loss_utils.py:227-230 -- an H2D copy per step that also breaks CUDA-graph capture)."""
        cache = self.__dict__.setdefault("_idx_cache", {})
        key = str(device)
        if key not in cache:
            cache[key] = torch.cat((self.head_vertices, self.belly_vertices, self.neck_vertices, self.back_vertices)).to(device)
        return cache[key]

    def forward(self, head_points, belly_points, neck_points, back_points, verts, cams, avg=True):
        groups = (self.head_vertices, self.belly_vertices, self.neck_vertices, self.back_vertices)
        targets = (head_points, belly_points, neck_points, back_points)
        idx = self._index_on(verts.device)
        if verts.is_cuda and self.renderer.proj_fn is geom_utils.orthographic_proj_withz:
            # one fused kernel per direction (csrc/vertex.cu k_corr_fwd / k_corr_bwd) instead of the ~250 launches of the
            # composition below: projection, per-part nearest target, weights, mean
            cache = self.__dict__.setdefault("_idx32_cache", {})
            key = (str(verts.device), int(verts.shape[1]))
            if key not in cache:
                # checked once per (device, vertex count): the kernels gather verts[:, idx] without a bounds test of their own
                if idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= verts.shape[1]):
                    raise IndexError("part vertex index out of range for a mesh of %d vertices" % verts.shape[1])
                # with its transposed table (vertex -> ascending j) for the deterministic backward's per-vertex gather
                cache[key] = (idx.to(torch.int32), _vertex_table(groups, int(verts.shape[1]), verts.device))
            sel, vert_table = cache[key]
            loss, vert2d = ops.corr_chamfer(verts, cams, sel, targets, self.nums, self.weights, vert_table)
            if avg:
                return torch.mean(loss), vert2d
            return loss
        vert2d = self.renderer.project_points(verts[:, idx, :], cams)  # [B, sum(sizes), 2]
        terms, start = [], 0
        for group, target, weight in zip(groups, targets, self.weights):
            stop = start + len(group)
            d_to_target, _, _, _ = distChamfer(vert2d[:, start:stop, :].contiguous(), target)
            terms.append(d_to_target * weight)
            start = stop
        loss = torch.mean(torch.cat(terms, dim=1), dim=1)
        if avg:
            return torch.mean(loss), vert2d
        return loss


def _vertex_table(groups, num_vertices, device):
    """The concatenated part selection transposed on the host (ops.vertex_incidence), uploaded to `device`."""
    rowptr, pos = ops.vertex_incidence(torch.cat(groups).numpy(), num_vertices)
    return torch.from_numpy(rowptr).to(device), torch.from_numpy(pos).to(device)


# ---------------------------------------------------------------------------------------------
# multi-hypothesis render losses
# ---------------------------------------------------------------------------------------------
def tile_hypotheses(x, num):
    """[B, ...] -> [B*num, ...]: every sample repeated once per camera hypothesis, hypotheses of one sample
    adjacent (the reference's `x.unsqueeze(1).repeat(1, num, ...).view(-1, ...)`, loss_utils.py:260-261,303-305)."""
    return x.unsqueeze(1).expand(x.size(0), num, *x.shape[1:]).reshape(x.size(0) * num, *x.shape[1:])


def expected_over_hypotheses(per_render, cam_probs):
    """[B*H] per-render losses -> scalar: probability-weighted sum over the H hypotheses, mean over B."""
    return (per_render.view(cam_probs.size(0), -1) * cam_probs).sum(dim=1).mean()


class MultiMaskLoss(nn.Module):
    """loss_utils.py:250-275: silhouette IoU over all camera hypotheses, weighted by `cam_probs`."""

    def __init__(self, image_size=256, renderer_type="softmax", num_hypo_cams=8):
        super().__init__()
        self.renderer = SoftRenderer(image_size, renderer_type)
        self.num_hypo_cams = num_hypo_cams
        self.image_size = image_size

    def forward(self, vs, fs, cams_all_hypo, cam_probs, masks_gt):
        H = self.num_hypo_cams
        # vertices / faces are NOT repeated per hypothesis (the reference materialises repeat(1, 8, ...) copies,
        # loss_utils.py:260-261): the vertex kernel broadcasts each mesh over its H cameras (SURVEY.md §8f-1)
        # only the alpha plane is used (loss_utils.py:262-263): the silhouette render skips the colour work, with the
        # same values and gradients
        mask_all_hypo = self.renderer.render_silhouettes(vs, fs, cams_all_hypo.view(-1, 7))
        per_render = neg_iou_loss(mask_all_hypo, tile_hypotheses(masks_gt, H), avg=False)
        return expected_over_hypotheses(per_render, cam_probs), mask_all_hypo


class NeuralRenderer(nn.Module):
    """nmr_pytorch.py:89-128 (`NeuralRenderer`) as MultiTextureLoss(renderer="nmr") uses it: orthographic projection with
    offset_z = 5, y flip, textured NMR render of detached geometry.  Camera hypotheses are broadcast like SoftRenderer's:
    vertices / faces / textures [B, ...], cams [B*H, 7] -> B*H renders."""

    def __init__(self, img_size=256):
        super().__init__()
        from ..neural_renderer import Renderer
        self.renderer = Renderer(image_size=img_size, anti_aliasing=True, camera_mode="look_at", perspective=False,
                                 background_color=[0, 0, 0])
        self.renderer.eye = [0, 0, -2.732]
        self.renderer.light_intensity_ambient = 0.8
        self.offset_z = 5.

    def ambient_light_only(self):
        self.renderer.light_intensity_ambient = 1
        self.renderer.light_intensity_directional = 0

    def forward(self, vertices, faces, cams, textures):
        H = cams.size(0) // vertices.size(0)
        verts = geom_utils.orthographic_proj_withz(tile_hypotheses(vertices, H), cams, offset_z=self.offset_z)
        verts[:, :, 1] *= -1  # nmr_pytorch.py:76-77
        return self.renderer.render_rgb(verts, tile_hypotheses(faces, H), textures)


class MultiTextureLoss(nn.Module):
    """loss_utils.py:277-331.  `texture_loss_type` defaults to "perceptual" like the reference; that branch needs the
    reference's LPIPS module (see PerceptualTextureLoss)."""

    def __init__(self, samples_per_gpu=32, num_hypo_cams=8, image_size=256, renderer_type="softmax",
                 texture_loss_type="perceptual", renderer="smr"):
        super().__init__()
        if renderer in "smr":   # substring tests, like the reference (:282, :309)
            self.renderer = SoftRenderer(image_size, renderer_type)
        else:
            self.renderer = NeuralRenderer(image_size)
        self.renderer.ambient_light_only()
        self.hard_renderer = SoftRenderer(image_size, "hard")
        if texture_loss_type in "perceptual":   # substring test, like the reference (:289)
            self.texture_loss = PerceptualTextureLoss()   # raises if the reference's LPIPS module is unavailable
        else:
            self.texture_loss = texture_loss_masks
        self.texture_cycle_fn = TexCycle(samples_per_gpu)
        self.num_hypo_cams = num_hypo_cams
        self.image_size = image_size
        self.which_renderer = renderer

    def forward(self, vs, fs, cams_all_hypo, cam_probs, proj_cam, rgbs, masks_gt, masks_pred, tx, tex_flow,
                dts_barrier):
        # textured softmax render of every hypothesis; vertices detached: only the texture learns here (:313)
        # ... and neither is the [B*8,F,T2,3] texture copy of loss_utils.py:305 (70.8 MB at batch 16): the raster kernels
        # read textures[b // 8] and accumulate the 8 hypotheses' texture gradients directly
        if self.which_renderer in "nmr":
            # loss_utils.py:310: the 36 texels of a face as a 6x6 image, repeated along the cube's first axis
            cube = tx.view(tx.size(0), tx.size(1), 6, 6, 3).unsqueeze(2).expand(-1, -1, 6, -1, -1, -1)
            texture_pred = self.renderer.forward(vs.detach(), fs, cams_all_hypo.view(-1, 7), cube)
        else:
            texture_rgba, _, _ = self.renderer.forward(vs.detach(), fs, cams_all_hypo.view(-1, 7), tx)
            texture_pred = texture_rgba[:, 0:3, :, :]
        tex_loss, tex_dt_loss, tex_cycle_loss = self._losses(vs, fs, cam_probs, proj_cam, rgbs, masks_gt, masks_pred,
                                                             texture_pred, tex_flow, dts_barrier)
        return tex_loss, tex_dt_loss, tex_cycle_loss, texture_pred

    def _losses(self, vs, fs, cam_probs, proj_cam, rgbs, masks_gt, masks_pred, texture_pred, tex_flow, dts_barrier):
        """(tex_loss, tex_dt_loss, tex_cycle_loss) of the rendered `texture_pred` (loss_utils.py:320-331)."""
        H = self.num_hypo_cams
        per_render = self.texture_loss(texture_pred, tile_hypotheses(rgbs, H), tile_hypotheses(masks_gt, H),
                                       masks_pred, avg=False)
        tex_loss = expected_over_hypotheses(per_render, cam_probs)
        tex_dt_loss = texture_dt_loss(tex_flow, dts_barrier)
        # visibility map from the HARD renderer; its p2f_info is identically zero (kernel.cu:417-431 is
        # softmax-only) -- reference quirk reproduced (SURVEY.md App. B-4)
        # loss_utils.py:327: `_, p2f_info, aggr_info = self.hard_renderer(...)` -- the image is dropped, so only the z-buffer's
        # winners are computed (visibility-only kernel on CUDA; identical p2f_info / aggr_info)
        vis = self.hard_renderer.visible_faces(vs.detach(), fs, proj_cam.detach())
        if vis is not None:   # CUDA: the visibility kernel hands TexCycle the visible-face bytes directly (no plane at all)
            p2f_info, visible = vis
            tex_cycle_loss, _ = self.texture_cycle_fn(tex_flow, p2f_info, None, visible=visible)
        else:
            p2f_info, aggr_info = self.hard_renderer.visibility(vs.detach(), fs, proj_cam.detach())
            face_ids = aggr_info[:, 1, :, :].reshape(vs.size(0), -1)
            tex_cycle_loss, _ = self.texture_cycle_fn(tex_flow, p2f_info.detach(), face_ids.detach())
        return tex_loss, tex_dt_loss, tex_cycle_loss


class MultiMaskTextureLoss(nn.Module):
    """MultiMaskLoss and MultiTextureLoss of one train_s2 step (experiments/train_s2.py:226-248) from ONE render.  Both
    render the same geometry from the same camera hypotheses in the same raster configuration, and alpha (prod) depends
    on neither light nor texture, so the textured render's alpha plane is the mask render's.  `SoftRenderer.render_split`
    renders once and splits the backward: the alpha plane's gradient reaches the geometry and cameras, the RGB planes'
    the textures only.  Not a reference name -- an addition; it returns what

        mask_loss, mask_all_hypo = MultiMaskLoss(...)(vs, fs, cams_all_hypo, cam_probs, masks_gt)
        tex_loss, tex_dt_loss, tex_cycle_loss, texture_pred = MultiTextureLoss(...)(
            vs.detach(), fs, cams_all_hypo.detach(), cam_probs.detach(), proj_cam, rgbs, masks_gt, mask_all_hypo, tx,
            tex_flow, dts_barrier)

    returns, with the same gradients (mask_all_hypo is the texture loss's `masks_pred`, undetached, as in the reference).
    The constructor takes the union of the two modules' arguments; with renderer="nmr" the two modules run as above."""

    def __init__(self, samples_per_gpu=32, num_hypo_cams=8, image_size=256, renderer_type="softmax",
                 texture_loss_type="perceptual", renderer="smr"):
        super().__init__()
        self.mask_loss_fn = MultiMaskLoss(image_size, renderer_type, num_hypo_cams)
        self.texture_loss_fn = MultiTextureLoss(samples_per_gpu, num_hypo_cams, image_size, renderer_type, texture_loss_type,
                                                renderer)
        self.num_hypo_cams = num_hypo_cams

    def forward(self, vs, fs, cams_all_hypo, cam_probs, proj_cam, rgbs, masks_gt, tx, tex_flow, dts_barrier):
        """-> (mask_loss, mask_all_hypo, tex_loss, tex_dt_loss, tex_cycle_loss, texture_pred)"""
        tl = self.texture_loss_fn
        if tl.which_renderer in "nmr":
            mask_loss, mask_all_hypo = self.mask_loss_fn(vs, fs, cams_all_hypo, cam_probs, masks_gt)
            out = tl(vs.detach(), fs, cams_all_hypo.detach(), cam_probs.detach(), proj_cam, rgbs, masks_gt, mask_all_hypo, tx,
                     tex_flow, dts_barrier)
            return (mask_loss, mask_all_hypo) + tuple(out)
        H = self.num_hypo_cams
        # the texture renderer's light (ambient only) colours the RGB planes; alpha is the mask render's
        rgba, _, _ = tl.renderer.render_split(vs, fs, cams_all_hypo.view(-1, 7), tx)
        mask_all_hypo = rgba[:, 3, :, :]
        per_render = neg_iou_loss(mask_all_hypo, tile_hypotheses(masks_gt, H), avg=False)
        mask_loss = expected_over_hypotheses(per_render, cam_probs)
        texture_pred = rgba[:, 0:3, :, :]
        tex_loss, tex_dt_loss, tex_cycle_loss = tl._losses(vs.detach(), fs, cam_probs.detach(), proj_cam, rgbs, masks_gt,
                                                           mask_all_hypo, texture_pred, tex_flow, dts_barrier)
        return mask_loss, mask_all_hypo, tex_loss, tex_dt_loss, tex_cycle_loss, texture_pred


# ---------------------------------------------------------------------------------------------
# part matching
# ---------------------------------------------------------------------------------------------
def _coordinate_maps(h, w, device):
    """scops_utils.py:12-19 (`get_coordinate_tensors(h, w)`): x_map[i,j] = j/h*2-1 over a (w,h) grid,
    y_map[i,j] = i/w*2-1 over (h,w) -- as written in the reference (square maps in practice)."""
    x_map = np.tile(np.arange(h), (w, 1)) / h * 2 - 1.0
    y_map = np.tile(np.arange(w), (h, 1)).T / w * 2 - 1.0
    return (torch.from_numpy(x_map.astype(np.float32)).to(device),
            torch.from_numpy(y_map.astype(np.float32)).to(device))


def batch_get_centers(pred_softmax, epsilon=1e-3):
    """scops_utils.py:37-54 vectorised: soft centroid of every (b, c) map (the reference loops over
    B x C in Python)."""
    B, C, H, W = pred_softmax.shape
    x_map, y_map = _coordinate_maps(H, W, pred_softmax.device)
    pm = pred_softmax + epsilon
    pdf = pm / pm.sum(dim=(2, 3), keepdim=True)
    xc = (pdf * x_map).sum(dim=(2, 3))
    yc = (pdf * y_map).sum(dim=(2, 3))
    return torch.stack((xc, yc), dim=2)


def label_image_one_hot(uv_img, uv_sampler, num_sym_faces, tex_size, num_labels=5):
    """The per-texel one-hot part ids of a UV label image (loss_utils.py:341-356): uv_img [1,1,H,W] float labels sampled
    at uv_sampler [1,F',T2,2] (grid_sample, align_corners=True), the last num_sym_faces faces appended again, rounded
    and one-hot encoded -> [1,F'+num_sym_faces,T2,num_labels].  `part_matching_loss` builds its `stex_one_hot` from
    `semantic_seg.png` with it, and `utils.semantic_template` from the label image it computes."""
    tex = torch.nn.functional.grid_sample(uv_img, uv_sampler, align_corners=True)
    tex = tex.view(tex.size(0), -1, tex.size(2), tex_size, tex_size).permute(0, 2, 3, 4, 1)
    tex = torch.cat([tex, tex[:, -num_sym_faces:]], 1)
    stex = torch.round(tex.reshape(tex.size(1), -1))
    nf, nt = stex.size()
    one_hot = torch.zeros(nf * nt, num_labels, device=stex.device)
    one_hot.scatter_(1, stex.view(-1, 1).long(), 1)
    return one_hot.view(1, nf, nt, num_labels)


class part_matching_loss(nn.Module):
    """loss_utils.py:333-440.  `stex_one_hot` [1,F,T2,5] (one-hot semantic part id per texel) replaces
    the `semantic_seg.png` + `uv_sampler` lookup of :341-356; when it is None the reference's file
    layout is read (needs imageio/PIL)."""

    def __init__(self, scops_path, uv_sampler, num_sym_faces, im_size=256, batch_size=32, loss_type="mse",
                 tex_size=6, num_cam=1, stex_one_hot=None):
        super().__init__()
        if stex_one_hot is None:
            from PIL import Image
            uv_img = np.asarray(Image.open(osp.join(scops_path, "semantic_seg.png"))).astype(np.float32)
            uv_img = torch.from_numpy(uv_img).view(1, 1, 128, 256).float().to(uv_sampler.device)
            stex_one_hot = label_image_one_hot(uv_img, uv_sampler, num_sym_faces, tex_size)
        n = batch_size * num_cam
        for k in (1, 2, 3, 4):
            self.register_buffer("stex%d" % k, stex_one_hot[:, :, :, k].unsqueeze(-1).repeat(n, 1, 1, 3))
        # the four part maps as ONE batch-shared 4-channel texture for the single-render path (SURVEY.md §8f-2)
        self.register_buffer("stex_parts", stex_one_hot[:, :, :, 1:5].contiguous().float(), persistent=False)
        self.renderer = SoftRenderer(im_size, "softmax")
        self.renderer.ambient_light_only()
        self.kl = nn.KLDivLoss(reduction="batchmean")
        proj = torch.zeros(n, 1, im_size, im_size)
        proj[:, 0, :, :] = 0.1
        self.register_buffer("proj", proj)
        self.register_buffer("weights", torch.tensor([0, 5.0, 0.0, 0.0, 5.0]).view(1, 5, 1, 1))
        self.loss_type = loss_type
        self.pack_parts = True  # ONE 4-channel render (CUDA) / 2 packed renders instead of the reference's 4 (same values)

    def forward(self, verts, faces, cams, part_segs, cam_probs=None, avg=True):
        bs = verts.size(0)
        if self.pack_parts and verts.is_cuda and self.renderer._fusable(verts):
            # The reference renders each one-hot part map as its own 3-identical-channel image (4 renders,
            # loss_utils.py:385-399).  Colour channels never interact in the rasteriser, so the four maps ride in the
            # four colour channels of ONE render (`color_channels = 4` kernels, one batch-shared [1,F,T2,4] texture):
            # one raster launch, identical values.  The channel-mean of the reference (mean of three equal numbers) is
            # reproduced on an expanded view.
            p, _, _ = self.renderer(verts, faces, cams, self.stex_parts)
            projs = [torch.mean(p[:, k:k + 1].expand(-1, 3, -1, -1), dim=1).unsqueeze(1) for k in range(4)]
        elif self.pack_parts:
            # generic path: parts 1-3 in the R/G/B channels of one render and part 4 in a second
            tex123 = torch.stack((self.stex1[:bs, :, :, 0], self.stex2[:bs, :, :, 0], self.stex3[:bs, :, :, 0]), dim=-1)
            p123, _, _ = self.renderer(verts, faces, cams, tex123)
            p4, _, _ = self.renderer(verts, faces, cams, self.stex4[:bs])
            projs = [torch.mean(p123[:, k:k + 1].expand(-1, 3, -1, -1), dim=1).unsqueeze(1) for k in range(3)]
            projs.append(torch.mean(p4[:, 0:3, :, :], dim=1).unsqueeze(1))
        else:
            projs = []
            for stex in (self.stex1, self.stex2, self.stex3, self.stex4):
                p, _, _ = self.renderer(verts, faces, cams, stex[:bs])
                projs.append(torch.mean(p[:, 0:3, :, :], dim=1).unsqueeze(1))
        return self.head(projs, part_segs, cam_probs, avg), projs

    def head(self, projs, part_segs, cam_probs=None, avg=True):
        """The loss from the four part maps `projs` ([B,1,H,W] each): the part-head kernels when every input is on the GPU,
        the maps are square, `part_segs` is data and B <= 65535 (DESIGN.md §13), else the torch composition."""
        c0 = self.proj[:projs[0].size(0)].detach()
        kld = self.loss_type in "kld"
        if not part_head_on_device(projs, c0, part_segs):
            return part_head_torch(projs, c0, part_segs, self.weights, kld, cam_probs, avg)
        bs, hw = part_segs.size(0), part_segs.size(2) * part_segs.size(3)
        terms = ops.part_matching_head(projs, c0, part_segs, self.weights, kld)
        if avg:
            loss_lmeqv = terms[:, 0].sum() / (bs * 8)
        else:
            loss_lmeqv = ((terms[:, 0] / 8).view(cam_probs.size()) * cam_probs).sum(dim=1).mean()
        if kld:
            loss_eqv = terms[:, 1].sum() / bs
        elif avg:
            loss_eqv = terms[:, 1].sum() / (bs * 5 * hw)
        else:
            loss_eqv = ((terms[:, 1] / (5 * hw)).view(cam_probs.size()) * cam_probs).sum(dim=1).mean()
        return (loss_eqv + loss_lmeqv) / 4.0


def part_head_on_device(projs, c0, part_segs):
    """Whether part_matching_loss's head runs on the part-head kernels: every input on the GPU, square maps, a
    `part_segs` that needs no gradient (the kernels differentiate the part maps only) and B <= 65535."""
    return (all(t.is_cuda for t in projs) and c0.is_cuda and part_segs.is_cuda and not part_segs.requires_grad
            and part_segs.dim() == 4 and part_segs.size(2) == part_segs.size(3) and part_segs.size(0) <= 65535)


def part_head_torch(projs, c0, part_segs, weights, kld, cam_probs=None, avg=True):
    """part_matching_loss's head as torch ops (loss_utils.py:401-440, scops_utils.py:37-54): the path of CPU tensors,
    non-square maps and a differentiable `part_segs`, and the reference the part-head kernels are tested against."""
    bs = part_segs.size(0)
    proj = torch.cat([c0] + list(projs), dim=1)
    centers_proj = batch_get_centers(nn.Softmax(dim=1)(proj)[:, 1:, :, :])
    centers_parts = batch_get_centers(nn.Softmax(dim=1)(part_segs)[:, 1:, :, :])
    if avg:
        loss_lmeqv = torch.nn.functional.mse_loss(centers_proj, centers_parts)
    else:
        loss_lmeqv = torch.nn.functional.mse_loss(centers_proj, centers_parts, reduction="none")
        loss_lmeqv = torch.sum(loss_lmeqv, dim=(1, 2)) / (loss_lmeqv.size(1) * loss_lmeqv.size(2))
        loss_lmeqv = (loss_lmeqv.view(cam_probs.size()) * cam_probs).sum(dim=1).mean()
    if kld:
        loss_eqv = torch.nn.functional.kl_div(torch.nn.functional.log_softmax(proj, dim=1),
                                              torch.nn.functional.softmax(part_segs, dim=1), reduction="batchmean")
    else:
        max_proj, _ = torch.max(proj.view(bs, 5, -1), dim=2)
        max_proj = max_proj.clamp_min(1e-5)
        proj_norm = proj / max_proj.view(bs, 5, 1, 1)
        max_part, _ = torch.max(part_segs.view(bs, 5, -1), dim=2)
        max_part = max_part.clamp_min(1e-5)
        part_norm = part_segs / max_part.view(bs, 5, 1, 1)
        if avg:
            loss_eqv = torch.mean(nn.MSELoss(reduction="none")(proj_norm, part_norm) * weights)
        else:
            _, cs, iis, _ = part_norm.size()
            loss_eqv = nn.MSELoss(reduction="none")(proj_norm, part_norm) * weights
            loss_eqv = torch.sum(loss_eqv, dim=(1, 2, 3)) / (cs * iis * iis)
            loss_eqv = (loss_eqv.view(cam_probs.size()) * cam_probs).sum(dim=1).mean()
    total_loss = loss_eqv + loss_lmeqv
    return total_loss / 4.0
