"""Tiny end-to-end exercise of every kernel, meant to be run under compute-sanitizer
(memcheck / racecheck / initcheck) on the GPU box:
    compute-sanitizer --tool memcheck python tools/sanitize_smoke.py
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from umr_b200 import raster, synth
from umr_b200.nnutils import chamfer_python, geom_utils, loss_utils, smr


def main():
    dev = torch.device("cuda:0")
    seed = int(os.environ.get("SEED", "0"))
    torch.manual_seed(seed)
    rng = np.random.default_rng(seed)
    v, f = synth.icosphere(2)
    B, IS = 2, 24
    verts = torch.from_numpy(synth.bird_like(v, rng, B)).to(dev).requires_grad_(True)
    faces = torch.from_numpy(f.astype(np.int64))[None].repeat(B, 1, 1).to(dev)
    cams = torch.from_numpy(synth.cameras(rng, B)).to(dev).requires_grad_(True)
    imgs = torch.from_numpy(synth.smooth_images(rng, B, IS)).to(dev)
    masks = torch.from_numpy(synth.ellipse_masks(rng, B, IS)).to(dev)
    flow = torch.from_numpy(synth.texture_flow(rng, B, f.shape[0], 2)).to(dev).requires_grad_(True)
    tex = geom_utils.sample_textures(flow, imgs).reshape(B, f.shape[0], 4, 3)
    total = 0
    for rtype in ("softmax", "hard"):
        r = smr.SoftRenderer(IS, rtype)
        out, p2f, aggr = r(verts, faces, cams, tex)
        total = total + loss_utils.neg_iou_loss(out[:, 3], masks) + loss_utils.texture_loss_masks(out[:, :3], imgs, masks, out[:, 3])
    cyc, _ = loss_utils.TexCycle()(flow, p2f.detach(), aggr[:, 1].reshape(B, -1).detach())
    dt = torch.rand(B, 1, IS, IS, device=dev)
    total = total + cyc + loss_utils.texture_dt_loss(flow, dt)
    pts = torch.rand(B, 10, 2, device=dev) - 0.5
    d1, d2, _, _ = chamfer_python.distChamfer(r.project_points(verts[:, :40], cams).contiguous(), pts)
    total = total + d1.mean() + d2.mean()
    # generic-mode kernels
    fv = torch.from_numpy(synth.raster_space_faces(verts.detach().cpu().numpy(), f, cams.detach().cpu().numpy())).to(dev).requires_grad_(True)
    vt = torch.rand(B, f.shape[0], 3, 3, device=dev, requires_grad=True)
    o2, _, _ = raster.soft_rasterize(fv, vt, IS, dist_func="barycentric", aggr_func_alpha="sum", texture_type="vertex",
                                     sigma_val=1e-4, dist_eps=1e-4, gamma_val=1e-3, anti_aliasing=True)
    total = total + o2.mean()
    # round-2 kernels: fused loss head, camera-hypothesis broadcast (vertex + raster kernels, shared textures),
    # the 32x32-tile forward + its streamed backward, mesh regularisers, distance transform, texture atlas
    from umr_b200 import ops
    from umr_b200 import soft_renderer as sr
    r2 = smr.SoftRenderer(IS, "softmax")
    r2.ambient_light_only()
    H = 4
    cams_h = torch.from_numpy(np.stack([synth.cameras(rng, H) for _ in range(B)])).view(-1, 7).to(dev)
    img_h, _, _ = r2(verts, faces, cams_h, tex)                      # [B*H] renders of B meshes / textures
    gt_h = imgs.repeat_interleave(H, 0)
    total = total + loss_utils.mask_texture_loss(img_h, gt_h, masks.repeat_interleave(H, 0), 2.5, 3.0)
    old_tile = raster.FORWARD_TILE
    raster.FORWARD_TILE = 32
    try:
        img32, _, _ = r2(verts, faces, cams, tex[:1])               # one batch-shared texture, 32x32-tile kernels
        total = total + img32.mean()
    finally:
        raster.FORWARD_TILE = old_tile
    # 4-colour-channel part-map render (one batch-shared texture) + texture-only backward for detached geometry
    parts = torch.rand(1, f.shape[0], 4, 4, device=dev)
    img4, _, _ = r2(verts, faces, cams, parts)
    assert img4.shape[1] == 5
    total = total + img4[:, :4].mean()
    tex_leaf = tex.detach().clone().requires_grad_(True)
    img_t, _, _ = r2(verts.detach(), faces, cams.detach(), tex_leaf)
    total = total + img_t[:, :3].mean()
    # visibility kernels (MultiTextureLoss's hard render): per-pixel planes, face-parallel visible-face bytes -> TexCycle
    rh = smr.SoftRenderer(IS, "hard")
    _, aggr_v = rh.visibility(verts, faces, cams)
    p2f_v, vis_bytes = rh.visible_faces(verts, faces, cams)
    assert aggr_v.shape[1] == 2 and vis_bytes.dtype == torch.uint8
    cyc2, _ = loss_utils.TexCycle()(flow, p2f_v, None, visible=vis_bytes)
    total = total + cyc2
    # fused CorrLossChamfer (projection + per-part nearest target + mean), also through a one-mesh expanded view
    pv = [torch.from_numpy(p) for p in synth.part_vertex_sets(rng, v.shape[0], sizes=(5, 9, 5, 9))]
    pp = [torch.from_numpy(p).to(dev) for p in synth.part_points(rng, B)]
    corr_fn = loss_utils.CorrLossChamfer(None, IS, part_vertices=pv)
    c1, _ = corr_fn(pp[0], pp[1], pp[2], pp[3], verts, cams)
    c2 = corr_fn(pp[0], pp[1], pp[2], pp[3], verts[:1].expand(B, -1, -1), cams, avg=False)
    total = total + c1 + c2.sum()
    fcpu = torch.from_numpy(f.astype(np.int64))
    total = total + 1e-3 * sr.LaplacianLoss(torch.from_numpy(v), fcpu).to(dev)(verts).sum() \
        + 1e-3 * sr.FlattenLoss(fcpu).to(dev)(verts).sum()
    dtb = ops.dt_barrier(masks)
    assert torch.isfinite(dtb).all()
    atlas, _ = sr.functional.create_texture_image(tex[0].detach(), 8)
    assert np.isfinite(atlas).all()
    # texture reload at the edges of the uv range (whole faces on u or v = 1, negative uv): corners clamped to the image
    uv_edge = torch.tensor([[[1.0, 1.0]] * 3, [[1.0, 0.0], [1.0, 0.5], [1.0, 1.0]], [[-0.5, -1.0]] * 3], device=dev)
    tex_edge = ops.load_textures(torch.rand(5, 4, 3, device=dev), uv_edge, torch.zeros(3, 9, 3, device=dev),
                                 torch.ones(3, dtype=torch.int32, device=dev))
    assert torch.isfinite(tex_edge).all()
    # batch crop / resize / mirror / normalisation (both launches), then the part points on its outputs
    from umr_b200.utils import crop_loader, image
    wins = [crop_loader.CropWindow(rng.integers(0, 256, (9, 7, 3), dtype=np.uint8), np.ones((9, 7), np.uint8), 2, 1, 11, True),
            crop_loader.CropWindow(rng.integers(0, 256, (5, 6, 1), dtype=np.uint8), np.ones((5, 6), np.uint8), 0, 3, 8, False)]
    cb = crop_loader.collate([{"crop": w} for w in wins])
    c_imgs, c_inp, c_masks, c_prob, c_segs = image.crop_batch(cb["crop_pack"].to(dev), cb["crop_table"], IS,
                                                              torch.rand(2, IS, IS, 5, device=dev) + 0.1)
    assert torch.isfinite(c_inp).all() and torch.isfinite(c_segs).all()
    image.part_points(c_prob, c_masks, num_samples=(2, 2, 2, 2))
    total.backward()
    torch.cuda.synchronize()
    assert torch.isfinite(verts.grad).all() and torch.isfinite(cams.grad).all() and torch.isfinite(flow.grad).all()
    print("sanitize_smoke ok: loss %.6f" % float(total))


if __name__ == "__main__":
    main()
