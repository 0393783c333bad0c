"""Generate tests/golden/crop/reference.npz from THE REFERENCE ITSELF: its `BaseDataset.__getitem__` (data/base.py, with
its utils/image.py and utils/transformations.py) on seeded synthetic uint8 images, then `set_input`'s two normalisations
(experiments/train_s2.py:169-192) in torch.

    python tests/golden/make_crop_golden.py <UMR checkout>

data/base.py is loaded by spec inside a stand-in package, so its relative imports resolve to the reference's own
utils.  The image read returns the synthetic image, `np.load` the synthetic part map, and `prob2center` / `sample_prob`
are stubbed (their part points are not under test here).  Per case the .npz holds the inputs (source image, mask, tight
box, parts, sfm pose, padding and jitter fractions, seed, part map) and the reference's outputs (the square box, the
flip, the float32 imgs / input_imgs / masks / part_prob / part_segs, kp and sfm_pose).
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch
import torchvision

HERE = os.path.dirname(os.path.abspath(__file__))
S = 64
KP_PERM = np.array([1, 2, 3, 4, 5, 6, 11, 12, 13, 10, 7, 8, 9, 14, 15]) - 1   # data/cub.py:79


def load_reference(reference):
    pkg = types.ModuleType("umr_ref")
    pkg.__path__ = []
    sys.modules["umr_ref"] = pkg
    mods = {}
    for name, rel in (("umr_ref.utils", None), ("umr_ref.data", None),
                      ("umr_ref.utils.image", "utils/image.py"),
                      ("umr_ref.utils.transformations", "utils/transformations.py"),
                      ("umr_ref.data.base", "data/base.py")):
        if rel is None:
            m = types.ModuleType(name)
            m.__path__ = []
            sys.modules[name] = m
        else:
            spec = importlib.util.spec_from_file_location(name, os.path.join(reference, rel))
            m = importlib.util.module_from_spec(spec)
            sys.modules[name] = m
            spec.loader.exec_module(m)
            setattr(sys.modules[name.rsplit(".", 1)[0]], name.rsplit(".", 1)[1], m)
        mods[name] = m
    return mods["umr_ref.data.base"], mods["umr_ref.utils.image"]


def cases():
    """(name, image shape, tight box [x1, y1, x2, y2] 1-indexed, pf, jf, part map?)"""
    return [
        ("grey", (50, 60), [12, 9, 44, 40], 0.05, 0.05, True),
        ("past_left_top", (48, 56, 3), [-6, -4, 30, 28], 0.05, 0.05, False),
        ("past_right_bottom", (48, 56, 3), [30, 25, 70, 60], 0.05, 0.05, False),
        ("outside", (40, 44, 3), [200, 5, 230, 35], 0.05, 0.05, False),
        ("L1", (30, 30, 3), [10, 12, 10, 12], 0.0, 0.0, False),
        ("L_lt_S", (60, 60, 3), [11, 11, 50, 50], 0.0, 0.0, True),
        ("L_eq_S", (70, 80, 3), [5, 3, 68, 66], 0.0, 0.0, False),
        ("L_2S_minus_1", (90, 90, 3), [-20, -17, 106, 109], 0.0, 0.0, False),
        ("L_2S", (90, 90, 3), [-20, -17, 107, 110], 0.0, 0.0, False),
        ("L_2S_plus_1", (90, 90, 3), [-20, -17, 108, 111], 0.0, 0.0, False),
        ("L_large", (100, 120, 3), [-200, -240, 400, 360], 0.05, 0.05, False),
        ("grey_flat_box", (40, 64), [3, 15, 60, 25], 0.05, 0.05, False),
    ]


def flip_for(seed):
    st = np.random.get_state()
    np.random.seed(seed)
    np.random.random(4)
    f = bool(np.random.rand(1) > 0.5)
    np.random.set_state(st)
    return f


def main(reference):
    base, ref_image = load_reference(reference)
    rng = np.random.default_rng(23)
    normalize = torchvision.transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])
    out = {}
    names = []
    for i, (name, shape, box, pf, jf, parts) in enumerate(cases()):
        # alternate the flip: the first seed from 100 i whose draw gives it
        seed = next(s for s in range(100 * i, 100 * i + 100) if flip_for(s) == bool(i % 2))
        yy, xx = np.mgrid[:shape[0], :shape[1]]
        wave = 64 * (1 + np.sin(xx / 7.0 + yy / 11.0))
        img = rng.integers(0, 256, shape) // 2 + (wave[..., None] if len(shape) == 3 else wave) * 0.9
        img = np.clip(img, 0, 255).astype(np.uint8)
        mask = (((yy - shape[0] / 2) / (shape[0] / 3)) ** 2 + ((xx - shape[1] / 2) / (shape[1] / 3)) ** 2 < 1)
        mask = mask.astype(np.uint8)
        kpts = np.stack([rng.uniform(-5, shape[1] + 5, 15), rng.uniform(-5, shape[0] + 5, 15),
                         (rng.random(15) > 0.3).astype(np.float64)])
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        rot = base.transformations.quaternion_matrix(q)[:3, :3]
        sfm_scale, sfm_trans = np.float64(rng.uniform(100, 300)), rng.uniform(0, 60, 2)
        pp = None
        if parts:
            pp = (np.round(rng.random((S, S, 5)) * 64) / 64).astype(np.float32)
            if name == "grey":
                pp[..., 3] = 0.0   # a part channel zero under the mask: set_input's 0 / 0
        anno = types.SimpleNamespace(rel_path="img_%d.jpg" % i, mask=mask,
                                     bbox=types.SimpleNamespace(x1=box[0], y1=box[1], x2=box[2], y2=box[3]), parts=kpts)
        anno_sfm = types.SimpleNamespace(scale=sfm_scale, trans=sfm_trans, rot=rot)
        opts = types.SimpleNamespace(img_size=S, jitter_frac=jf, padding_frac=pf, use_scops=pp is not None,
                                     scops_path="scops", split="train")
        ds = base.BaseDataset.__new__(base.BaseDataset)
        ds.opts, ds.img_size, ds.jitter_frac, ds.padding_frac = opts, S, jf, pf
        ds.filter_key, ds.mirror, ds.kp_perm, ds.scops_path = None, True, KP_PERM, "scops"
        ds.head_points_num = ds.neck_points_num = ds.belly_points_num = ds.back_points_num = 1
        ds.anno, ds.anno_sfm, ds.img_dir = [anno], [anno_sfm], "imgs"
        boxes = []
        real_square, real_load = ref_image.square_bbox, np.load
        ref_image.square_bbox = lambda b: boxes.append(real_square(b)) or boxes[-1]
        base.scipy.misc.imread = lambda path: img
        np.load = lambda path: pp.copy()
        ref_image.prob2center = lambda *a, **k: np.zeros(2)
        ref_image.sample_prob = lambda *a, **k: np.zeros((1, 2))
        try:
            np.random.seed(seed)
            elem = ds[0]
        finally:
            ref_image.square_bbox, np.load = real_square, real_load
        # set_input (train_s2.py:169-192) on a batch of one
        img_t = torch.from_numpy(elem["img"][None]).type(torch.FloatTensor)
        input_t = img_t.clone()
        input_t[0] = normalize(input_t[0])
        mask_t = torch.from_numpy(elem["mask"][None]).type(torch.FloatTensor)
        rec = dict(src=img, src_mask=mask, bbox=np.array(box, np.float64), parts=kpts, sfm_scale=sfm_scale,
                   sfm_trans=sfm_trans, sfm_rot=rot, fracs=np.array([pf, jf]), seed=np.int64(seed),
                   sq_bbox=np.array(boxes[0], np.float64), flip=np.bool_(flip_for(seed)),
                   imgs=img_t[0].numpy(), input_imgs=input_t[0].numpy(), masks=mask_t[0].numpy(),
                   kp=elem["kp"], sfm_pose=elem["sfm_pose"])
        if pp is not None:
            rec["part_in"] = pp
            rec["part_prob"] = np.asarray(elem["part_prob"], np.float32)
            segs = torch.from_numpy(rec["part_prob"][None].copy()).type(torch.FloatTensor).permute(0, 3, 1, 2)
            for ch in range(5):
                sl = segs[:, ch, :, :] * mask_t
                k, _ = torch.max(sl.view(sl.size(0), -1), dim=1)
                segs[:, ch, :, :] = sl / k.view(-1, 1, 1)
            rec["part_segs"] = segs[0].numpy()
        for k, v in rec.items():
            out["%s/%s" % (name, k)] = v
        names.append(name)
    out["cases"] = np.array(names)
    os.makedirs(os.path.join(HERE, "crop"), exist_ok=True)
    path = os.path.join(HERE, "crop", "reference.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
