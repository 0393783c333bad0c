"""Generate tests/golden/semantic_template/reference.npz from THE REFERENCE ITSELF: `ShapenetTester.compute_uv` of its
experiments/avg_uv.py (:133-307) run on CPU on seeded synthetic inputs.

    python tests/golden/make_semantic_template_golden.py <UMR checkout>

The model, data loader, renderer, texture loss, colour maps and `sr.Mesh` are stubs that replay the seeded inputs;
`.cuda()` is the identity, `grid_sample` is pinned to align_corners=True (the torch-1.1 default the reference was
written for), `np.int` / `np.float` are restored and `scipy.misc` is stubbed.  The template mesh is icosphere(3) (642
vertices, every one on at least five faces, so the reference's vertex loop runs) with num_sym_faces = 624 and T = 6.

The .npz holds the inputs (part_segs [NB,B,C,S,S], uvimage_pred [NB,B,2,H,W], uv_sampler [F',T2,2], faces [F,3]) and
what the reference made of them: the exemplar `best_uv` [C,H,W], `semantic_prob` [H,W,C], the `semantic_seg.png`
label image and the head, neck, back and belly vertex lists.
"""
import functools
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

NB, B, C, S, H, W, T, K = 2, 8, 5, 16, 16, 32, 6, 5
NUM_SYM = 624
PARTS = ("head", "neck", "back", "belly")


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__path__ = []
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


class _Mesh(object):
    def __init__(self, *a, **k):
        pass

    def save_obj(self, *a, **k):
        pass


class _Model(object):
    """Replays one seeded set of outputs per batch, in loader order, once per pass."""

    def __init__(self, verts, faces, sampler, uv, rng):
        self.verts = torch.from_numpy(verts)
        self.faces = torch.from_numpy(faces.astype(np.int64))
        self.mean_v = self.verts
        self.uv_sampler = torch.from_numpy(sampler)[None]
        self.texture_predictor = types.SimpleNamespace(num_sym_faces=NUM_SYM)
        self.outputs = [dict(delta_v=torch.from_numpy(rng.normal(0, 0.01, (B,) + verts.shape).astype(np.float32)),
                             cam=torch.from_numpy(rng.normal(0, 1, (B, 7)).astype(np.float32)),
                             uvimage_pred=torch.from_numpy(uv[i]),
                             tex_flow=torch.zeros(B, faces.shape[0], T, T, 2)) for i in range(NB)]
        self.calls = 0

    def __call__(self, imgs):
        out = self.outputs[self.calls % NB]
        self.calls += 1
        return out

    def get_mean_shape(self):
        return self.verts


def main(reference):
    import semantic_template_oracle as sto
    from umr_b200 import synth

    rng = np.random.default_rng(23)
    segs = np.stack([sto.part_segs(rng, B, C, S) for _ in range(NB)])
    uv = np.stack([sto.uvimage_pred(rng, B, H, W, spread=1.05) for _ in range(NB)])
    verts, faces = synth.icosphere(3)
    sampler = sto.uv_sampler(verts, faces[:faces.shape[0] - NUM_SYM], T)
    losses = [torch.from_numpy(rng.uniform(1, 2, B).astype(np.float32)) for _ in range(NB)]

    np.int, np.float = int, float
    real_cuda, real_grid_sample = torch.Tensor.cuda, torch.nn.functional.grid_sample
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.functional.grid_sample = functools.partial(real_grid_sample, align_corners=True)
    _module("scipy.misc")
    _module("soft_renderer", Mesh=_Mesh)
    _module("soft_renderer.functional")
    _module("neural_renderer")
    _module("refpkg")
    _module("refpkg.experiments")
    _module("refpkg.nnutils", loss_utils=_module("refpkg.nnutils.loss_utils"),
            test_utils=_module("refpkg.nnutils.test_utils", Tester=object),
            geom_utils=_module("refpkg.nnutils.geom_utils",
                               sample_textures=lambda flow, img: torch.zeros(1, flow.shape[1], T, T, img.shape[1])),
            smr=_module("refpkg.nnutils.smr", SoftRenderer=object), cub_mesh_s1=_module("refpkg.nnutils.cub_mesh_s1"))
    _module("refpkg.data", cub=_module("refpkg.data.cub"))
    _module("refpkg.utils", tf_visualizer=_module("refpkg.utils.tf_visualizer", green=str),
            transformations=_module("refpkg.utils.transformations"), image=_module("refpkg.utils.image"))
    spec = importlib.util.spec_from_file_location("refpkg.experiments.avg_uv",
                                                  os.path.join(reference, "experiments", "avg_uv.py"))
    ref = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = ref
    spec.loader.exec_module(ref)

    out_dir = tempfile.mkdtemp()
    opts = types.SimpleNamespace(symmetric=False, batch_size=B, tex_size=T, num_parts=C - 1, out_dir=out_dir)
    ref.opts = opts
    tester = ref.ShapenetTester.__new__(ref.ShapenetTester)
    tester.opts = opts
    tester.model = _Model(verts, faces, sampler, uv, rng)
    tester.mean_shape = tester.model.get_mean_shape()
    tester.faces = tester.model.faces.view(1, -1, 3)
    tester.renderer = types.SimpleNamespace(forward=lambda v, f, c: (torch.zeros(v.shape[0], 4, S, S), None, None))
    tester.texture_loss_fn = lambda *a, **k: losses[(tester.model.calls - 1) % NB].clone()   # the batch just run
    tester.colorize = lambda a: np.zeros((3,) + np.asarray(a).shape[:2], np.float32)
    tester.batch_colorize = lambda t: torch.zeros(t.shape[0], 3, t.shape[1], t.shape[2])
    tester.resnet_transform = lambda x: x
    tester.dataloader = [dict(img=torch.zeros(B, 3, S, S), mask=torch.zeros(B, S, S),
                              part_prob=torch.from_numpy(segs[i]).permute(0, 2, 3, 1).contiguous(), img_path=None)
                         for i in range(NB)]
    try:
        tester.compute_uv()
    finally:
        torch.Tensor.cuda, torch.nn.functional.grid_sample = real_cuda, real_grid_sample

    from PIL import Image
    out = dict(part_segs=segs, uvimage_pred=uv, uv_sampler=sampler, faces=faces, num_sym_faces=np.int64(NUM_SYM),
               k=np.int64(K), best_uv=tester.best_uv[0].numpy(),
               semantic_prob=np.load(os.path.join(out_dir, "semantic_prob.npy")),
               semantic_seg=np.asarray(Image.open(os.path.join(out_dir, "semantic_seg.png"))))
    for name in PARTS:
        out[name] = np.load(os.path.join(out_dir, "%s_vertices.npy" % name)).astype(np.int64)
    path = os.path.join(HERE, "semantic_template", "reference.npz")   # apart from the raster goldens test_oracle.py globs
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes;", {n: len(out[n]) for n in PARTS})


if __name__ == "__main__":
    main(sys.argv[1])
