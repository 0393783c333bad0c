"""Generate tests/golden/part_points/reference.npz from THE REFERENCE ITSELF: `prob2center` and `sample_prob` of its
utils/image.py (:168-206) on seeded SCOPS-like inputs, with every torch.multinomial draw recorded.

    python tests/golden/make_part_points_golden.py <UMR checkout>

The .npz holds the inputs (part_prob [B,S,S,5] float32, mask [B,S,S] as the loader has it, after cv2.resize), and per
(image, channel) the reference's centre, its multinomial draws in draw order and the points it kept.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

CHANNELS = (1, 2, 3, 4)
NUM_SAMPLES = (10, 10, 30, 30)   # data/base.py:67-68, head / neck / back / belly


def main(reference):
    import part_points_oracle as ppo
    spec = importlib.util.spec_from_file_location("ref_image", os.path.join(reference, "utils", "image.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    prob, mask = ppo.scops_like(np.random.default_rng(17), 3, 32)
    mask = np.round(mask * 8) / 8   # float32-exact soft rim
    real = torch.multinomial
    recorded = []

    def multinomial(pdf, num_samples):
        out = real(pdf, num_samples)
        recorded.append(out.numpy().copy())
        return out
    torch.manual_seed(5)
    ref.torch.multinomial = multinomial
    centres, draws, kept = [], [], []
    try:
        for b in range(prob.shape[0]):
            for ch, n in zip(CHANNELS, NUM_SAMPLES):
                c = ref.prob2center(prob[b], mask[b], ch=ch)
                pts = ref.sample_prob(prob[b], mask[b], c, num_samples=n, ch=ch)
                centres.append(c.numpy())
                kept.append(pts.numpy())
                draws.append(recorded[-1])
    finally:
        ref.torch.multinomial = real
    out = dict(part_prob=prob, mask=mask.astype(np.float32), channels=np.array(CHANNELS), num_samples=np.array(NUM_SAMPLES),
               centres=np.array(centres, np.float32).reshape(prob.shape[0], len(CHANNELS), 2))
    for k, n in enumerate(NUM_SAMPLES):
        out["draws_%d" % k] = np.stack(draws[k::len(CHANNELS)])
        out["points_%d" % k] = np.stack(kept[k::len(CHANNELS)])
    path = os.path.join(HERE, "part_points", "reference.npz")   # apart from the raster goldens test_oracle.py globs
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
