"""Generates tests/golden/dense_crf.pt from oracle/dense_crf.py: a 24 x 20 synthetic frame (fp32 and its bytes), seeded
logits for 5 classes, both lattices (packed keys, counts) and Q after 10 mean-field iterations.  Run from the repository
root: python tests/golden/make_golden_dense_crf.py"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
from oracle import dense_crf as dc  # noqa: E402
from oracle.slic import synthetic_image  # noqa: E402


def make():
    img = synthetic_image(24, 20, seed=4)
    bgr = dc.crf_image_bytes(img)
    logits = (np.random.default_rng(11).normal(size=(5, 24, 20)) * 3).astype(np.float32)
    spatial = dc.Lattice(dc.spatial_features(24, 20))
    bilateral = dc.Lattice(dc.bilateral_features(bgr))
    return {"img": torch.from_numpy(img), "bgr": torch.from_numpy(bgr.copy()), "logits": torch.from_numpy(logits),
            "spatial_keys": torch.from_numpy(spatial.packed.view(np.int64)), "spatial_counts": torch.from_numpy(spatial.counts),
            "bilateral_keys": torch.from_numpy(bilateral.packed.view(np.int64)),
            "bilateral_counts": torch.from_numpy(bilateral.counts),
            "q": torch.from_numpy(dc.dense_crf(logits, bgr))}


if __name__ == "__main__":
    torch.save(make(), os.path.join(os.path.dirname(os.path.abspath(__file__)), "dense_crf.pt"))
