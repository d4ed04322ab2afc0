"""Generate tests/golden/efficientnet_pyramid.pt by running the REFERENCE's own torchvision feature pyramid and pooling.

Run with a checkout of the reference repository and torchvision installed:
``WVN_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_efficientnet.py``

  * the reference's ``TorchVisionInterface(device="cpu", model_type="efficientnet_b0", input_size=448,
    pretrained=False)`` (feature_extractor/torchvision_interface.py, path-imported from the reference tree) with the
    seeded weights of ``weights.synthetic_efficientnet_b0_state_dict`` loaded into its ``model`` (``strict=False``: the
    extractor has no ``classifier``), on one seeded 448 x 448 image.  Its return nodes
    ``features.{2,3,4,6}.0.block.0.2`` and ``features.8.2`` (the SiLU inside each ``Conv2dNormActivation``) do not
    exist under torchvision >= 0.2x, whose ``create_feature_extractor`` treats ``Conv2dNormActivation`` as a leaf, and
    the constructor raises there.  The module's ``create_feature_extractor`` is therefore wrapped to ask for the
    modules themselves, ``features.{2,3,4,6}.0.block.0`` and ``features.8``, whose outputs are those SiLU outputs;
    everything else runs as the reference wrote it;
  * the reference's ``FeatureExtractor.sparsify_features`` (its source, executed from the reference file) on that
    pyramid with grid segments of cell_size 32;
  * the same call with grid segments of cell_size 16, recorded as the exception it raises (a segment missing from the
    14 x 14 level).
The maps are large, so each is stored as its per-channel sums plus every 97th element, and the pooled rows as every
7th column.
"""
from __future__ import annotations

import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import _reference_method  # noqa: E402
from oracle import ref_import  # noqa: E402
from wild_visual_navigation_b200.feature_extractor.weights import synthetic_efficientnet_b0_state_dict  # noqa: E402

STRIDE = 97
COL_STRIDE = 7
SIZE = 448
# the reference's return nodes -> the modules whose outputs they are
NODE_TRANSLATION = {f"features.{s}.0.block.0.2": f"features.{s}.0.block.0" for s in (2, 3, 4, 6)}
NODE_TRANSLATION["features.8.2"] = "features.8"


def grid_seg(cell):
    ys = torch.arange(SIZE) // cell
    return ys[:, None] * (SIZE // cell) + ys[None, :]


def main():
    assert ref_import.available(), "set WVN_REFERENCE_ROOT to a checkout of the reference repository"
    ref_import.load()  # the stub package with WVN_ROOT_DIR
    tvi = ref_import._load("wild_visual_navigation.feature_extractor.torchvision_interface",
                           "wild_visual_navigation/feature_extractor/torchvision_interface.py")
    original = tvi.create_feature_extractor
    tvi.create_feature_extractor = lambda model, return_nodes: original(
        model, return_nodes={NODE_TRANSLATION[k]: v for k, v in return_nodes.items()})
    sparsify = _reference_method("wild_visual_navigation/feature_extractor/feature_extractor.py", "sparsify_features")
    me = types.SimpleNamespace(_feature_type="torchvision", _segmentation_type="grid")
    img = torch.rand(1, 3, SIZE, SIZE, generator=torch.Generator().manual_seed(2024))
    ti = tvi.TorchVisionInterface(device="cpu", model_type="efficientnet_b0", input_size=SIZE, pretrained=False)
    missing, unexpected = ti.model.load_state_dict(synthetic_efficientnet_b0_state_dict(seed=1), strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    pyr = ti.inference(img.clone())
    assert list(pyr) == [f"feat{i}" for i in range(1, 6)], list(pyr)
    feat32 = sparsify(me, pyr, grid_seg(32))
    try:
        sparsify(me, pyr, grid_seg(16))
        raised = None
    except Exception as e:  # noqa: BLE001 - recorded, not handled
        raised = type(e).__name__
    out = {"image_seed": 2024, "stride": STRIDE, "col_stride": COL_STRIDE, "weights_seed": 1,
           "nodes": dict(NODE_TRANSLATION),
           "shapes": {k: tuple(v.shape) for k, v in pyr.items()},
           "channel_sums": {k: v.double().sum((0, 2, 3)) for k, v in pyr.items()},
           "samples": {k: v.reshape(-1)[::STRIDE].clone() for k, v in pyr.items()},
           "grid32_feat": feat32[:, ::COL_STRIDE].clone(),
           "grid16_raises": raised}
    torch.save(out, os.path.join(HERE, "efficientnet_pyramid.pt"))
    print("efficientnet_pyramid.pt", os.path.getsize(os.path.join(HERE, "efficientnet_pyramid.pt")), out["shapes"],
          raised)


if __name__ == "__main__":
    main()
