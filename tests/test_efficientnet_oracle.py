"""CPU tests of the EfficientNet-B0 feature backbone's oracle, weights and argument checks.

  oracle vs torchvision     efficientnet_b0 behind create_feature_extractor on the block-output nodes (the modules
                            whose SiLU outputs the reference's return nodes name), seeded weights, 224 and 448, within
                            fp32 rounding (skipped without torchvision)
  reference goldens         the pyramid and grid-32 pooling of the reference's own code (tests/golden/efficientnet_pyramid.pt)
  batch-norm folding        folded vs unfolded oracle in float64; fp32 in, fp32 out
  seeded weights            every tap's RMS in [0.1, 10] at 448; deterministic
  checkpoints / arguments   ResNet and EfficientNet-B4 state dicts, B4 / B7 model types, pretrained=True without a
                            checkpoint, segmentation types: ValueError
"""
import os

import pytest
import torch

from oracle import efficientnet as E
from wild_visual_navigation_b200.feature_extractor import weights as W

SHAPES = [(96, 2), (144, 4), (240, 8), (672, 16), (1280, 32)]


@pytest.fixture(scope="module")
def seeded():
    return W.synthetic_efficientnet_b0_state_dict(seed=1)


def _img(S, B=1, seed=0, dtype=torch.float32):
    return torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(seed), dtype=dtype)


@pytest.mark.parametrize("S", [224, 448])
def test_oracle_matches_torchvision(S, seeded):
    tv = pytest.importorskip("torchvision")
    from torchvision.models.feature_extraction import create_feature_extractor

    model = tv.models.efficientnet_b0(weights=None)
    missing, unexpected = model.load_state_dict(seeded, strict=False)
    assert not unexpected and all(k.startswith("classifier.") for k in missing)
    fx = create_feature_extractor(model.eval(), return_nodes=E.TAP_NODES)
    img = _img(S, B=2, seed=S)
    with torch.no_grad():
        want = fx(E.normalize(img))
        got = E.efficientnet_pyramid(img, seeded)
    assert list(got) == [f"feat{i}" for i in range(1, 6)]
    for (c, s), k in zip(SHAPES, want):
        assert got[k].shape == want[k].shape == (2, c, S // s, S // s)
        err = (got[k] - want[k]).abs().max().item()
        assert err <= 1e-5 * max(1.0, want[k].abs().max().item()), (k, err)


def test_oracle_vs_reference_goldens(seeded, golden_dir):
    """tests/golden/efficientnet_pyramid.pt (make_golden_efficientnet.py): the reference's TorchVisionInterface (return
    nodes translated to the block outputs) and sparsify_features on one seeded 448 image with these seeded weights."""
    gold = torch.load(os.path.join(golden_dir, "efficientnet_pyramid.pt"))
    img = _img(448, seed=gold["image_seed"])
    with torch.no_grad():
        pyr = E.efficientnet_pyramid(img, seeded)
    assert list(pyr) == list(gold["shapes"])
    for k, t in pyr.items():
        assert tuple(t.shape) == gold["shapes"][k]
        want = gold["samples"][k]
        assert (t.reshape(-1)[:: gold["stride"]] - want).abs().max().item() <= 1e-5 * max(1.0, want.abs().max().item()), k
        sums = t.double().sum((0, 2, 3))
        assert torch.allclose(sums, gold["channel_sums"][k], rtol=1e-5, atol=1e-3 * t[0, 0].numel() ** 0.5), k
    ys = torch.arange(448) // 32
    feat = E.pool_pyramid(ys[:, None] * 14 + ys[None, :], pyr, 196)
    assert feat.shape == (196, 2432)
    assert torch.allclose(feat[:, :: gold["col_stride"]], gold["grid32_feat"], rtol=1e-5, atol=1e-5)
    # cell_size 16: a segment has no cell on the 14 x 14 level; the reference raises, the centroid rule fills it
    assert gold["grid16_raises"] == "AttributeError"
    ys = torch.arange(448) // 16
    assert torch.isfinite(E.pool_pyramid(ys[:, None] * 28 + ys[None, :], pyr, 784)).all()


def test_folded_oracle_matches_unfolded(seeded):
    sd = {k: v.double() if v.is_floating_point() else v for k, v in seeded.items()}
    folded = W.fold_efficientnet_bn(sd)
    assert all(w.dtype == torch.float64 and b.dtype == torch.float64 for w, b in folded.values())
    img = _img(96, dtype=torch.float64)
    a = E.efficientnet_pyramid(img, sd)
    b = E.efficientnet_pyramid(img, E.folded_state_dict(folded), folded=True)
    for k in a:
        assert ((a[k] - b[k]).abs().max() / a[k].abs().max()).item() <= 1e-10, k
    # fp32 weights fold in fp32, and the fp32 folded trunk stays within fp32 rounding of the unfolded one
    folded32 = W.fold_efficientnet_bn(seeded)
    assert all(w.dtype == torch.float32 for w, _ in folded32.values())
    a32 = E.efficientnet_pyramid(img.float(), seeded)
    b32 = E.efficientnet_pyramid(img.float(), E.folded_state_dict(folded32), folded=True)
    for k in a:
        assert ((a32[k] - b32[k]).norm() / a32[k].norm()).item() <= 1e-5, k


def test_seeded_weights_keep_taps_at_a_realistic_scale(seeded):
    with torch.no_grad():
        pyr = E.efficientnet_pyramid(_img(448, seed=5), seeded)
    for (c, s), t in zip(SHAPES, pyr.values()):
        assert t.shape == (1, c, 448 // s, 448 // s)
        rms = t.pow(2).mean().sqrt().item()
        assert 0.1 <= rms <= 10, (c, rms)
    again = W.synthetic_efficientnet_b0_state_dict(seed=1)
    assert all(torch.equal(again[k], seeded[k]) for k in again)


def test_checkpoint_family_is_checked(seeded, tmp_path):
    from wild_visual_navigation_b200.feature_extractor.weights import synthetic_resnet_state_dict

    with pytest.raises(ValueError, match="got a ResNet state dict"):
        W.check_efficientnet_family(synthetic_resnet_state_dict(18), "efficientnet_b0")
    with pytest.raises(ValueError, match="model_type"):
        W.check_efficientnet_family(seeded, "efficientnet_b4")
    tv = pytest.importorskip("torchvision")
    with pytest.raises(ValueError, match="got an EfficientNet-B4 state dict"):
        W.check_efficientnet_family(tv.models.efficientnet_b4(weights=None).state_dict(), "efficientnet_b0")
    # torchvision's own B0 state dict passes; classifier.* and num_batches_tracked are dropped
    kept = W.check_efficientnet_family(tv.models.efficientnet_b0(weights=None).state_dict(), "efficientnet_b0")
    assert not any(k.startswith("classifier.") or k.endswith("num_batches_tracked") for k in kept)
    assert "features.8.1.running_var" in kept and "features.1.0.block.1.fc2.bias" in kept
    path = tmp_path / "efficientnet_b0.pth"
    torch.save(seeded, path)
    loaded = W.load_efficientnet_state_dict("efficientnet_b0", str(path))
    assert torch.equal(loaded["features.7.0.block.3.0.weight"], seeded["features.7.0.block.3.0.weight"])
    # without a checkpoint: pretrained=False is seeded (torchvision's random init), pretrained=True refuses
    with pytest.warns(UserWarning, match="seeded"):
        again = W.load_efficientnet_state_dict("efficientnet_b0", pretrained=False)
    assert all(torch.equal(again[k], seeded[k]) for k in seeded)
    with pytest.raises(ValueError, match="pretrained=True needs torchvision's ImageNet checkpoint"):
        W.load_efficientnet_state_dict("efficientnet_b0")


def test_efficientnet_arguments_are_checked(monkeypatch):
    from wild_visual_navigation_b200.feature_extractor import FeatureExtractor, TorchVisionInterface

    monkeypatch.delenv("WVN_EFFICIENTNET_WEIGHTS", raising=False)
    for mt in ("efficientnet_b4", "efficientnet_b7"):
        with pytest.raises(ValueError, match="outside the H100 hot path \\(resnet18"):
            TorchVisionInterface("cuda", mt, 448)
    # B0 is built, but its ImageNet weights (pretrained=True, the default) come only from a checkpoint
    with pytest.raises(ValueError, match="pretrained=True needs"):
        TorchVisionInterface("cuda", "efficientnet_b0", 448)
    with pytest.raises(ValueError, match="pretrained=True needs"):
        FeatureExtractor("cuda", segmentation_type="grid", feature_type="torchvision", model_type="efficientnet_b0")
    with pytest.raises(ValueError, match="multiple of 32"):
        TorchVisionInterface("cuda", "efficientnet_b0", pretrained=False)  # the reference's default input_size 488
    for seg in ("random", "none", None):
        with pytest.raises(ValueError, match="torchvision"):
            FeatureExtractor("cuda", segmentation_type=seg, feature_type="torchvision", model_type="efficientnet_b0")
    with pytest.raises(ValueError, match="efficientnet_b0"):
        FeatureExtractor("cuda", segmentation_type="grid", feature_type="torchvision")
