"""CPU tests of the torchvision ResNet feature backbone's oracle, weights and argument checks.

  oracle vs torchvision     resnet18 / resnet50 behind create_feature_extractor with the reference's return nodes,
                            seeded weights, within 1e-5 (skipped without torchvision)
  batch-norm folding        folded vs unfolded oracle within 1e-6 in float64
  seeded weights            every tap's RMS in [0.1, 10] at 448
  checkpoints / arguments   wrong family, model_type, input_size, segmentation types: ValueError
  missing segments          hand-built cases of the centroid rule of oracle.resnet.pool_pyramid
  reference goldens         pyramids and grid-32 pooling of the reference's own code (tests/golden/resnet_pyramid.pt)
"""
import warnings

import pytest
import torch

from oracle import resnet as R
from wild_visual_navigation_b200.feature_extractor import weights as W

RETURN_NODES = {
    18: {"layer1.1.relu_1": "feat1", "layer2.1.relu_1": "feat2", "layer3.1.relu_1": "feat3", "layer4.1.relu_1": "feat4"},
    50: {"layer2.0.relu": "feat1", "layer3.0.relu": "feat2", "layer4.0.relu": "feat3", "layer4.2.relu_2": "feat4"},
}
SHAPES = {18: [(64, 4), (128, 8), (256, 16), (512, 32)], 50: [(128, 4), (256, 8), (512, 16), (2048, 32)]}


@pytest.fixture(scope="module")
def seeded():
    return {d: W.synthetic_resnet_state_dict(d, seed=1) for d in (18, 50)}


def _img(S, B=1, seed=0, dtype=torch.float32):
    return torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(seed), dtype=dtype)


@pytest.mark.parametrize("depth", [18, 50])
def test_oracle_matches_torchvision(depth, seeded):
    tv = pytest.importorskip("torchvision")
    from torchvision.models.feature_extraction import create_feature_extractor

    model = getattr(tv.models, f"resnet{depth}")(weights=None)
    missing, unexpected = model.load_state_dict(seeded[depth], strict=False)
    assert not unexpected and all(k.startswith("fc.") for k in missing)
    fx = create_feature_extractor(model.eval(), return_nodes=RETURN_NODES[depth])
    img = _img(224, B=2)
    mean = torch.tensor(R.MEAN)[:, None, None]
    std = torch.tensor(R.STD)[:, None, None]
    with torch.no_grad():
        want = fx((img - mean) / std)
        got = R.resnet_pyramid(img, seeded[depth], depth)
    assert list(got) == ["feat1", "feat2", "feat3", "feat4"]
    for k in want:
        assert got[k].shape == want[k].shape
        err = (got[k] - want[k]).abs().max().item()
        assert err <= 1e-5 * max(1.0, want[k].abs().max().item()), (k, err)


@pytest.mark.parametrize("depth", [18, 50])
def test_folded_oracle_matches_unfolded_in_float64(depth, seeded):
    sd = {k: v.double() if v.is_floating_point() else v for k, v in seeded[depth].items()}
    folded = {}
    for name, (w, b) in W.fold_resnet_bn(sd, depth).items():
        assert w.dtype == torch.float64
        folded[name + ".weight"], folded[name + ".bias"] = w, b
    img = _img(96, dtype=torch.float64)
    a = R.resnet_pyramid(img, sd, depth)
    b = R.resnet_pyramid(img, folded, depth, folded=True)
    for k in a:
        assert ((a[k] - b[k]).abs().max() / a[k].abs().max()).item() <= 1e-6, k


@pytest.mark.parametrize("depth", [18, 50])
def test_seeded_weights_keep_taps_at_a_realistic_scale(depth, seeded):
    with torch.no_grad():
        pyr = R.resnet_pyramid(_img(448, seed=5), seeded[depth], depth)
    for (c, s), t in zip(SHAPES[depth], pyr.values()):
        assert t.shape == (1, c, 448 // s, 448 // s)
        rms = t.pow(2).mean().sqrt().item()
        assert 0.1 <= rms <= 10, (depth, c, rms)
    # the generator is deterministic
    again = W.synthetic_resnet_state_dict(depth, seed=1)
    assert all(torch.equal(again[k], seeded[depth][k]) for k in again)


def test_checkpoint_family_is_checked(seeded, tmp_path):
    with pytest.raises(ValueError, match="ResNet-50"):
        W.check_resnet_family(seeded[18], "resnet50")
    with pytest.raises(ValueError, match="ResNet-18"):
        W.check_resnet_family(seeded[50], "resnet18")
    with pytest.raises(ValueError, match="model_type"):
        W.check_resnet_family(seeded[50], "efficientnet_b0")
    # fc.* is optional (strict=False), num_batches_tracked is ignored; DINO's resnet50 checkpoint has no fc
    sd = dict(seeded[50], **{"fc.weight": torch.zeros(1000, 2048), "fc.bias": torch.zeros(1000)})
    kept = W.check_resnet_family(sd, "resnet50_dino")
    assert "fc.weight" not in kept and "conv1.weight" in kept and "bn1.running_var" in kept
    path = tmp_path / "dino_resnet50_pretrain.pth"
    torch.save(seeded[50], path)
    loaded = W.load_resnet_state_dict("resnet50_dino", str(path))
    assert torch.equal(loaded["layer4.2.conv3.weight"], seeded[50]["layer4.2.conv3.weight"])
    with pytest.raises(ValueError):
        W.load_resnet_state_dict("resnet18", str(path))
    with pytest.warns(UserWarning, match="seeded"):
        W.load_resnet_state_dict("resnet18")


def test_interface_and_extractor_arguments_are_checked():
    from wild_visual_navigation_b200.feature_extractor import FeatureExtractor, TorchVisionInterface

    with pytest.raises(ValueError, match="outside the H100 hot path"):
        TorchVisionInterface("cuda", "efficientnet_b0", 448)
    with pytest.raises(ValueError, match="multiple of 32"):
        TorchVisionInterface("cuda", "resnet18")  # the reference's default input_size 488
    for seg in ("random", "none", None):
        with pytest.raises(ValueError, match="torchvision"):
            FeatureExtractor("cuda", segmentation_type=seg, feature_type="torchvision", model_type="resnet18")
    with pytest.raises(ValueError, match="model_type"):
        FeatureExtractor("cuda", segmentation_type="grid", feature_type="torchvision")


def _pyramid(S, channels=(2, 3, 4, 5), seed=0):
    g = torch.Generator().manual_seed(seed)
    return {f"feat{i + 1}": torch.randn(1, c, S // s, S // s, generator=g, dtype=torch.float64)
            for i, (c, s) in enumerate(zip(channels, (4, 8, 16, 32)))}


def test_pool_pyramid_means_over_downsampled_segments():
    S = 64
    seg = (torch.arange(S)[:, None] // 32) * 2 + torch.arange(S)[None, :] // 32  # grid-32: present at every level
    pyr = _pyramid(S)
    got = R.pool_pyramid(seg, pyr, 4)
    for s in range(4):
        r, c = divmod(s, 2)
        want = torch.cat([f[0, :, r * f.shape[2] // 2:(r + 1) * f.shape[2] // 2,
                                c * f.shape[3] // 2:(c + 1) * f.shape[3] // 2].mean((1, 2)) for f in pyr.values()])
        assert torch.allclose(got[s], want, rtol=0, atol=1e-12)


def test_pool_pyramid_missing_segment_takes_the_centroid_cell():
    S = 64
    seg = torch.zeros(S, S, dtype=torch.int64)
    # segment 1: a 3 x 3 block at rows 41..43, cols 9..11 — the finest level samples rows / cols 40 and 44, so it is
    # missing from every level; its centroid is (col 10, row 42)
    seg[41:44, 9:12] = 1
    # segment 2: rows 0..63 at col 1 — sampled by no level (they sample cols 0, 4, 8, ...), centroid (1, 31.5)
    seg[:, 1] = 2
    pyr = _pyramid(S)
    got = R.pool_pyramid(seg, pyr, 4)
    for s, (cx, cy) in ((1, (10.0, 42.0)), (2, (1.0, 31.5))):
        want = torch.cat([f[0, :, min(int(cy // (S // f.shape[2])), f.shape[2] - 1),
                            min(int(cx // (S // f.shape[3])), f.shape[3] - 1)] for f in pyr.values()])
        assert torch.equal(got[s], want), s
    # ids 3 (absent from the frame) get a NaN row, as the plain pooling's empty segments do
    assert torch.isnan(got[3]).all()
    # segment 0 is present everywhere: its level-4 feature is the mean over the 2 x 2 cells it owns
    lvl4 = pyr["feat4"][0]
    assert torch.allclose(got[0, -5:], lvl4.reshape(5, -1).mean(1))


@pytest.mark.parametrize("depth", [18, 50])
def test_oracle_vs_reference_goldens(depth, seeded, golden_dir):
    """tests/golden/resnet_pyramid.pt (make_golden_resnet.py): the reference's TorchVisionInterface and
    sparsify_features on one seeded 448 image with these seeded weights."""
    import os

    gold = torch.load(os.path.join(golden_dir, "resnet_pyramid.pt"))
    ref = gold[f"resnet{depth}"]
    img = _img(448, seed=gold["image_seed"])
    with torch.no_grad():
        pyr = R.resnet_pyramid(img, seeded[depth], depth)
    for k, t in pyr.items():
        assert tuple(t.shape) == ref["shapes"][k]
        want = ref["samples"][k]
        assert (t.reshape(-1)[:: gold["stride"]] - want).abs().max().item() <= 1e-5 * max(1.0, want.abs().max().item()), k
        sums = t.double().sum((0, 2, 3))
        assert torch.allclose(sums, ref["channel_sums"][k], rtol=1e-5, atol=1e-3 * t[0, 0].numel() ** 0.5), k
    ys = torch.arange(448) // 32
    feat = R.pool_pyramid(ys[:, None] * 14 + ys[None, :], pyr, 196)
    assert torch.allclose(feat[:, :: gold["col_stride"]], ref["grid32_feat"], rtol=1e-5, atol=1e-5)
    # cell_size 16: a segment has no cell on the 14 x 14 level; the reference raises, the centroid rule fills it
    assert ref["grid16_raises"] == "AttributeError"
    ys = torch.arange(448) // 16
    feat16 = R.pool_pyramid(ys[:, None] * 28 + ys[None, :], pyr, 784)
    assert torch.isfinite(feat16).all()
