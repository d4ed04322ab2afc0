"""DINOv2 on the CPU: the oracle's restatement against ``transformers.Dinov2Model``, the position-embedding
interpolation, the synthetic weights, the LayerScale fold and the checkpoint family checks.

``transformers`` interpolates position embeddings with ``size=`` rather than DINOv2's ``scale_factor`` form, so the
cross-check hands it embeddings already at the target grid, and the interpolation is held to the recalled formula
on its own (``test_dinov2_pos_embed_interpolation``)."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle.dino_vit import ViTConfig, interpolate_pos_encoding, synthetic_state_dict
from oracle.dinov2_vit import dinov2_config, dinov2_tokens, synthetic_dinov2_state_dict


def rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _img(B, S, seed):
    return torch.randn(B, 3, S, S, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("backbone_type,image_size", [("vit_small", 224), ("vit_small", 448), ("vit_base", 224)])
def test_oracle_matches_transformers_dinov2(backbone_type, image_size):
    transformers = pytest.importorskip("transformers")
    cfg = dinov2_config(backbone_type, image_size)
    sd = synthetic_dinov2_state_dict(cfg, seed=3, attn_std=0.09 if backbone_type == "vit_small" else 0.09 / 2 ** 0.5)
    hc = transformers.Dinov2Config(hidden_size=cfg.dim, num_hidden_layers=cfg.depth, num_attention_heads=cfg.heads,
                                   mlp_ratio=cfg.mlp_dim // cfg.dim, patch_size=14, image_size=image_size,
                                   layerscale_value=1.0, layer_norm_eps=cfg.ln_eps, hidden_act="gelu", qkv_bias=True,
                                   use_swiglu_ffn=False, attn_implementation="eager")
    model = transformers.Dinov2Model(hc).eval()
    D = cfg.dim
    m = {"embeddings.cls_token": sd["cls_token"], "embeddings.mask_token": sd["mask_token"],
         "embeddings.position_embeddings": interpolate_pos_encoding(sd["pos_embed"], cfg.grid, cfg.grid),
         "embeddings.patch_embeddings.projection.weight": sd["patch_embed.proj.weight"],
         "embeddings.patch_embeddings.projection.bias": sd["patch_embed.proj.bias"],
         "layernorm.weight": sd["norm.weight"], "layernorm.bias": sd["norm.bias"]}
    for i in range(cfg.depth):
        s, d = f"blocks.{i}.", f"encoder.layer.{i}."
        for leaf in ("norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias", "mlp.fc1.weight", "mlp.fc1.bias",
                     "mlp.fc2.weight", "mlp.fc2.bias"):
            m[d + leaf] = sd[s + leaf]
        for j, name in enumerate(("query", "key", "value")):
            m[d + f"attention.attention.{name}.weight"] = sd[s + "attn.qkv.weight"][j * D:(j + 1) * D]
            m[d + f"attention.attention.{name}.bias"] = sd[s + "attn.qkv.bias"][j * D:(j + 1) * D]
        m[d + "attention.output.dense.weight"] = sd[s + "attn.proj.weight"]
        m[d + "attention.output.dense.bias"] = sd[s + "attn.proj.bias"]
        m[d + "layer_scale1.lambda1"] = sd[s + "ls1.gamma"]
        m[d + "layer_scale2.lambda1"] = sd[s + "ls2.gamma"]
    model.load_state_dict(m, strict=True)
    x = _img(2, image_size, 0)
    with torch.no_grad():
        ref = model(pixel_values=x).last_hidden_state[:, 1:]
    got = dinov2_tokens(x, sd, cfg)
    assert got.shape == (2, cfg.grid ** 2, D)
    err = (got - ref).abs().max().item()
    print(f"{backbone_type} @{image_size}: max |oracle - Dinov2Model| = {err:.2e}")
    assert err <= 2e-5


@pytest.mark.parametrize("image_size,grid", [(448, 32), (224, 16), (518, 37)])
def test_dinov2_pos_embed_interpolation(image_size, grid):
    """DINOv2's interpolate_pos_encoding: bicubic with scale_factor ((g + 0.1) / 37, (g + 0.1) / 37), no antialias,
    from the 37 x 37 pre-training grid; the oracle and the product both follow it, and 518 passes through."""
    from wild_visual_navigation_b200.ops import interpolate_pos_embed

    cfg = dinov2_config("vit_small", image_size)
    assert cfg.grid == grid and cfg.pretrain_grid == 37
    pe = synthetic_dinov2_state_dict(cfg, seed=5)["pos_embed"]
    assert pe.shape == (1, 1 + 37 * 37, 384)
    ora, prod = interpolate_pos_encoding(pe, grid, grid), interpolate_pos_embed(pe, grid)
    if grid == 37:
        assert ora is pe and prod is pe
        return
    patch = pe[:, 1:].reshape(1, 37, 37, 384).permute(0, 3, 1, 2)
    s = (grid + 0.1) / 37
    want = F.interpolate(patch, scale_factor=(s, s), mode="bicubic", align_corners=False, antialias=False)
    want = torch.cat((pe[:, :1], want.permute(0, 2, 3, 1).reshape(1, -1, 384)), dim=1)
    assert ora.shape == (1, 1 + grid * grid, 384)
    assert torch.equal(ora, want) and torch.equal(prod, want)


def test_product_and_oracle_synthetic_weights_identical():
    from wild_visual_navigation_b200.feature_extractor.weights import synthetic_dinov2_state_dict as product_sd

    for backbone_type, dim, mlp in (("vit_small", 384, 1536), ("vit_base", 768, 3072)):
        a = synthetic_dinov2_state_dict(dinov2_config(backbone_type), seed=7, attn_std=0.05)
        b = product_sd(dim, 12, mlp, seed=7, attn_std=0.05)
        assert a.keys() == b.keys()
        assert all(torch.equal(a[k], b[k]) for k in a)
    g1, g2 = a["blocks.0.ls1.gamma"], a["blocks.0.ls2.gamma"]
    assert g1.std() > 0.1 and g2.std() > 0.1 and (g1 - g2).abs().mean() > 0.1   # per channel, and ls1 != ls2


def test_layerscale_fold_matches_unfolded_oracle_and_a_swap_does_not():
    """The product's fold (gammas into proj / fc2 rows and biases) run through the oracle without LayerScale equals
    the oracle with LayerScale within 1e-6 (in float64, so that only the algebra is compared: in fp32 the two orders
    of rounding alone differ by about 1e-6 rel-L2 after 12 blocks); folding ls1 and ls2 the wrong way round, or not
    at all, moves the tokens far beyond the 2e-2 GPU parity tolerance (so the parity tests can see either mistake)."""
    from wild_visual_navigation_b200.ops import fold_layerscale

    cfg = dinov2_config("vit_small", 224)
    sd = synthetic_dinov2_state_dict(cfg, seed=1)
    x = _img(1, 224, 1)
    sd64 = {k: v.double() for k, v in sd.items()}
    ref64 = dinov2_tokens(x.double(), sd64, cfg)
    folded = fold_layerscale(sd64, cfg.depth)
    assert not any("gamma" in k for k in folded)
    err = (dinov2_tokens(x.double(), folded, cfg) - ref64).abs().max().item()
    assert err <= 1e-6, err
    ref = dinov2_tokens(x, sd, cfg)
    assert rel_l2(dinov2_tokens(x, fold_layerscale(sd, cfg.depth), cfg), ref) <= 1e-5
    swapped = dict(sd)
    for i in range(cfg.depth):
        swapped[f"blocks.{i}.ls1.gamma"], swapped[f"blocks.{i}.ls2.gamma"] = sd[f"blocks.{i}.ls2.gamma"], sd[f"blocks.{i}.ls1.gamma"]
    assert rel_l2(dinov2_tokens(x, fold_layerscale(swapped, cfg.depth), cfg), ref) > 0.1
    plain = {k: v for k, v in sd.items() if "gamma" not in k}
    assert rel_l2(dinov2_tokens(x, plain, cfg), ref) > 0.1


def test_dino_v1_state_dict_without_layerscale():
    """A DINO v1 state dict has no gammas: the fold leaves it as it is, and the DINOv2 oracle's block is then DINO's
    (oracle/dino_vit.py) to the last bit."""
    from oracle.dino_vit import vit_tokens
    from wild_visual_navigation_b200.ops import fold_layerscale

    cfg = ViTConfig(image_size=64, patch_size=8, dim=64, depth=2, heads=1, mlp_dim=128, pretrain_grid=8)
    sd = synthetic_state_dict(cfg, seed=2)
    assert fold_layerscale(sd, cfg.depth) is sd
    x = _img(2, 64, 3)
    assert torch.equal(dinov2_tokens(x, sd, cfg), vit_tokens(x, sd, cfg))


# ------------------------------------------------------------------------------------------------ checkpoint loading
def _v2(seed=1):
    from wild_visual_navigation_b200.feature_extractor.weights import synthetic_dinov2_state_dict as product_sd

    return product_sd(384, 12, 1536, seed=seed)


def test_dinov2_checkpoint_drops_mask_token(tmp_path):
    from wild_visual_navigation_b200.feature_extractor.weights import check_backbone_family, load_dino_state_dict

    sd = _v2()
    out = check_backbone_family({"backbone." + k: v for k, v in sd.items()}, "dinov2")
    assert "mask_token" not in out and "blocks.11.ls2.gamma" in out and out.keys() == sd.keys() - {"mask_token"}
    path = tmp_path / "dinov2_vits14_pretrain.pth"
    torch.save(sd, path)
    loaded = load_dino_state_dict("vit_small", 8, str(path), backbone="dinov2")
    assert loaded.keys() == out.keys() and torch.equal(loaded["pos_embed"], sd["pos_embed"])


def test_register_tokens_and_wrong_family_raise(tmp_path):
    from wild_visual_navigation_b200.feature_extractor.weights import (check_backbone_family, load_dino_state_dict,
                                                                      synthetic_dino_state_dict)

    reg = dict(_v2(), register_tokens=torch.zeros(1, 4, 384))
    with pytest.raises(ValueError, match="register tokens"):
        check_backbone_family(reg, "dinov2")
    v1 = synthetic_dino_state_dict(384, 12, 1536, 8, 28)
    with pytest.raises(ValueError, match="DINOv2 checkpoint"):
        check_backbone_family(v1, "dinov2")
    v1_14 = synthetic_dino_state_dict(384, 12, 1536, 14, 16)      # patch 14 but no LayerScale
    with pytest.raises(ValueError, match="DINOv2 checkpoint"):
        check_backbone_family(v1_14, "dinov2")
    with pytest.raises(ValueError, match="backbone='dinov2'"):
        check_backbone_family(_v2(), "dino")
    assert check_backbone_family(v1, "dino").keys() == v1.keys()
    path = tmp_path / "dino_deitsmall8_pretrain.pth"
    torch.save(v1, path)
    with pytest.raises(ValueError):
        load_dino_state_dict("vit_small", 14, str(path), backbone="dinov2")


def test_synthetic_dinov2_default_geometry():
    from wild_visual_navigation_b200.feature_extractor.weights import load_dino_state_dict

    with pytest.warns(UserWarning, match="DINOV2"):
        sd = load_dino_state_dict("vit_base", 8, None, backbone="dinov2")
    assert sd["patch_embed.proj.weight"].shape == (768, 3, 14, 14)
    assert sd["pos_embed"].shape == (1, 1 + 37 * 37, 768) and "blocks.11.ls1.gamma" in sd
    assert math.isclose(float(sd["blocks.0.ls1.gamma"].min()), 0.1, abs_tol=0.05)
