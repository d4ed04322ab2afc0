"""DINOv2 with register tokens on the CPU: the oracle against ``transformers.Dinov2WithRegistersModel`` end to end
(its position-embedding interpolation included: the model gets the 37 x 37 pre-training grid and interpolates itself),
the register models' antialiased interpolation, the synthetic weights and the checkpoint family checks."""
import pytest
import torch
import torch.nn.functional as F

from oracle.dinov2_reg_vit import dinov2_reg_tokens, interpolate_pos_encoding_antialias, synthetic_dinov2_reg_state_dict
from oracle.dinov2_vit import dinov2_config

GPU_REL_L2 = 2e-2   # tests/test_dinov2_reg_gpu.py's token bar


def rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _img(B, S, seed):
    return torch.randn(B, 3, S, S, generator=torch.Generator().manual_seed(seed))


def _attn_std(backbone_type):
    return 0.09 if backbone_type == "vit_small" else 0.09 / 2 ** 0.5


@pytest.mark.parametrize("backbone_type,image_size", [("vit_small", 224), ("vit_small", 448), ("vit_small", 518),
                                                      ("vit_base", 224)])
def test_oracle_matches_transformers_dinov2_with_registers(backbone_type, image_size):
    transformers = pytest.importorskip("transformers")
    cfg = dinov2_config(backbone_type, image_size)
    sd = synthetic_dinov2_reg_state_dict(cfg, seed=3, attn_std=_attn_std(backbone_type))
    R = sd["register_tokens"].shape[1]
    # image_size=518: the model's position embedding is the pre-training grid (37^2 + 1), interpolated by the model
    hc = transformers.Dinov2WithRegistersConfig(
        hidden_size=cfg.dim, num_hidden_layers=cfg.depth, num_attention_heads=cfg.heads,
        mlp_ratio=cfg.mlp_dim // cfg.dim, patch_size=14, image_size=518, num_register_tokens=R, layerscale_value=1.0,
        layer_norm_eps=cfg.ln_eps, hidden_act="gelu", qkv_bias=True, use_swiglu_ffn=False, attn_implementation="eager")
    model = transformers.Dinov2WithRegistersModel(hc).eval().float()
    D = cfg.dim
    m = {"embeddings.cls_token": sd["cls_token"], "embeddings.mask_token": sd["mask_token"],
         "embeddings.register_tokens": sd["register_tokens"], "embeddings.position_embeddings": sd["pos_embed"],
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
    x = _img(2 if image_size <= 448 else 1, image_size, 0)
    with torch.no_grad():
        ref = model(pixel_values=x).last_hidden_state[:, 1 + R:]
    got = dinov2_reg_tokens(x, sd, cfg)
    assert got.shape == ref.shape == (x.shape[0], cfg.grid ** 2, D)
    err = (got - ref).abs().max().item()
    print(f"{backbone_type} @{image_size}: max |oracle - Dinov2WithRegistersModel| = {err:.2e}")
    assert err <= 2e-5


@pytest.mark.parametrize("image_size,grid", [(448, 32), (224, 16), (518, 37)])
def test_register_pos_embed_interpolation(image_size, grid):
    """The register models interpolate with ``size=(g, g)``, bicubic, antialias: the product and the oracle equal
    F.interpolate bit for bit, 518 passes through, and at 448 the result differs from the no-register formula."""
    from wild_visual_navigation_b200.ops import interpolate_pos_embed, interpolate_pos_embed_antialias

    cfg = dinov2_config("vit_small", image_size)
    pe = synthetic_dinov2_reg_state_dict(cfg, seed=5)["pos_embed"]
    ora, prod = interpolate_pos_encoding_antialias(pe, grid, grid), interpolate_pos_embed_antialias(pe, grid)
    if grid == 37:
        assert ora is pe and prod is pe
        return
    patch = pe[:, 1:].reshape(1, 37, 37, 384).permute(0, 3, 1, 2)
    want = F.interpolate(patch, size=(grid, grid), mode="bicubic", align_corners=False, antialias=True)
    want = torch.cat((pe[:, :1], want.permute(0, 2, 3, 1).reshape(1, -1, 384)), dim=1)
    assert ora.shape == (1, 1 + grid * grid, 384)
    assert torch.equal(ora, want) and torch.equal(prod, want)
    if grid == 32:
        diff = (interpolate_pos_embed(pe, grid) - want).abs().max().item()
        print(f"448: max |no-register formula - register formula| = {diff:.2e}")
        assert diff > 1e-3


def test_product_and_oracle_register_weights_identical_and_registers_matter():
    """The product's and the oracle's generators agree bit for bit; zeroing the registers, dropping them, or giving
    them pos[0] moves the ViT-S/14 tokens at 224 by several times the GPU token bar."""
    from wild_visual_navigation_b200.feature_extractor.weights import synthetic_dinov2_reg_state_dict as product_sd

    for backbone_type, dim, mlp in (("vit_small", 384, 1536), ("vit_base", 768, 3072)):
        a = synthetic_dinov2_reg_state_dict(dinov2_config(backbone_type), seed=7, attn_std=0.05)
        b = product_sd(dim, 12, mlp, seed=7, attn_std=0.05)
        assert a.keys() == b.keys() and a["register_tokens"].shape == (1, 4, dim)
        assert all(torch.equal(a[k], b[k]) for k in a)
    cfg = dinov2_config("vit_small", 224)
    sd = synthetic_dinov2_reg_state_dict(cfg, seed=3)
    x = _img(1, 224, 0)
    ref = dinov2_reg_tokens(x, sd, cfg)
    zeroed = dict(sd, register_tokens=torch.zeros_like(sd["register_tokens"]))
    with_pos = dict(sd, register_tokens=sd["register_tokens"] + sd["pos_embed"][:, :1])
    dropped = dict(sd, register_tokens=sd["register_tokens"][:, :0])
    moved = {name: rel_l2(dinov2_reg_tokens(x, s, cfg), ref) for name, s in
             (("zeroed", zeroed), ("pos0", with_pos), ("dropped", dropped))}
    print("rel-L2 moves at 224:", {k: f"{v:.3f}" for k, v in moved.items()})
    assert min(moved.values()) > 3 * GPU_REL_L2


def test_without_registers_is_dinov2():
    """Zero register tokens: the register oracle is the DINOv2 oracle at the pre-training grid (where the two
    interpolations both pass through), to the last bit."""
    from oracle.dinov2_vit import dinov2_tokens

    cfg = dinov2_config("vit_small", 518)
    cfg.depth = 2
    sd = synthetic_dinov2_reg_state_dict(cfg, seed=2)
    x = _img(1, 518, 3)
    assert torch.equal(dinov2_reg_tokens(x, dict(sd, register_tokens=sd["register_tokens"][:, :0]), cfg),
                       dinov2_tokens(x, sd, cfg))


# ------------------------------------------------------------------------------------------------ checkpoint loading
def _reg(seed=1, dim=384, mlp=1536):
    from wild_visual_navigation_b200.feature_extractor.weights import synthetic_dinov2_reg_state_dict as product_sd

    return product_sd(dim, 12, mlp, seed=seed)


@pytest.mark.parametrize("prefix", ["", "backbone.", "module."])
def test_dinov2_reg_checkpoint_loading(tmp_path, prefix):
    from wild_visual_navigation_b200.feature_extractor.weights import check_backbone_family, load_dino_state_dict

    sd = _reg()
    out = check_backbone_family({prefix + k: v for k, v in sd.items()}, "dinov2_reg")
    assert out.keys() == sd.keys() - {"mask_token"} and out["register_tokens"].shape == (1, 4, 384)
    path = tmp_path / "dinov2_vits14_reg4_pretrain.pth"
    torch.save({prefix + k: v for k, v in sd.items()}, path)
    loaded = load_dino_state_dict("vit_small", 8, str(path), backbone="dinov2_reg")
    assert loaded.keys() == out.keys() and torch.equal(loaded["register_tokens"], sd["register_tokens"])


def test_register_count_is_read_from_the_checkpoint():
    from wild_visual_navigation_b200.feature_extractor.weights import synthetic_dinov2_reg_state_dict as product_sd

    sd = product_sd(384, 2, 1536, seed=1, registers=2)
    assert sd["register_tokens"].shape == (1, 2, 384)
    cfg = dinov2_config("vit_small", 224)
    cfg.depth = 2
    tok = dinov2_reg_tokens(_img(1, 224, 1), sd, cfg)
    assert tok.shape == (1, 256, 384)


def test_wrong_family_raises_both_ways(tmp_path):
    from wild_visual_navigation_b200.feature_extractor.weights import (check_backbone_family, load_dino_state_dict,
                                                                      synthetic_dino_state_dict,
                                                                      synthetic_dinov2_state_dict)

    reg, v2 = _reg(), synthetic_dinov2_state_dict(384, 12, 1536)
    with pytest.raises(ValueError, match="register tokens") as e:
        check_backbone_family(reg, "dinov2")
    assert "backbone='dinov2_reg'" in str(e.value)
    with pytest.raises(ValueError, match="register_tokens"):
        check_backbone_family(v2, "dinov2_reg")
    with pytest.raises(ValueError, match="backbone 'dino'"):
        check_backbone_family(reg, "dino")
    with pytest.raises(ValueError, match="backbone 'dino'"):
        check_backbone_family(v2, "dino")
    v1 = synthetic_dino_state_dict(384, 12, 1536, 8, 28)
    with pytest.raises(ValueError, match="DINOv2 checkpoint"):
        check_backbone_family(v1, "dinov2_reg")
    v1_reg = dict(synthetic_dino_state_dict(384, 12, 1536, 14, 16), register_tokens=torch.zeros(1, 4, 384))
    with pytest.raises(ValueError, match="DINOv2 checkpoint"):          # registers but no LayerScale
        check_backbone_family(v1_reg, "dinov2_reg")
    path = tmp_path / "dinov2_vits14_pretrain.pth"
    torch.save(v2, path)
    with pytest.raises(ValueError):
        load_dino_state_dict("vit_small", 14, str(path), backbone="dinov2_reg")


def test_synthetic_dinov2_reg_default_geometry():
    from wild_visual_navigation_b200.feature_extractor.weights import load_dino_state_dict

    with pytest.warns(UserWarning, match="DINOV2_REG"):
        sd = load_dino_state_dict("vit_base", 8, None, backbone="dinov2_reg")
    assert sd["patch_embed.proj.weight"].shape == (768, 3, 14, 14) and sd["register_tokens"].shape == (1, 4, 768)
    assert sd["pos_embed"].shape == (1, 1 + 37 * 37, 768) and "blocks.11.ls1.gamma" in sd
