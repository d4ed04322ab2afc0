"""DINOv2 ViT-L/14 (``backbone_type="vit_large"``: D = 1024, 24 blocks, 16 heads, MLP 4096, erf-GELU) on the CPU.

  oracle            ``oracle/dinov2_vit.py`` / ``oracle/dinov2_reg_vit.py`` at the ViT-L/14 configuration (built from
                    ``VIT_SHAPES["vit_large"]``) against ``transformers.Dinov2Model`` /
                    ``Dinov2WithRegistersModel`` with 1024 hidden, 24 layers and 16 heads, at the ViT-S/B bar (2e-5)
  seeded weights    the product's ``vit_large`` dicts (plain and ``_reg``): shapes, key names, identical to the oracle's
  size checks       a ViT-S or ViT-B checkpoint given for ``vit_large``, or the reverse, raises naming both sizes
  DINO v1           ``backbone="dino"`` has no ViT-L and refuses ``vit_large``
  FeatureExtractor  ``feature_dim`` 1024, and the ``stego_backbone_type`` checks
"""
import pytest
import torch

from oracle.dino_vit import ViTConfig
from oracle.dinov2_reg_vit import dinov2_reg_tokens, synthetic_dinov2_reg_state_dict
from oracle.dinov2_vit import PATCH, PRETRAIN_GRID, dinov2_tokens, synthetic_dinov2_state_dict
from wild_visual_navigation_b200.feature_extractor import weights as W

# qkv std that keeps the attention logits' spread of the ViT-S/B tests (it scales with D)
ATTN_STD = 0.09 * (384 / 1024) ** 0.5


def large_config(image_size):
    s = W.VIT_SHAPES["vit_large"]
    return ViTConfig(image_size, PATCH, s["dim"], s["depth"], s["heads"], s["mlp_dim"], PRETRAIN_GRID)


def _img(B, S, seed):
    return torch.randn(B, 3, S, S, generator=torch.Generator().manual_seed(seed))


def _hf_layers(sd, cfg):
    D = cfg.dim
    m = {"embeddings.cls_token": sd["cls_token"], "embeddings.mask_token": sd["mask_token"],
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
    return m


def _hf_kwargs(cfg):
    return dict(hidden_size=cfg.dim, num_hidden_layers=cfg.depth, num_attention_heads=cfg.heads,
                mlp_ratio=cfg.mlp_dim // cfg.dim, patch_size=14, layerscale_value=1.0, layer_norm_eps=cfg.ln_eps,
                hidden_act="gelu", qkv_bias=True, use_swiglu_ffn=False, attn_implementation="eager")


def test_oracle_matches_transformers_dinov2_large():
    transformers = pytest.importorskip("transformers")
    from oracle.dino_vit import interpolate_pos_encoding

    cfg = large_config(224)
    sd = synthetic_dinov2_state_dict(cfg, seed=3, attn_std=ATTN_STD)
    model = transformers.Dinov2Model(transformers.Dinov2Config(image_size=224, **_hf_kwargs(cfg))).eval()
    assert (model.config.hidden_size, model.config.num_hidden_layers, model.config.num_attention_heads) == (1024, 24, 16)
    m = _hf_layers(sd, cfg)
    # transformers interpolates with size=, so it gets the embeddings already at the grid (as test_dinov2_oracle.py)
    m["embeddings.position_embeddings"] = interpolate_pos_encoding(sd["pos_embed"], cfg.grid, cfg.grid)
    model.load_state_dict(m, strict=True)
    x = _img(2, 224, 0)
    with torch.no_grad():
        ref = model(pixel_values=x).last_hidden_state[:, 1:]
    got = dinov2_tokens(x, sd, cfg)
    assert got.shape == (2, 256, 1024)
    err = (got - ref).abs().max().item()
    print(f"vit_large @224: max |oracle - Dinov2Model| = {err:.2e}")
    assert err <= 2e-5


def test_oracle_matches_transformers_dinov2_large_with_registers():
    """End to end, the register models' antialiased interpolation included (the model gets the 37 x 37 grid)."""
    transformers = pytest.importorskip("transformers")
    cfg = large_config(224)
    sd = synthetic_dinov2_reg_state_dict(cfg, seed=3, attn_std=ATTN_STD)
    hc = transformers.Dinov2WithRegistersConfig(image_size=518, num_register_tokens=4, **_hf_kwargs(cfg))
    model = transformers.Dinov2WithRegistersModel(hc).eval().float()
    m = dict(_hf_layers(sd, cfg), **{"embeddings.register_tokens": sd["register_tokens"],
                                     "embeddings.position_embeddings": sd["pos_embed"]})
    model.load_state_dict(m, strict=True)
    x = _img(2, 224, 0)
    with torch.no_grad():
        ref = model(pixel_values=x).last_hidden_state[:, 5:]
    got = dinov2_reg_tokens(x, sd, cfg)
    assert got.shape == ref.shape == (2, 256, 1024)
    err = (got - ref).abs().max().item()
    print(f"vit_large-reg @224: max |oracle - Dinov2WithRegistersModel| = {err:.2e}")
    assert err <= 2e-5


# ------------------------------------------------------------------------------------------------ seeded weights
@pytest.fixture(scope="module")
def large_sds():
    s = W.VIT_SHAPES["vit_large"]
    return (W.synthetic_dinov2_state_dict(s["dim"], s["depth"], s["mlp_dim"], seed=7, attn_std=0.05),
            W.synthetic_dinov2_reg_state_dict(s["dim"], s["depth"], s["mlp_dim"], seed=7, attn_std=0.05))


def test_vit_large_shape():
    assert W.VIT_SHAPES["vit_large"] == dict(dim=1024, depth=24, heads=16, mlp_dim=4096)


def test_seeded_vit_large_dicts(large_sds):
    """Same key layout as ViT-S/B (24 blocks), ViT-L/14 shapes, and bit-identical to the oracle's generators."""
    v2, reg = large_sds
    small = W.synthetic_dinov2_state_dict(384, 12, 1536, seed=7)
    blocks = lambda sd: {k.split(".", 2)[2] for k in sd if k.startswith("blocks.")}  # noqa: E731
    assert blocks(v2) == blocks(small)
    assert {k for k in v2 if not k.startswith("blocks.")} == {k for k in small if not k.startswith("blocks.")}
    assert {int(k.split(".")[1]) for k in v2 if k.startswith("blocks.")} == set(range(24))
    assert reg.keys() == v2.keys() | {"register_tokens"}
    shapes = {"cls_token": (1, 1, 1024), "pos_embed": (1, 1 + 37 * 37, 1024), "mask_token": (1, 1024),
              "patch_embed.proj.weight": (1024, 3, 14, 14), "patch_embed.proj.bias": (1024,),
              "norm.weight": (1024,), "norm.bias": (1024,), "blocks.23.attn.qkv.weight": (3072, 1024),
              "blocks.23.attn.qkv.bias": (3072,), "blocks.23.attn.proj.weight": (1024, 1024),
              "blocks.23.mlp.fc1.weight": (4096, 1024), "blocks.23.mlp.fc1.bias": (4096,),
              "blocks.23.mlp.fc2.weight": (1024, 4096), "blocks.23.ls1.gamma": (1024,), "blocks.23.ls2.gamma": (1024,)}
    for k, shp in shapes.items():
        assert tuple(v2[k].shape) == shp and tuple(reg[k].shape) == shp, k
    assert tuple(reg["register_tokens"].shape) == (1, 4, 1024)
    cfg = large_config(448)
    for ours, theirs in ((v2, synthetic_dinov2_state_dict(cfg, seed=7, attn_std=0.05)),
                         (reg, synthetic_dinov2_reg_state_dict(cfg, seed=7, attn_std=0.05))):
        assert ours.keys() == theirs.keys() and all(torch.equal(ours[k], theirs[k]) for k in ours)


def test_seeded_default_geometry():
    with pytest.warns(UserWarning, match="DINOV2_REG"):
        sd = W.load_dino_state_dict("vit_large", 8, None, backbone="dinov2_reg")
    assert sd["patch_embed.proj.weight"].shape == (1024, 3, 14, 14) and sd["register_tokens"].shape == (1, 4, 1024)
    assert "blocks.23.ls2.gamma" in sd and "blocks.24.norm1.weight" not in sd


# ------------------------------------------------------------------------------------------------ size checks
def test_size_checks_both_ways(large_sds, tmp_path):
    v2, reg = large_sds
    small = W.synthetic_dinov2_state_dict(384, 12, 1536, seed=1)
    base_reg = W.synthetic_dinov2_reg_state_dict(768, 12, 3072, seed=1)
    assert W.check_backbone_family(v2, "dinov2", "vit_large").keys() == v2.keys() - {"mask_token"}
    assert W.check_backbone_family(reg, "dinov2_reg", "vit_large").keys() == reg.keys() - {"mask_token"}
    cases = [(small, "dinov2", "vit_large", "vit_small"), (base_reg, "dinov2_reg", "vit_large", "vit_base"),
             (v2, "dinov2", "vit_small", "vit_large"), (reg, "dinov2_reg", "vit_base", "vit_large")]
    for sd, backbone, want, got in cases:
        with pytest.raises(ValueError) as e:
            W.check_backbone_family(sd, backbone, want)
        msg = str(e.value)
        assert f"'{want}'" in msg and got in msg, msg
    # 1024 wide but 12 blocks deep: named by its width and depth
    shallow = {k: v for k, v in v2.items() if not k.startswith("blocks.") or int(k.split(".")[1]) < 12}
    with pytest.raises(ValueError, match="D = 1024 with 12 blocks"):
        W.check_backbone_family(shallow, "dinov2", "vit_large")
    # the checkpoint route checks the size too
    path = tmp_path / "dinov2_vits14_pretrain.pth"
    torch.save(small, path)
    with pytest.raises(ValueError, match="vit_small"):
        W.load_dino_state_dict("vit_large", 14, str(path), backbone="dinov2")


def test_dino_v1_has_no_vit_large():
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    with pytest.raises(ValueError, match="backbone 'dino' has no 'vit_large'"):
        W.load_dino_state_dict("vit_large", 8, None, backbone="dino")
    with pytest.raises(ValueError, match="backbone 'dino' has no 'vit_large'"):
        DinoInterface("cuda", backbone="dino", backbone_type="vit_large")
    with pytest.raises(ValueError, match="backbone_type 'vit_huge'"):
        DinoInterface("cuda", backbone="dinov2", backbone_type="vit_huge")


# ------------------------------------------------------------------------------------------------ FeatureExtractor
class _FakeDino:
    """Stands in for DinoInterface: records its arguments (no device here)."""

    made = []

    def __init__(self, device, **kw):
        self.kw = kw
        self.grid = kw["input_size"] // 14
        _FakeDino.made.append(kw)


class _FakeStego:
    made = []

    def __init__(self, device, **kw):
        self.kw = kw
        self._dino = None
        _FakeStego.made.append(kw)


@pytest.fixture()
def fake_backbones(monkeypatch):
    from wild_visual_navigation_b200.feature_extractor import feature_extractor as fx

    _FakeDino.made.clear()
    _FakeStego.made.clear()
    monkeypatch.setattr(fx, "DinoInterface", _FakeDino)
    monkeypatch.setattr(fx, "StegoInterface", _FakeStego)
    return fx


@pytest.mark.parametrize("feature_type", ["dinov2", "dinov2_reg"])
def test_feature_extractor_width_is_1024(fake_backbones, feature_type):
    fe = fake_backbones.FeatureExtractor("cuda", segmentation_type="grid", feature_type=feature_type, input_size=224,
                                         backbone_type="vit_large")
    assert fe.feature_dim == 1024
    assert _FakeDino.made[-1]["backbone"] == feature_type and _FakeDino.made[-1]["backbone_type"] == "vit_large"
    # stego segmentation: STEGO's DINO backbone takes stego_backbone_type, the features stay ViT-L
    fe = fake_backbones.FeatureExtractor("cuda", segmentation_type="stego", feature_type=feature_type, input_size=224,
                                         backbone_type="vit_large", stego_backbone_type="vit_base")
    assert fe.feature_dim == 1024
    assert _FakeStego.made[-1]["backbone_type"] == "vit_base" and _FakeDino.made[-1]["backbone_type"] == "vit_large"


def test_feature_extractor_stego_follows_backbone_type_by_default(fake_backbones):
    fake_backbones.FeatureExtractor("cuda", segmentation_type="stego", feature_type="dinov2", input_size=224,
                                    backbone_type="vit_base")
    assert _FakeStego.made[-1]["backbone_type"] == "vit_base"


def test_stego_backbone_type_errors(fake_backbones):
    FE = fake_backbones.FeatureExtractor
    with pytest.raises(ValueError, match="stego_backbone_type"):
        FE("cuda", segmentation_type="stego", feature_type="dinov2", backbone_type="vit_large")
    with pytest.raises(ValueError, match="stego_backbone_type"):
        FE("cuda", segmentation_type="stego", feature_type="dinov2_reg", backbone_type="vit_large",
           stego_backbone_type="vit_large")
    with pytest.raises(ValueError, match="stego_backbone_type"):
        FE("cuda", segmentation_type="stego", feature_type="dinov2", backbone_type="vit_large",
           stego_backbone_type="vit_tiny")
    # STEGO's backbone gives the features: the two types must agree
    with pytest.raises(ValueError, match="stego_backbone_type"):
        FE("cuda", segmentation_type="stego", feature_type="dino", backbone_type="vit_small",
           stego_backbone_type="vit_base")
    # DINO v1 features have no ViT-L, with or without STEGO
    with pytest.raises(ValueError, match="backbone 'dino' has no 'vit_large'"):
        FE("cuda", segmentation_type="grid", feature_type="dino", backbone_type="vit_large")
    with pytest.raises(ValueError, match="backbone 'dino' has no 'vit_large'"):
        FE("cuda", segmentation_type="stego", feature_type="dino", backbone_type="vit_large")
    assert not _FakeDino.made and not _FakeStego.made


def test_hot_path_step_refuses_stego_on_vit_large():
    """HotPathStep hands stego_backbone_type to FeatureExtractor: without it, the refusal comes before any device work."""
    from wild_visual_navigation_b200 import HotPathStep

    with pytest.raises(ValueError, match="stego_backbone_type"):
        HotPathStep("cuda", None, None, feature_type="dinov2", backbone_type="vit_large")
