"""DINOv2 ViT-g/14 (``backbone_type="vit_giant"``: D = 1536, 40 blocks, 24 heads, SwiGLU FFN of 4096) on the CPU.

  oracle            an fp32 restatement of the ViT-g/14 block (below; ``oracle/dinov2_vit.py``'s block has the GELU
                    MLP only) against ``transformers.Dinov2Model(use_swiglu_ffn=True)`` and
                    ``Dinov2WithRegistersModel(use_swiglu_ffn=True)`` at ViT-g width, reduced depth, 56 and 112 input,
                    to 1e-5
  w12 packing       the library's packed row order of ``mlp.w12`` is a permutation with the tile layout EPI_SWIGLU
                    reads, and unpacking it gives the checkpoint back exactly
  seeded weights    the SwiGLU layout of ``synthetic_dinov2_state_dict(ffn="swiglu")`` (plain and ``_reg``)
  family / size     ``check_backbone_family`` takes ``vit_giant`` for ``dinov2`` and ``dinov2_reg`` (``mask_token``
                    dropped, position embeddings interpolated to the run's grid), refuses a GELU-MLP dict given as
                    ``vit_giant`` and a SwiGLU dict given as another size, naming both; DINO v1 refuses ``vit_giant``
  FeatureExtractor  ``feature_dim`` 1536, and STEGO segmentation needs ``stego_backbone_type``

The ViT-g/14 block, as released (``SwiGLUFFNFused``): x += ls1 * proj(attn(norm1(x))); [x1 | x2] = w12(norm2(x));
x += ls2 * w3(silu(x1) * x2).
"""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle.dino_vit import ViTConfig, interpolate_pos_encoding
from oracle.dinov2_reg_vit import interpolate_pos_encoding_antialias
from oracle.dinov2_vit import PATCH, PRETRAIN_GRID
from wild_visual_navigation_b200.feature_extractor import weights as W

D, H = 1536, 4096
# qkv std that keeps the attention logits' spread of the ViT-S/B tests (it scales with D)
ATTN_STD = 0.09 * (384 / D) ** 0.5


def giant_config(image_size, depth=None):
    s = W.VIT_SHAPES["vit_giant"]
    return ViTConfig(image_size, PATCH, s["dim"], s["depth"] if depth is None else depth, s["heads"], s["mlp_dim"],
                     PRETRAIN_GRID)


def giant_state_dict(depth, seed, registers=False, device="cpu"):
    s = W.VIT_SHAPES["vit_giant"]
    make = W.synthetic_dinov2_reg_state_dict if registers else W.synthetic_dinov2_state_dict
    return make(s["dim"], depth, s["mlp_dim"], seed=seed, attn_std=ATTN_STD, ffn="swiglu", device=device)


def swiglu_block(x, sd, prefix, heads, eps):
    """One DINOv2 ViT-g/14 block in fp32 (module docstring)."""
    B, N, C = x.shape
    h = F.layer_norm(x, (C,), sd[prefix + "norm1.weight"], sd[prefix + "norm1.bias"], eps)
    qkv = F.linear(h, sd[prefix + "attn.qkv.weight"], sd[prefix + "attn.qkv.bias"])
    q, k, v = qkv.reshape(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    attn = ((q @ k.transpose(-2, -1)) * 0.125).softmax(dim=-1)
    h = F.linear((attn @ v).transpose(1, 2).reshape(B, N, C), sd[prefix + "attn.proj.weight"],
                 sd[prefix + "attn.proj.bias"])
    x = x + h * sd[prefix + "ls1.gamma"]
    h = F.layer_norm(x, (C,), sd[prefix + "norm2.weight"], sd[prefix + "norm2.bias"], eps)
    x1, x2 = F.linear(h, sd[prefix + "mlp.w12.weight"], sd[prefix + "mlp.w12.bias"]).chunk(2, dim=-1)
    h = F.linear(F.silu(x1) * x2, sd[prefix + "mlp.w3.weight"], sd[prefix + "mlp.w3.bias"])
    return x + h * sd[prefix + "ls2.gamma"]


@torch.no_grad()
def giant_tokens(img_norm, sd, cfg):
    """Normalised image (B,3,S,S) -> ``x_norm_patchtokens`` (B, h*w, D) of DINOv2 ViT-g/14, with register tokens when
    ``sd`` has them (then with the register models' antialiased position-embedding interpolation)."""
    x = F.conv2d(img_norm, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=cfg.patch_size)
    B, C, gh, gw = x.shape
    reg = sd.get("register_tokens")
    interp = interpolate_pos_encoding if reg is None else interpolate_pos_encoding_antialias
    x = torch.cat((sd["cls_token"].expand(B, -1, -1), x.flatten(2).transpose(1, 2)), dim=1)
    x = x + interp(sd["pos_embed"], gh, gw)
    R = 0 if reg is None else reg.shape[1]
    if R:
        x = torch.cat((x[:, :1], reg.expand(B, -1, -1), x[:, 1:]), dim=1)
    for i in range(cfg.depth):
        x = swiglu_block(x, sd, f"blocks.{i}.", cfg.heads, cfg.ln_eps)
    return F.layer_norm(x, (C,), sd["norm.weight"], sd["norm.bias"], cfg.ln_eps)[:, 1 + R:]


# ------------------------------------------------------------------------------------------------ vs transformers
def _img(B, S, seed):
    return torch.randn(B, 3, S, S, generator=torch.Generator().manual_seed(seed))


def _hf_layers(sd, depth):
    m = {"embeddings.cls_token": sd["cls_token"], "embeddings.mask_token": sd["mask_token"],
         "embeddings.patch_embeddings.projection.weight": sd["patch_embed.proj.weight"],
         "embeddings.patch_embeddings.projection.bias": sd["patch_embed.proj.bias"],
         "layernorm.weight": sd["norm.weight"], "layernorm.bias": sd["norm.bias"]}
    for i in range(depth):
        s, d = f"blocks.{i}.", f"encoder.layer.{i}."
        for leaf in ("norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias"):
            m[d + leaf] = sd[s + leaf]
        for ours, theirs in (("w12", "weights_in"), ("w3", "weights_out")):
            m[d + f"mlp.{theirs}.weight"] = sd[s + f"mlp.{ours}.weight"]
            m[d + f"mlp.{theirs}.bias"] = sd[s + f"mlp.{ours}.bias"]
        for j, name in enumerate(("query", "key", "value")):
            m[d + f"attention.attention.{name}.weight"] = sd[s + "attn.qkv.weight"][j * D:(j + 1) * D]
            m[d + f"attention.attention.{name}.bias"] = sd[s + "attn.qkv.bias"][j * D:(j + 1) * D]
        m[d + "attention.output.dense.weight"] = sd[s + "attn.proj.weight"]
        m[d + "attention.output.dense.bias"] = sd[s + "attn.proj.bias"]
        m[d + "layer_scale1.lambda1"] = sd[s + "ls1.gamma"]
        m[d + "layer_scale2.lambda1"] = sd[s + "ls2.gamma"]
    return m


def _hf_kwargs(cfg):
    # mlp_ratio 4 -> SwiGLU hidden (int(4 * 1536 * 2 / 3) + 7) // 8 * 8 = 4096
    return dict(hidden_size=cfg.dim, num_hidden_layers=cfg.depth, num_attention_heads=cfg.heads, mlp_ratio=4,
                patch_size=14, layerscale_value=1.0, layer_norm_eps=cfg.ln_eps, hidden_act="gelu", qkv_bias=True,
                use_swiglu_ffn=True, attn_implementation="eager")


@pytest.fixture(scope="module")
def shallow_sds():
    return {"dinov2": giant_state_dict(2, seed=3), "dinov2_reg": giant_state_dict(2, seed=4, registers=True)}


@pytest.mark.parametrize("image_size", [56, 112])
def test_oracle_matches_transformers_dinov2_giant(shallow_sds, image_size):
    transformers = pytest.importorskip("transformers")
    cfg = giant_config(image_size, depth=2)
    sd = shallow_sds["dinov2"]
    model = transformers.Dinov2Model(transformers.Dinov2Config(image_size=image_size, **_hf_kwargs(cfg))).eval()
    assert model.encoder.layer[0].mlp.weights_in.weight.shape == (2 * H, D)
    m = _hf_layers(sd, cfg.depth)
    # transformers interpolates with size=, so it gets the embeddings already at the grid (as test_dinov2_oracle.py)
    m["embeddings.position_embeddings"] = interpolate_pos_encoding(sd["pos_embed"], cfg.grid, cfg.grid)
    model.load_state_dict(m, strict=True)
    x = _img(2, image_size, 0)
    with torch.no_grad():
        ref = model(pixel_values=x).last_hidden_state[:, 1:]
    got = giant_tokens(x, sd, cfg)
    assert got.shape == ref.shape == (2, cfg.grid**2, D)
    err = (got - ref).abs().max().item()
    print(f"vit_giant @{image_size}: max |oracle - Dinov2Model| = {err:.2e}")
    assert err <= 1e-5


@pytest.mark.parametrize("image_size", [56, 112])
def test_oracle_matches_transformers_dinov2_giant_with_registers(shallow_sds, image_size):
    """End to end, the register models' antialiased interpolation included (the model gets the 37 x 37 grid)."""
    transformers = pytest.importorskip("transformers")
    cfg = giant_config(image_size, depth=2)
    sd = shallow_sds["dinov2_reg"]
    hc = transformers.Dinov2WithRegistersConfig(image_size=518, num_register_tokens=4, **_hf_kwargs(cfg))
    model = transformers.Dinov2WithRegistersModel(hc).eval().float()
    m = dict(_hf_layers(sd, cfg.depth), **{"embeddings.register_tokens": sd["register_tokens"],
                                           "embeddings.position_embeddings": sd["pos_embed"]})
    model.load_state_dict(m, strict=True)
    x = _img(2, image_size, 1)
    with torch.no_grad():
        ref = model(pixel_values=x).last_hidden_state[:, 5:]
    got = giant_tokens(x, sd, cfg)
    assert got.shape == ref.shape == (2, cfg.grid**2, D)
    err = (got - ref).abs().max().item()
    print(f"vit_giant-reg @{image_size}: max |oracle - Dinov2WithRegistersModel| = {err:.2e}")
    assert err <= 1e-5


# ------------------------------------------------------------------------------------------------ w12 packing
def packed_rows(rows):
    """The library's packed row order of w12 (wvn_swiglu_packed_rows): packed row p holds checkpoint row perm[p]."""
    import ctypes

    import __graft_entry__ as g

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.exists(os.path.join(root, "wild_visual_navigation_b200", "libwvn_b200.so")):
        g.build()
    from wild_visual_navigation_b200 import _C

    out = torch.empty(rows, dtype=torch.int64)
    _C.check(_C.lib().wvn_swiglu_packed_rows(rows, ctypes.c_void_p(out.data_ptr())))
    return out


@pytest.mark.parametrize("rows", [256, 2 * H])
def test_w12_packing_is_an_exactly_invertible_permutation(rows):
    perm = packed_rows(rows)
    assert torch.equal(perm.sort().values, torch.arange(rows))
    # each 256-row tile: 128 gate rows, then the value rows of the same hidden units
    tiles = perm.view(-1, 2, 128)
    t = torch.arange(rows // 256)[:, None] * 128 + torch.arange(128)
    assert torch.equal(tiles[:, 0], t) and torch.equal(tiles[:, 1], t + rows // 2)
    w = torch.randn(rows, 24, generator=torch.Generator().manual_seed(rows))
    packed = w[perm]
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(rows)
    assert torch.equal(packed[inv], w)


def test_w12_packing_refuses_partial_tiles():
    import ctypes

    from wild_visual_navigation_b200 import _C

    packed_rows(256)   # builds the library if needed
    out = torch.empty(384, dtype=torch.int64)
    assert _C.lib().wvn_swiglu_packed_rows(384, ctypes.c_void_p(out.data_ptr())) != 0


# ------------------------------------------------------------------------------------------------ seeded weights
def test_vit_giant_shape():
    assert W.VIT_SHAPES["vit_giant"] == dict(dim=1536, depth=40, heads=24, mlp_dim=4096, ffn="swiglu")
    assert (int(4 * 1536 * 2 / 3) + 7) // 8 * 8 == W.VIT_SHAPES["vit_giant"]["mlp_dim"]
    assert W.vit_ffn("vit_giant") == "swiglu" and all(W.vit_ffn(t) == "mlp" for t in ("vit_small", "vit_base", "vit_large"))


def test_seeded_swiglu_layout(shallow_sds):
    v2, reg = shallow_sds["dinov2"], shallow_sds["dinov2_reg"]
    shapes = {"cls_token": (1, 1, D), "pos_embed": (1, 1 + 37 * 37, D), "mask_token": (1, D),
              "patch_embed.proj.weight": (D, 3, 14, 14), "blocks.1.attn.qkv.weight": (3 * D, D),
              "blocks.1.mlp.w12.weight": (2 * H, D), "blocks.1.mlp.w12.bias": (2 * H,),
              "blocks.1.mlp.w3.weight": (D, H), "blocks.1.mlp.w3.bias": (D,), "blocks.1.ls2.gamma": (D,)}
    for k, shp in shapes.items():
        assert tuple(v2[k].shape) == shp and tuple(reg[k].shape) == shp, k
    assert not any(".fc1." in k or ".fc2." in k for k in v2)
    assert reg.keys() == v2.keys() | {"register_tokens"} and tuple(reg["register_tokens"].shape) == (1, 4, D)
    again = giant_state_dict(2, seed=3)
    assert all(torch.equal(v2[k], again[k]) for k in v2)


# ------------------------------------------------------------------------------------------------ family / size checks
def _deepen(sd, depth):
    """``sd``'s layout at ``depth`` blocks, as shape-only (meta) tensors: the checks read keys and shapes only."""
    out = {k: torch.empty(v.shape, device="meta") for k, v in sd.items() if not k.startswith("blocks.")}
    for k, v in sd.items():
        if k.startswith("blocks.0."):
            for i in range(depth):
                out[f"blocks.{i}." + k[len("blocks.0."):]] = torch.empty(v.shape, device="meta")
    return out


def test_family_checks_accept_vit_giant(shallow_sds):
    full = {b: _deepen(sd, 40) for b, sd in shallow_sds.items()}
    for backbone, sd in full.items():
        kept = W.check_backbone_family(sd, backbone, "vit_giant")
        assert kept.keys() == sd.keys() - {"mask_token"}
    with pytest.raises(ValueError, match="register tokens"):
        W.check_backbone_family(full["dinov2_reg"], "dinov2", "vit_giant")
    with pytest.raises(ValueError, match="register tokens"):
        W.check_backbone_family(full["dinov2"], "dinov2_reg", "vit_giant")


def test_ffn_refusals_name_both_sizes(shallow_sds):
    giant = _deepen(shallow_sds["dinov2"], 40)
    gelu_giant = {k: v for k, v in giant.items() if ".mlp." not in k}
    for i in range(40):
        gelu_giant[f"blocks.{i}.mlp.fc1.weight"] = torch.empty(6144, D, device="meta")
        gelu_giant[f"blocks.{i}.mlp.fc1.bias"] = torch.empty(6144, device="meta")
        gelu_giant[f"blocks.{i}.mlp.fc2.weight"] = torch.empty(D, 6144, device="meta")
        gelu_giant[f"blocks.{i}.mlp.fc2.bias"] = torch.empty(D, device="meta")
    with pytest.raises(ValueError) as e:
        W.check_backbone_family(gelu_giant, "dinov2", "vit_giant")
    msg = str(e.value)
    assert "'vit_giant'" in msg and "SwiGLU FFN" in msg and "GELU MLP" in msg and "D = 1536 with 40 blocks" in msg, msg
    for other in ("vit_small", "vit_base", "vit_large"):
        with pytest.raises(ValueError) as e:
            W.check_backbone_family(giant, "dinov2", other)
        msg = str(e.value)
        assert f"'{other}'" in msg and "vit_giant (D = 1536, 40 blocks)" in msg, msg
    # a ViT-L checkpoint given as vit_giant
    large = W.synthetic_dinov2_state_dict(1024, 24, 4096, seed=1)
    with pytest.raises(ValueError, match="vit_large"):
        W.check_backbone_family(large, "dinov2", "vit_giant")


def test_checkpoint_route_checks_ffn(tmp_path):
    sd = giant_state_dict(2, seed=5)
    path = tmp_path / "shallow_vitg14.pth"
    torch.save(sd, path)
    with pytest.raises(ValueError, match="vit_giant"):
        W.load_dino_state_dict("vit_giant", 14, str(path), backbone="dinov2")


@pytest.mark.parametrize("registers", [False, True])
def test_position_embeddings_interpolate_at_1536(registers):
    """The handle's position-embedding interpolation (ops) at ViT-g width equals the oracle's, for both variants."""
    from wild_visual_navigation_b200.ops import interpolate_pos_embed, interpolate_pos_embed_antialias

    pos = torch.randn(1, 1 + 37 * 37, D, generator=torch.Generator().manual_seed(9)) * 0.02
    for grid in (16, 32):
        if registers:
            got, ref = interpolate_pos_embed_antialias(pos, grid), interpolate_pos_encoding_antialias(pos, grid, grid)
        else:
            got, ref = interpolate_pos_embed(pos, grid), interpolate_pos_encoding(pos, grid, grid)
        assert got.shape == ref.shape == (1, 1 + grid * grid, D)
        assert (got - ref).abs().max().item() <= 1e-6


def test_dino_v1_has_no_vit_giant():
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    with pytest.raises(ValueError, match="backbone 'dino' has no 'vit_giant'"):
        W.load_dino_state_dict("vit_giant", 8, None, backbone="dino")
    with pytest.raises(ValueError, match="backbone 'dino' has no 'vit_giant'"):
        DinoInterface("cuda", backbone="dino", backbone_type="vit_giant")


# ------------------------------------------------------------------------------------------------ FeatureExtractor
class _FakeDino:
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
def test_feature_extractor_width_is_1536(fake_backbones, feature_type):
    FE = fake_backbones.FeatureExtractor
    fe = FE("cuda", segmentation_type="grid", feature_type=feature_type, input_size=224, backbone_type="vit_giant")
    assert fe.feature_dim == 1536 and _FakeDino.made[-1]["backbone_type"] == "vit_giant"
    fe = FE("cuda", segmentation_type="stego", feature_type=feature_type, input_size=224, backbone_type="vit_giant",
            stego_backbone_type="vit_small")
    assert fe.feature_dim == 1536
    assert _FakeStego.made[-1]["backbone_type"] == "vit_small" and _FakeDino.made[-1]["backbone_type"] == "vit_giant"
    with pytest.raises(ValueError, match="stego_backbone_type"):
        FE("cuda", segmentation_type="stego", feature_type=feature_type, backbone_type="vit_giant")
    with pytest.raises(ValueError, match="stego_backbone_type"):
        FE("cuda", segmentation_type="stego", feature_type=feature_type, backbone_type="vit_giant",
           stego_backbone_type="vit_giant")


def test_hot_path_step_refuses_stego_on_vit_giant():
    from wild_visual_navigation_b200 import HotPathStep

    with pytest.raises(ValueError, match="stego_backbone_type"):
        HotPathStep("cuda", None, None, feature_type="dinov2", backbone_type="vit_giant")
