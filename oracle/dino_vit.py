"""ORACLE (test infrastructure only) — CPU/PyTorch fp32 restatement of the DINO ViT backbone.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline legs may import
this package; the product (``wild_visual_navigation_b200``) never does.

What it restates
----------------
The reference calls ``stego.backbones.backbone.get_backbone(cfg)`` and then ``self._model(img)``
(``wild_visual_navigation/feature_extractor/dino_interface.py:12,45,84``).  That package
(``leggedrobotics/self_supervised_segmentation``, *unpinned*, installed from a sibling clone:
reference ``README.md:103-123``, ``docker/first_run.sh:3-4``) is NOT vendored in
the reference repository; it wraps facebookresearch/dino's ``vision_transformer.py``.  This file
restates the published DINO algorithm [EXTERNAL-RECALLED, SURVEY.md §8 a3]:

* ``PatchEmbed``: ``Conv2d(3, D, p, p)`` -> flatten -> ``(B, N, D)``
* ``cls_token`` prepended, ``pos_embed`` added after bicubic interpolation from the
  pre-training grid with DINO's ``+0.1`` scale-factor trick (``interpolate_pos_encoding``)
* ``depth`` pre-LN blocks: ``x += proj(softmax(q k^T * dh^-0.5) v)``; ``x += fc2(GELU_erf(fc1(LN(x))))``
  with ``qkv_bias=True``, LayerNorm eps 1e-6
* the featurizer returns ``norm(x)`` of the last block (``get_intermediate_feat(n=1)``), drops
  CLS and reshapes to ``(B, D, h, w)``.

State-dict keys follow the DINO checkpoints (``dino_deitsmall8_pretrain.pth`` ...), so real
weights drop in.  PARITY STATUS: the reference pins no numbers for this stage (SURVEY.md §8c);
the restatement is cross-checked against torchvision's independent ``VisionTransformer``
implementation in ``tests/test_oracle.py`` — "parity unpinned" against upstream weights.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch
import torch.nn.functional as F


@dataclass
class ViTConfig:
    image_size: int = 448
    patch_size: int = 8
    dim: int = 384
    depth: int = 12
    heads: int = 6
    mlp_dim: int = 1536
    pretrain_grid: int = 28  # DINO checkpoints: 224 / 8
    ln_eps: float = 1e-6

    @property
    def grid(self) -> int:
        return self.image_size // self.patch_size  # conv-floor semantics

    @staticmethod
    def from_name(backbone_type: str = "vit_small", patch_size: int = 8, image_size: int = 448) -> "ViTConfig":
        if backbone_type == "vit_small":
            return ViTConfig(image_size, patch_size, 384, 12, 6, 1536, 224 // patch_size)
        if backbone_type == "vit_base":
            return ViTConfig(image_size, patch_size, 768, 12, 12, 3072, 224 // patch_size)
        raise ValueError(f"unknown backbone_type {backbone_type}")


def synthetic_state_dict(cfg: ViTConfig, seed: int = 1, attn_std: float = 0.09) -> dict:
    """Seeded DINO-layout weights (no network here, SURVEY.md §8d).

    trunc-normal-like N(0, 0.02) for embeddings / MLP weights as in DINO's init, but a larger
    std for qkv so attention logits have a realistic spread (std ~3) and small random biases /
    LayerNorm affine terms so every fused epilogue term is exercised by the parity tests.
    """
    g = torch.Generator().manual_seed(seed)

    def n(*shape, std):
        return torch.randn(*shape, generator=g) * std

    D, M = cfg.dim, cfg.mlp_dim
    sd = {
        "cls_token": n(1, 1, D, std=0.02),
        "pos_embed": n(1, 1 + cfg.pretrain_grid**2, D, std=0.02),
        "patch_embed.proj.weight": n(D, 3, cfg.patch_size, cfg.patch_size, std=0.05),
        "patch_embed.proj.bias": n(D, std=0.02),
        "norm.weight": 1.0 + n(D, std=0.05),
        "norm.bias": n(D, std=0.02),
    }
    for i in range(cfg.depth):
        b = f"blocks.{i}."
        sd[b + "norm1.weight"] = 1.0 + n(D, std=0.05)
        sd[b + "norm1.bias"] = n(D, std=0.02)
        sd[b + "attn.qkv.weight"] = n(3 * D, D, std=attn_std)
        sd[b + "attn.qkv.bias"] = n(3 * D, std=0.02)
        sd[b + "attn.proj.weight"] = n(D, D, std=0.02)
        sd[b + "attn.proj.bias"] = n(D, std=0.02)
        sd[b + "norm2.weight"] = 1.0 + n(D, std=0.05)
        sd[b + "norm2.bias"] = n(D, std=0.02)
        sd[b + "mlp.fc1.weight"] = n(M, D, std=0.04)
        sd[b + "mlp.fc1.bias"] = n(M, std=0.02)
        sd[b + "mlp.fc2.weight"] = n(D, M, std=0.02)
        sd[b + "mlp.fc2.bias"] = n(D, std=0.02)
    return sd


def interpolate_pos_encoding(pos_embed: torch.Tensor, grid_h: int, grid_w: int) -> torch.Tensor:
    """DINO ``VisionTransformer.interpolate_pos_encoding`` [EXTERNAL-RECALLED].

    pos_embed: (1, 1+N, D) at the pre-training grid.  Returns (1, 1 + grid_h*grid_w, D)."""
    n_pre = pos_embed.shape[1] - 1
    if n_pre == grid_h * grid_w and grid_h == grid_w:
        return pos_embed
    dim = pos_embed.shape[-1]
    side = int(math.sqrt(n_pre))
    class_pos = pos_embed[:, 0]
    patch_pos = pos_embed[:, 1:]
    # "we add a small number to avoid floating point error in the interpolation"
    w0, h0 = grid_w + 0.1, grid_h + 0.1
    patch_pos = F.interpolate(
        patch_pos.reshape(1, side, side, dim).permute(0, 3, 1, 2),
        scale_factor=(h0 / side, w0 / side),
        mode="bicubic",
    )
    assert patch_pos.shape[-2] == grid_h and patch_pos.shape[-1] == grid_w
    patch_pos = patch_pos.permute(0, 2, 3, 1).reshape(1, -1, dim)
    return torch.cat((class_pos.unsqueeze(0), patch_pos), dim=1)


# bench.py's GPU-eager leg also times the variant a maintainer would get by swapping the materialised attention for
# torch's fused kernel (BASELINE.md §3.2); parity tests always use the materialised form the upstream code has.
USE_SDPA = False


def vit_block(x: torch.Tensor, sd: dict, prefix: str, heads: int, eps: float) -> torch.Tensor:
    B, N, C = x.shape
    dh = C // heads
    h = F.layer_norm(x, (C,), sd[prefix + "norm1.weight"], sd[prefix + "norm1.bias"], eps)
    qkv = F.linear(h, sd[prefix + "attn.qkv.weight"], sd[prefix + "attn.qkv.bias"])
    qkv = qkv.reshape(B, N, 3, heads, dh).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    if USE_SDPA:
        h = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, N, C)
    else:
        attn = (q @ k.transpose(-2, -1)) * (dh**-0.5)  # materialised, as upstream does
        attn = attn.softmax(dim=-1)
        h = (attn @ v).transpose(1, 2).reshape(B, N, C)
    x = x + F.linear(h, sd[prefix + "attn.proj.weight"], sd[prefix + "attn.proj.bias"])
    h = F.layer_norm(x, (C,), sd[prefix + "norm2.weight"], sd[prefix + "norm2.bias"], eps)
    h = F.gelu(F.linear(h, sd[prefix + "mlp.fc1.weight"], sd[prefix + "mlp.fc1.bias"]))  # erf GELU
    return x + F.linear(h, sd[prefix + "mlp.fc2.weight"], sd[prefix + "mlp.fc2.bias"])


@torch.no_grad()
def vit_tokens(img_norm: torch.Tensor, sd: dict, cfg: ViTConfig) -> torch.Tensor:
    """Normalised image (B,3,S,S) -> final-norm patch tokens (B, h*w, D), CLS dropped."""
    x = F.conv2d(img_norm, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=cfg.patch_size)
    B, D, gh, gw = x.shape
    x = x.flatten(2).transpose(1, 2)
    x = torch.cat((sd["cls_token"].expand(B, -1, -1), x), dim=1)
    x = x + interpolate_pos_encoding(sd["pos_embed"], gh, gw)
    for i in range(cfg.depth):
        x = vit_block(x, sd, f"blocks.{i}.", cfg.heads, cfg.ln_eps)
    x = F.layer_norm(x, (D,), sd["norm.weight"], sd["norm.bias"], cfg.ln_eps)
    return x[:, 1:, :]


@torch.no_grad()
def vit_feature_map(img_norm: torch.Tensor, sd: dict, cfg: ViTConfig) -> torch.Tensor:
    """What ``self._model(resized_img)`` returns in dino_interface.py:84: (B, D, h, w)."""
    tok = vit_tokens(img_norm, sd, cfg)
    B, P, D = tok.shape
    g = cfg.grid
    return tok.reshape(B, g, g, D).permute(0, 3, 1, 2).contiguous()
