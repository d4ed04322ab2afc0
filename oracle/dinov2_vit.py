"""ORACLE (test infrastructure only) — CPU/PyTorch fp32 restatement of the DINOv2 ViT backbone.

Only ``tests/`` may import this module; the product (``wild_visual_navigation_b200``) never does.

The reference reaches DINOv2 through the same un-vendored ``stego.backbones.backbone.get_backbone`` that wraps the
``facebookresearch/dinov2`` hub models (``backbone="dinov2"``).  This file restates the published DINOv2 ViT-S/14 and
ViT-B/14 (no register tokens) [EXTERNAL-RECALLED], on top of the DINO restatement in ``oracle/dino_vit.py``:

* ``PatchEmbed`` = ``Conv2d(3, D, 14, 14)``; pre-training at 518 x 518, so ``pos_embed`` is ``(1, 1 + 37^2, D)``
* position embeddings interpolated by ``interpolate_pos_encoding`` with DINO's ``+0.1`` scale-factor form (bicubic,
  no antialias) — ``oracle.dino_vit.interpolate_pos_encoding`` from side 37
* pre-LN blocks with LayerScale: ``x += ls1.gamma * proj(attn(norm1(x)))``, ``x += ls2.gamma * fc2(GELU_erf(fc1(
  norm2(x))))``; ``qkv_bias=True``, head dim 64, LayerNorm eps 1e-6
* output ``x_norm_patchtokens`` = ``norm(x)[:, 1:]``, reshaped to ``(B, D, h, w)``.

Checkpoints (``dinov2_vit{s,b}14_pretrain.pth``) use DINO's key names plus ``blocks.N.ls{1,2}.gamma`` and an unused
``mask_token``.  Cross-checked against ``transformers.Dinov2Model`` in ``tests/test_dinov2_oracle.py``; parity
against upstream weights is unpinned, as for DINO.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import wvn_path
from .dino_vit import ViTConfig, interpolate_pos_encoding, synthetic_state_dict

PATCH, PRETRAIN_GRID = 14, 37


def dinov2_config(backbone_type: str = "vit_small", image_size: int = 448) -> ViTConfig:
    """DINOv2 ViT-S/14 / ViT-B/14: patch 14, position-embedding grid 37."""
    cfg = ViTConfig.from_name(backbone_type, PATCH, image_size)
    cfg.pretrain_grid = PRETRAIN_GRID
    return cfg


def synthetic_dinov2_state_dict(cfg: ViTConfig, seed: int = 1, attn_std: float = 0.09) -> dict:
    """Seeded DINOv2-layout weights: ``synthetic_state_dict`` at patch 14 / grid 37, then per-channel LayerScale gammas
    in [0.1, 1.0), drawn independently for ``ls1`` and ``ls2`` of every block, and the unused ``mask_token``."""
    sd = synthetic_state_dict(cfg, seed, attn_std)
    g = torch.Generator().manual_seed(seed + 1)
    for i in range(cfg.depth):
        sd[f"blocks.{i}.ls1.gamma"] = 0.1 + 0.9 * torch.rand(cfg.dim, generator=g)
        sd[f"blocks.{i}.ls2.gamma"] = 0.1 + 0.9 * torch.rand(cfg.dim, generator=g)
    sd["mask_token"] = torch.zeros(1, cfg.dim)
    return sd


def dinov2_block(x: torch.Tensor, sd: dict, prefix: str, heads: int, eps: float) -> torch.Tensor:
    """One DINOv2 block; without ``ls{1,2}.gamma`` in ``sd`` it is DINO's block."""
    B, N, C = x.shape
    dh = C // heads
    h = F.layer_norm(x, (C,), sd[prefix + "norm1.weight"], sd[prefix + "norm1.bias"], eps)
    qkv = F.linear(h, sd[prefix + "attn.qkv.weight"], sd[prefix + "attn.qkv.bias"])
    q, k, v = qkv.reshape(B, N, 3, heads, dh).permute(2, 0, 3, 1, 4)
    attn = ((q @ k.transpose(-2, -1)) * (dh**-0.5)).softmax(dim=-1)  # materialised, as upstream does
    h = F.linear((attn @ v).transpose(1, 2).reshape(B, N, C), sd[prefix + "attn.proj.weight"], sd[prefix + "attn.proj.bias"])
    if prefix + "ls1.gamma" in sd:
        h = h * sd[prefix + "ls1.gamma"]
    x = x + h
    h = F.layer_norm(x, (C,), sd[prefix + "norm2.weight"], sd[prefix + "norm2.bias"], eps)
    h = F.gelu(F.linear(h, sd[prefix + "mlp.fc1.weight"], sd[prefix + "mlp.fc1.bias"]))  # erf GELU
    h = F.linear(h, sd[prefix + "mlp.fc2.weight"], sd[prefix + "mlp.fc2.bias"])
    if prefix + "ls2.gamma" in sd:
        h = h * sd[prefix + "ls2.gamma"]
    return x + h


@torch.no_grad()
def dinov2_tokens(img_norm: torch.Tensor, sd: dict, cfg: ViTConfig) -> torch.Tensor:
    """Normalised image (B,3,S,S) -> ``x_norm_patchtokens`` (B, h*w, D)."""
    x = F.conv2d(img_norm, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=cfg.patch_size)
    B, D, gh, gw = x.shape
    x = torch.cat((sd["cls_token"].expand(B, -1, -1), x.flatten(2).transpose(1, 2)), dim=1)
    x = x + interpolate_pos_encoding(sd["pos_embed"], gh, gw)
    for i in range(cfg.depth):
        x = dinov2_block(x, sd, f"blocks.{i}.", cfg.heads, cfg.ln_eps)
    return F.layer_norm(x, (D,), sd["norm.weight"], sd["norm.bias"], cfg.ln_eps)[:, 1:, :]


@torch.no_grad()
def dinov2_feature_map(img_norm: torch.Tensor, sd: dict, cfg: ViTConfig) -> torch.Tensor:
    """(B, D, h, w), what the backbone hands to ``DinoInterface``."""
    tok = dinov2_tokens(img_norm, sd, cfg)
    return tok.reshape(tok.shape[0], cfg.grid, cfg.grid, -1).permute(0, 3, 1, 2).contiguous()


@torch.no_grad()
def dinov2_inference(img: torch.Tensor, sd: dict, cfg: ViTConfig) -> torch.Tensor:
    """``DinoInterface.inference`` with the DINOv2 backbone: transform -> backbone -> bilinear(align_corners=True) to
    (H, H), as ``oracle.wvn_path.dino_inference`` does for DINO."""
    feats = dinov2_feature_map(wvn_path.wvn_transform(img, cfg.image_size), sd, cfg)
    H = img.shape[2]
    return F.interpolate(feats, (H, H), mode="bilinear", align_corners=True)
