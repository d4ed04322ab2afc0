"""ORACLE (test infrastructure only) — CPU/PyTorch fp32 restatement of DINOv2 with register tokens.

Only ``tests/`` may import this module; the product (``wild_visual_navigation_b200``) never does.

The published ViT-S/14-reg and ViT-B/14-reg (Darcet et al., "Vision Transformers Need Registers", 2024;
``facebookresearch/dinov2`` hub ``dinov2_vit{s,b}14_reg``) [EXTERNAL-RECALLED], on top of ``oracle/dinov2_vit.py``,
which it reuses unchanged:

* ``x = cat(cls_token, patch_embed(img)) + interp(pos_embed)``: the position embedding covers CLS and the patches;
* ``register_tokens`` (1, R, D) inserted right after CLS, with no position embedding: ``[CLS, reg_0 .. reg_{R-1},
  patch_0 ..]``;
* the DINOv2 blocks (LayerScale) over all 1 + R + P tokens, then the final norm;
* output ``x_norm_patchtokens`` = ``norm(x)[:, 1 + R:]``.

The hub builds the register models with ``interpolate_antialias=True, interpolate_offset=0.0``, so their position
embeddings are interpolated by ``F.interpolate(size=(h, w), mode="bicubic", antialias=True)``, not by DINO's +0.1
scale-factor form (``interpolate_pos_encoding_antialias``).  Checkpoints (``dinov2_vit{s,b}14_reg4_pretrain.pth``) use
the DINOv2 keys plus ``register_tokens``.  Cross-checked end to end, interpolation included, against
``transformers.Dinov2WithRegistersModel`` in ``tests/test_dinov2_reg_oracle.py``.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from . import wvn_path
from .dino_vit import ViTConfig
from .dinov2_vit import dinov2_block, synthetic_dinov2_state_dict

REGISTERS, REGISTER_STD = 4, 0.02


def synthetic_dinov2_reg_state_dict(cfg: ViTConfig, seed: int = 1, attn_std: float = 0.09,
                                    registers: int = REGISTERS) -> dict:
    """``synthetic_dinov2_state_dict`` plus ``register_tokens`` (1, R, D) ~ N(0, 0.02^2) from their own generator
    (seed + 2)."""
    sd = synthetic_dinov2_state_dict(cfg, seed, attn_std)
    g = torch.Generator().manual_seed(seed + 2)
    sd["register_tokens"] = torch.randn(1, registers, cfg.dim, generator=g) * REGISTER_STD
    return sd


def interpolate_pos_encoding_antialias(pos_embed: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """The register models' interpolation: bicubic with antialias to ``size=(h, w)``; CLS row unchanged.  The
    pre-training grid passes through."""
    n_pre = pos_embed.shape[1] - 1
    if n_pre == h * w and h == w:
        return pos_embed
    dim = pos_embed.shape[-1]
    side = int(math.sqrt(n_pre))
    patch = F.interpolate(pos_embed[:, 1:].reshape(1, side, side, dim).permute(0, 3, 1, 2).float(), size=(h, w),
                          mode="bicubic", align_corners=False, antialias=True)
    return torch.cat((pos_embed[:, :1], patch.permute(0, 2, 3, 1).reshape(1, -1, dim)), dim=1)


@torch.no_grad()
def dinov2_reg_tokens(img_norm: torch.Tensor, sd: dict, cfg: ViTConfig) -> torch.Tensor:
    """Normalised image (B,3,S,S) -> ``x_norm_patchtokens`` (B, h*w, D) of DINOv2 with ``sd["register_tokens"]``."""
    x = F.conv2d(img_norm, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=cfg.patch_size)
    B, D, gh, gw = x.shape
    x = torch.cat((sd["cls_token"].expand(B, -1, -1), x.flatten(2).transpose(1, 2)), dim=1)
    x = x + interpolate_pos_encoding_antialias(sd["pos_embed"], gh, gw)
    reg = sd["register_tokens"]
    R = reg.shape[1]
    x = torch.cat((x[:, :1], reg.expand(B, -1, -1), x[:, 1:]), dim=1)
    for i in range(cfg.depth):
        x = dinov2_block(x, sd, f"blocks.{i}.", cfg.heads, cfg.ln_eps)
    return F.layer_norm(x, (D,), sd["norm.weight"], sd["norm.bias"], cfg.ln_eps)[:, 1 + R:, :]


@torch.no_grad()
def dinov2_reg_inference(img: torch.Tensor, sd: dict, cfg: ViTConfig) -> torch.Tensor:
    """``DinoInterface.inference`` with the register backbone: transform -> backbone -> bilinear(align_corners=True)
    to (H, H)."""
    tok = dinov2_reg_tokens(wvn_path.wvn_transform(img, cfg.image_size), sd, cfg)
    feats = tok.reshape(tok.shape[0], cfg.grid, cfg.grid, -1).permute(0, 3, 1, 2).contiguous()
    H = img.shape[2]
    return F.interpolate(feats, (H, H), mode="bilinear", align_corners=True)
