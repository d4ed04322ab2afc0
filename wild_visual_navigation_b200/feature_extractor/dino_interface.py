"""DinoInterface (reference: wild_visual_navigation/feature_extractor/dino_interface.py:16-108).

Same constructor arguments, ``inference`` / ``change_device`` and properties.  The transform
(``Resize(input_size, NEAREST) + CenterCrop + Normalize``, :52-59) is folded into the patch
loader kernel, the backbone is the wgmma ViT (csrc/), and the bilinear ``align_corners=True``
upsampling to ``(H, H)`` (:87-90) is only materialised by ``inference`` because its contract
returns the dense tensor; fused consumers call ``inference_tokens`` instead.
"""
from __future__ import annotations

import torch

from .. import ops
from .weights import DINOV2_PATCH, VIT_SHAPES, check_backbone_family, check_backbone_type, load_dino_state_dict


class _Cfg(dict):
    """Tiny stand-in for the OmegaConf node the reference stores in ``self._cfg``."""

    __getattr__ = dict.__getitem__

    def is_empty(self):
        return len(self) == 0


class DinoInterface:
    """``backbone="dino"``: DINO ViT-S / ViT-B at ``patch_size`` 8 or 16.  ``backbone="dinov2"``: DINOv2 ViT-S/14 /
    ViT-B/14 / ViT-L/14 / ViT-g/14 (no register tokens).  ``backbone="dinov2_reg"``: DINOv2 ViT-S/14-reg / ViT-B/14-reg /
    ViT-L/14-reg (4 register tokens; only the patch tokens are returned), and ViT-g/14 / ViT-g/14-reg likewise.
    ``backbone_type`` is "vit_small", "vit_base" or, for DINOv2 only, "vit_large" or "vit_giant" (ViT-g/14: D = 1536,
    40 blocks, 24 heads and a SwiGLU FFN; ``vit_giant`` follows the naming of the other sizes, and the name upstream
    STEGO's ``get_backbone`` gives this model is not pinned); a checkpoint of another width, depth or FFN raises
    ValueError.  DINOv2 is released at patch 14 only, so both run at patch 14 whatever
    ``patch_size`` says (the reference's ROS default passes ``patch_size=8`` with ``dinov2``); ``vit_patch_size`` still
    returns the configured value, as the reference's property does, while ``grid`` is the token grid actually run."""

    def __init__(self, device: str, backbone: str = "dino", input_size: int = 448, backbone_type: str = "vit_small",
                 patch_size: int = 8, projection_type: str = None, dropout_p: float = 0,
                 pretrained_weights: str = None, cfg=None, max_batch: int = 32, chunk: int = 0, state_dict=None,
                 head_weights=None):
        if cfg is not None and len(cfg) > 0:
            self._cfg = _Cfg(cfg)
        else:
            self._cfg = _Cfg(backbone=backbone, backbone_type=backbone_type, input_size=input_size,
                             patch_size=patch_size, projection_type=projection_type, dropout_p=dropout_p,
                             pretrained_weights=pretrained_weights)
        if self._cfg.backbone not in ("dino", "dinov2", "dinov2_reg"):
            raise ValueError(f"backbone '{self._cfg.backbone}' is outside the H100 hot path (DINO / DINOv2 ViT only)")
        if not str(device).startswith("cuda"):
            raise RuntimeError("wild_visual_navigation_b200 runs on CUDA (sm_90a) devices only — no CPU fallback")
        self._device = device
        backbone = self._cfg.backbone
        check_backbone_type(backbone, self._cfg.backbone_type)
        shp = VIT_SHAPES[self._cfg.backbone_type]
        patch = DINOV2_PATCH if backbone in ("dinov2", "dinov2_reg") else self._cfg.patch_size
        if state_dict is not None:
            sd = check_backbone_family(state_dict, backbone, self._cfg.backbone_type)
        else:
            sd = load_dino_state_dict(self._cfg.backbone_type, patch, self._cfg.pretrained_weights, backbone=backbone,
                                      device=device)
        with torch.cuda.device(torch.device(device)):
            self._model = ops.ViTBackbone(self._cfg.input_size, patch, shp["dim"], shp["depth"],
                                          shp["heads"], shp["mlp_dim"], sd, max_batch=max_batch, chunk=chunk,
                                          head_weights=head_weights)

    def change_device(self, device):
        if torch.device(device) != torch.device(self._device):
            raise RuntimeError("the backbone's weights and workspaces are bound to the device it was created on")

    @property
    def grid(self):
        return self._model.grid

    @property
    def feature_dim(self):
        return self._model.dim

    @torch.no_grad()
    def inference_tokens(self, img: torch.Tensor) -> torch.Tensor:
        """(B,3,H,W) in [0,1] -> final-norm patch tokens (B, h*w, D) fp32 — the fused path's product.
        Also accepts the camera frames as they arrive, (B,H,W,3) uint8 RGB: ``ros_image_to_torch``
        (ros_converter.py:113-126) and ``ImageProjector.resize_image`` (image_projector.py:199-200) are then
        folded into the patch loader (4x less host->device traffic, no fp32 image round trip)."""
        if img.dtype == torch.uint8:
            return self._model.forward(img.to(self._device))
        return self._model.forward(img.to(self._device, dtype=torch.float32))

    @torch.no_grad()
    def inference(self, img: torch.Tensor) -> torch.Tensor:
        """(B,3,H,W) -> dense per-pixel features (B, D, H, H), exactly the reference's contract
        (including the (H, H) quirk for non-square inputs, dino_interface.py:87-88)."""
        tokens = self.inference_tokens(img)
        H = img.shape[2]
        return ops.upsample_dense(tokens, self.grid, self.grid, H, H)

    @property
    def input_size(self):
        return self._cfg.input_size

    @property
    def backbone(self):
        return self._cfg.backbone

    @property
    def backbone_type(self):
        return self._cfg.backbone_type

    @property
    def vit_patch_size(self):
        return self._cfg.patch_size
