"""TorchVisionInterface (reference: wild_visual_navigation/feature_extractor/torchvision_interface.py:22-101).

``model_type`` ``resnet18``, ``resnet50`` or ``resnet50_dino`` (ResNet-50 with DINO's self-supervised weights).  The
reference wraps the torchvision model in ``create_feature_extractor`` and returns a feature pyramid ``{feat1..feat4}``:
  * resnet18: ``layer{1,2,3,4}.1.relu_1`` — the stage outputs, 64 / 128 / 256 / 512 channels at strides 4 / 8 / 16 / 32;
  * resnet50(_dino): ``layer{2,3,4}.0.relu`` — the ReLU after bn1 in each stage's first block, 128 / 256 / 512 channels
    at strides 4 / 8 / 16 — and ``layer4.2.relu_2``, the trunk output, 2048 channels at stride 32.
``model_type`` ``efficientnet_b0`` returns five levels ``{feat1..feat5}``: the SiLU outputs of
``features.{2,3,4,6}.0.block.0`` (each of those stages' first expand conv), 96 / 144 / 240 / 672 channels at strides
2 / 4 / 8 / 16, and of ``features.8`` (the head), 1280 channels at stride 32 — the reference's return nodes
``features.{2,3,4,6}.0.block.0.2`` / ``features.8.2``, which recent torchvision no longer traces.  ``efficientnet_b4``
and ``efficientnet_b7`` are not built.  For EfficientNet-B0, ``pretrained`` keeps torchvision's meaning: without a
checkpoint (``state_dict``, ``pretrained_weights`` or ``$WVN_EFFICIENTNET_WEIGHTS``), ``pretrained=True`` (ImageNet
weights, which cannot be downloaded here) raises ValueError and ``pretrained=False`` runs seeded weights.
Here the trunk is the library's ResNet or EfficientNet handle (csrc/resnet_kernels.cu, csrc/effnet_kernels.cu and the
wgmma GEMM), with batch norm folded into the convs.  ``Resize(S, BILINEAR) + CenterCrop(S)`` leave an S x S image unchanged, so of the transform only
``Normalize`` acts; it is applied in the stem's loader.  The pyramid is computed in NHWC bf16; ``inference`` / ``forward``
return it as the reference does (fp32 NCHW), ``inference_taps`` gives the NHWC bf16 maps the pooling kernel reads.
"""
from __future__ import annotations

import torch

from .. import ops
from .weights import (EFFNET_MODELS, RESNET_MODELS, check_efficientnet_family, check_resnet_family, fold_efficientnet_bn,
                      fold_resnet_bn, load_efficientnet_state_dict, load_resnet_state_dict)

MODEL_TYPES = tuple(RESNET_MODELS) + EFFNET_MODELS


class TorchVisionInterface:
    def __init__(self, device, model_type, input_size: int = 488, pretrained: bool = True, max_batch: int = 32,
                 state_dict=None, pretrained_weights: str = None):
        if model_type not in MODEL_TYPES:
            raise ValueError(f"model_type '{model_type}' is outside the H100 hot path ({', '.join(MODEL_TYPES)})")
        if input_size % 32 != 0:
            # the reference's unused default 488 is one such size; its callers pass 448
            raise ValueError(f"input_size {input_size} must be a multiple of 32 (the pyramid's nearest-downsampled "
                             f"segmentation is only exact then)")
        if not str(device).startswith("cuda"):
            raise RuntimeError("wild_visual_navigation_b200 runs on CUDA (sm_90a) devices only — no CPU fallback")
        self.device = device
        self.model_type = model_type
        self.input_size = input_size
        self.pretrained = pretrained
        if model_type in EFFNET_MODELS:
            sd = (check_efficientnet_family(state_dict, model_type) if state_dict is not None
                  else load_efficientnet_state_dict(model_type, pretrained_weights, pretrained))
            with torch.cuda.device(torch.device(device)):
                self._model = ops.EfficientNetBackbone(input_size, fold_efficientnet_bn(sd), max_batch=max_batch)
        else:
            depth = RESNET_MODELS[model_type]
            if state_dict is not None:
                sd = check_resnet_family(state_dict, model_type)
            else:
                sd = load_resnet_state_dict(model_type, pretrained_weights)
            with torch.cuda.device(torch.device(device)):
                self._model = ops.ResNetBackbone(input_size, depth, fold_resnet_bn(sd, depth), max_batch=max_batch)
        self.pyramid_keys = tuple(f"feat{i + 1}" for i in range(len(self._model.taps)))

    def change_device(self, device):
        if torch.device(device) != torch.device(self.device):
            raise RuntimeError("the backbone's weights and workspaces are bound to the device it was created on")

    @property
    def feature_dim(self):
        return sum(t[0] for t in self._model.taps)

    def _check(self, img):
        if img.dtype != torch.float32 or img.dim() != 4 or tuple(img.shape[1:]) != (3, self.input_size, self.input_size):
            # the reference's Resize would resample other sizes with antialiased bilinear filtering, which is not restated
            raise ValueError(f"TorchVisionInterface takes float32 images (B, 3, {self.input_size}, {self.input_size}); "
                             f"got {str(img.dtype)} {tuple(img.shape)}")

    @torch.no_grad()
    def inference_taps(self, img: torch.Tensor):
        """(B,3,S,S) fp32 in [0,1] -> the pyramid levels (four for a ResNet, five for EfficientNet-B0) as NHWC bf16
        maps [B, S/s, S/s, c] (for EfficientNet-B0, views of the first c channels of maps at a pitch of round_up(c, 64))."""
        self._check(img)
        return self._model.forward(img.to(self.device))

    @torch.no_grad()
    def forward(self, img: torch.Tensor):
        """(B,3,S,S) -> {feat1..feat4} (ResNets) or {feat1..feat5} (EfficientNet-B0): fp32 NCHW maps, the reference's
        pyramid dict."""
        return self.dense(self.inference_taps(img))

    def dense(self, taps):
        """inference_taps' maps -> the reference's pyramid dict (fp32 NCHW)."""
        return {k: t.permute(0, 3, 1, 2).float().contiguous() for k, t in zip(self.pyramid_keys, taps)}

    __call__ = forward

    @torch.no_grad()
    def inference(self, img: torch.Tensor, interpolate: bool = False):
        return self.forward(img)
