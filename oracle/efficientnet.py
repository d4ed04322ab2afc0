"""ORACLE (test infrastructure only) — CPU/PyTorch restatement of the reference's EfficientNet-B0 feature pyramid.

Only ``tests/`` may import this module; the product (``wild_visual_navigation_b200``) never does.

The reference's ``TorchVisionInterface`` (feature_extractor/torchvision_interface.py) runs torchvision's
``efficientnet_b0`` in eval mode behind ``create_feature_extractor`` with the return nodes
``features.{2,3,4,6}.0.block.0.2`` and ``features.8.2`` -> feat1..feat5.  Recent torchvision no longer traces into
``Conv2dNormActivation``, so those nodes do not exist any more; they are the SiLU outputs of ``features.{2,3,4,6}.0
.block.0`` (each of those stages' first expand conv) and of ``features.8`` (the head), and tapping these modules gives
the same tensors.  Of the transform, only ``Normalize`` acts on an S x S input.

B0 here, with ``torch.nn.functional`` (eval-mode batch norm, eps 1e-5; stochastic depth is the identity in eval):
  stem       3 x 3 / 2 conv 3 -> 32, batch norm, SiLU
  MBConv     [expand 1 x 1 + bn + SiLU (ratio 6)], depthwise k x k / s + bn + SiLU, squeeze-excitation (average pool,
             fc1 -> max(1, in / 4) with bias, SiLU, fc2 with bias, sigmoid, channel multiply), project 1 x 1 + bn,
             + the block input when the stride is 1 and the width does not change
  stages     (ratio, k, stride, out, blocks) = (1,3,1,16,1) (6,3,2,24,2) (6,5,2,40,2) (6,3,2,80,3) (6,5,1,112,3)
             (6,5,2,192,4) (6,3,1,320,1)
  head       1 x 1 conv 320 -> 1280, batch norm, SiLU
``tests/test_efficientnet_oracle.py`` ties it to torchvision itself.

``bf16=True`` (with ``folded``) rounds where the product stores bf16: the normalised image, the GEMM weights (stem,
expand, project, head), and every map the product writes — the stem, expand, depthwise (after SiLU), gated (after the
squeeze-excitation multiply), project and head outputs.  The depthwise weights and the squeeze-excitation stay fp32, as
in the product, and its average pool sums the bf16-rounded depthwise output.

The pooling is ``oracle.resnet.pool_pyramid``, which takes any number of levels.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .resnet import centroids, normalize, pool_pyramid  # noqa: F401  (re-exported: the five-level pooling)

STAGES = ((1, 3, 1, 16, 1), (6, 3, 2, 24, 2), (6, 5, 2, 40, 2), (6, 3, 2, 80, 3), (6, 5, 1, 112, 3), (6, 5, 2, 192, 4),
          (6, 3, 1, 320, 1))
BN_EPS = 1e-5
TAP_STAGES = (2, 3, 4, 6)  # feat1..feat4: the expand conv of these stages' first blocks; feat5: the head
TAP_NODES = {"features.2.0.block.0": "feat1", "features.3.0.block.0": "feat2", "features.4.0.block.0": "feat3",
             "features.6.0.block.0": "feat4", "features.8": "feat5"}


def _bf16(t):
    return t.bfloat16().to(t.dtype)


def efficientnet_pyramid(img: torch.Tensor, sd: dict, folded: bool = False, bf16: bool = False) -> dict:
    """img (B,3,S,S) in [0,1] -> {feat1..feat5} NCHW.  ``sd``: torchvision-layout state dict, or with ``folded`` a dict
    of ``{module}.weight`` / ``{module}.bias`` with batch norm folded in (weights.fold_efficientnet_bn's modules) and the
    squeeze-excitations' ``{module}.fc{1,2}.weight`` [out, in] / ``.bias``."""
    assert folded or not bf16
    r = _bf16 if bf16 else (lambda t: t)

    def conv(x, m, stride=1, groups=1, act=True, res=None):
        if folded:
            w, b = sd[m + ".weight"], sd[m + ".bias"]
            if groups == 1 and bf16:
                w = _bf16(w)  # GEMM weights are bf16; depthwise weights stay fp32
            x = F.conv2d(x, w, b, stride=stride, padding=(w.shape[-1] - 1) // 2, groups=groups)
        else:
            w = sd[m + ".0.weight"]
            x = F.conv2d(x, w, stride=stride, padding=(w.shape[-1] - 1) // 2, groups=groups)
            bn = m + ".1."
            x = F.batch_norm(x, sd[bn + "running_mean"], sd[bn + "running_var"], sd[bn + "weight"], sd[bn + "bias"],
                             False, 0.0, BN_EPS)
        if res is not None:
            x = x + res
        return r(F.silu(x) if act else x)

    def fc(x, name):
        w = sd[name + ".weight"]
        return F.linear(x, w if w.dim() == 2 else w[:, :, 0, 0], sd[name + ".bias"])

    taps = []
    x = conv(r(normalize(img)), "features.0", stride=2)
    cin = 32
    for s, (ratio, k, stride0, cout, n) in enumerate(STAGES, start=1):
        for i in range(n):
            p = f"features.{s}.{i}.block."
            stride = stride0 if i == 0 else 1
            cexp = cin * ratio
            j = 0
            y = x
            if ratio != 1:
                y = conv(y, p + "0")
                if i == 0 and s in TAP_STAGES:
                    taps.append(y)
                j = 1
            y = conv(y, p + str(j), stride=stride, groups=cexp)
            se = p + str(j + 1)
            g = torch.sigmoid(fc(F.silu(fc(y.mean((2, 3)), se + ".fc1")), se + ".fc2"))
            y = r(y * g[:, :, None, None])
            x = conv(y, p + str(j + 2), act=False, res=x if stride == 1 and cin == cout else None)
            cin = cout
    taps.append(conv(x, "features.8"))
    return {f"feat{i + 1}": t for i, t in enumerate(taps)}


def folded_state_dict(folded_modules: dict) -> dict:
    """weights.fold_efficientnet_bn's {module: (w, b)} -> the flat ``{module}.weight`` / ``.bias`` dict
    efficientnet_pyramid(folded=True) reads."""
    out = {}
    for m, (w, b) in folded_modules.items():
        out[m + ".weight"], out[m + ".bias"] = w, b
    return out
