"""ORACLE (test infrastructure only) — CPU/PyTorch fp32 restatement of the reference's torchvision feature pyramid.

Only ``tests/`` may import this module; the product (``wild_visual_navigation_b200``) never does.

The reference's ``TorchVisionInterface`` (feature_extractor/torchvision_interface.py:22-101) runs torchvision's
``resnet18`` / ``resnet50`` in eval mode behind ``create_feature_extractor`` with these return nodes:
  resnet18: layer{1,2,3,4}.1.relu_1 (stage outputs)            -> feat1..feat4
  resnet50: layer2.0.relu, layer3.0.relu, layer4.0.relu (the ReLU after bn1 of each stage's first block),
            layer4.2.relu_2 (trunk output)                      -> feat1..feat4
and ``Resize(S) + CenterCrop(S) + Normalize(ImageNet)`` in front, of which only Normalize acts on an S x S input.
Here the trunk is restated with ``torch.nn.functional`` (conv2d, eval-mode batch_norm with eps 1e-5, relu,
max_pool2d); ResNet-50 is torchvision's v1.5 (stride in the 3 x 3 conv).  ``tests/test_resnet_oracle.py`` ties it to
torchvision itself.

``pool_pyramid`` restates ``FeatureExtractor.sparsify_features``' dict branch (feature_extractor.py:314-366) for one
frame: per level, the segmentation is nearest-downsampled (``F.interpolate(seg, scale_factor=h_l / H)``, i.e.
``seg[i * H / h_l, j * W / w_l]``), and a segment's level feature is the mean of the level's map over its cells.  Where
a segment has no cell at a level the reference raises AttributeError; here (as in the product) it takes the cell
``(clamp(floor(y * h_l / H)), clamp(floor(x * w_l / W)))`` under its full-resolution centroid (x, y).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

BLOCKS = {18: (2, 2, 2, 2), 50: (3, 4, 6, 3)}
BN_EPS = 1e-5
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def normalize(img: torch.Tensor) -> torch.Tensor:
    mean = torch.tensor(MEAN, dtype=img.dtype, device=img.device)[:, None, None]
    std = torch.tensor(STD, dtype=img.dtype, device=img.device)[:, None, None]
    return (img - mean) / std


def _bf16(t):
    return t.bfloat16().to(t.dtype)


def _conv_bn_(x, sd, conv, bn, stride, relu=True, res=None, folded=False, bf16=False):
    w = sd[conv + ".weight"]
    pad = w.shape[-1] // 2
    if bf16:
        # the product's storage precision: bf16 weights and activations, fp32 sums, bias and residual added before the
        # ReLU and one rounding of the result
        x = F.conv2d(x, _bf16(w), sd[conv + ".bias"], stride=stride, padding=pad)
        if res is not None:
            x = x + res
        return _bf16(F.relu(x) if relu else x)
    if folded:
        x = F.conv2d(x, w, sd[conv + ".bias"], stride=stride, padding=pad)
    else:
        x = F.conv2d(x, w, stride=stride, padding=pad)
        x = F.batch_norm(x, sd[bn + ".running_mean"], sd[bn + ".running_var"], sd[bn + ".weight"], sd[bn + ".bias"],
                         False, 0.0, BN_EPS)
    if res is not None:
        x = x + res
    return F.relu(x) if relu else x


def resnet_pyramid(img: torch.Tensor, sd: dict, depth: int, folded: bool = False, bf16: bool = False) -> dict:
    """img (B,3,S,S) in [0,1] -> {feat1..feat4} NCHW.  ``sd``: torchvision-layout state dict, or with ``folded`` a dict
    of ``{conv}.weight`` / ``{conv}.bias`` with batch norm folded in (downsample conv named ``layer{L}.0.downsample``).
    ``bf16`` (with ``folded``) rounds the normalised image, every weight and every conv output to bf16, as the product
    stores them, so that what remains between the two is the order of the fp32 sums."""
    assert folded or not bf16
    ds = "downsample" if folded else "downsample.0"
    taps = []
    x = normalize(img)
    if bf16:
        x = _bf16(x)

    def _conv_bn(*a, **k):
        return _conv_bn_(*a, bf16=bf16, **k)

    x = _conv_bn(x, sd, "conv1", "bn1", 2, folded=folded)
    x = F.max_pool2d(x, 3, 2, 1)
    for L, n in enumerate(BLOCKS[depth], start=1):
        for blk in range(n):
            p = f"layer{L}.{blk}."
            stride = 2 if blk == 0 and L > 1 else 1
            res = x
            if p + ds + ".weight" in sd:
                res = _conv_bn(x, sd, p + ds, p + "downsample.1", stride, relu=False, folded=folded)
            if depth == 50:
                y = _conv_bn(x, sd, p + "conv1", p + "bn1", 1, folded=folded)
                if blk == 0 and L > 1:
                    taps.append(y)
                y = _conv_bn(y, sd, p + "conv2", p + "bn2", stride, folded=folded)
                x = _conv_bn(y, sd, p + "conv3", p + "bn3", 1, res=res, folded=folded)
            else:
                y = _conv_bn(x, sd, p + "conv1", p + "bn1", stride, folded=folded)
                x = _conv_bn(y, sd, p + "conv2", p + "bn2", 1, res=res, folded=folded)
        if depth == 18:
            taps.append(x)
    if depth == 50:
        taps.append(x)
    return {f"feat{i + 1}": t for i, t in enumerate(taps)}


def centroids(seg: torch.Tensor, smax: int) -> torch.Tensor:
    """(col, row) mean of each id's pixels of seg (H,W) as float32 of the float64 quotient (NaN for an absent id), the
    same numbers as the product's segment reduction."""
    H, W = seg.shape
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    s = seg.reshape(-1).cpu()
    ok = (s >= 0) & (s < smax)
    cnt = torch.zeros(smax, dtype=torch.float64).index_add_(0, s[ok], torch.ones(int(ok.sum()), dtype=torch.float64))
    sx = torch.zeros(smax, dtype=torch.float64).index_add_(0, s[ok], xs.reshape(-1)[ok])
    sy = torch.zeros(smax, dtype=torch.float64).index_add_(0, s[ok], ys.reshape(-1)[ok])
    return torch.stack((sx / cnt, sy / cnt), 1).float()


def pool_pyramid(seg: torch.Tensor, pyramid: dict, smax: int, centers: torch.Tensor = None) -> torch.Tensor:
    """seg (H,W) int64 ids, pyramid {feat_l: (1, C_l, h_l, w_l)} -> (smax, sum C_l): rows of ids without pixels are NaN."""
    H, W = seg.shape
    if centers is None:
        centers = centroids(seg, smax)
    centers = centers.cpu()
    rows = []
    levels = [v[0] for v in pyramid.values()]
    segs = [seg[:: H // f.shape[1], :: W // f.shape[2]] for f in levels]  # nearest: seg[i * H / h_l, j * W / w_l]
    for s in range(smax):
        cx, cy = centers[s].tolist()
        if cx != cx:
            rows.append(torch.full((sum(f.shape[0] for f in levels),), float("nan"), dtype=levels[0].dtype,
                                   device=levels[0].device))
            continue
        parts = []
        for f, sl in zip(levels, segs):
            m = sl == s
            if bool(m.any()):
                parts.append(f[:, m].mean(dim=1))
            else:
                h, w = f.shape[1:]
                i = min(max(int(torch.floor(torch.tensor(cy, dtype=torch.float32) / (H // h))), 0), h - 1)
                j = min(max(int(torch.floor(torch.tensor(cx, dtype=torch.float32) / (W // w))), 0), w - 1)
                parts.append(f[:, i, j])
        rows.append(torch.cat(parts))
    return torch.stack(rows)
