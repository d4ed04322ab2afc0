"""Backbone / head weight sources.

The reference downloads DINO checkpoints from dl.fbaipublicfiles.com at construction
([EXTERNAL] stego.backbones.backbone.get_backbone) and STEGO Lightning checkpoints from disk
(stego_interface.py:23,43).  There is no network here, so:
  * ``pretrained_weights`` / ``$WVN_DINO_WEIGHTS`` may point at a DINO ``.pth`` state dict
    (keys cls_token, pos_embed, patch_embed.proj.*, blocks.N.*, norm.*), which is used as is;
  * otherwise seeded DINO-style random weights are generated (SURVEY.md §8d) — results are then
    numerically meaningful only for parity / throughput work, and a warning says so.
DINOv2 (``backbone="dinov2"``, the ``dinov2_vit{s,b,l}14_pretrain.pth`` checkpoints) uses the same key names plus the
LayerScale gammas ``blocks.N.ls{1,2}.gamma`` and an unused ``mask_token``; DINOv2 with registers
(``backbone="dinov2_reg"``, ``dinov2_vit{s,b,l,g}14_reg4_pretrain.pth``) adds ``register_tokens`` (1, R, D).  ViT-L/14
(``backbone_type="vit_large"``) and ViT-g/14 (``backbone_type="vit_giant"``, ``dinov2_vitg14{,_reg4}_pretrain.pth``)
exist for DINOv2 only.  ViT-g/14's FFN is SwiGLU (``SwiGLUFFNFused``): ``blocks.N.mlp.w12`` (2 H rows: the gate half,
then the value half) and ``blocks.N.mlp.w3`` in place of ``mlp.fc1`` / ``mlp.fc2``, hidden width
H = (int(4 D 2 / 3) + 7) // 8 * 8 = 4096.  The name ``vit_giant`` follows the ``vit_small`` / ``vit_base`` /
``vit_large`` pattern; the name upstream STEGO's ``get_backbone`` would give this model is not known here.
The torchvision ResNets (``TorchVisionInterface``) take torchvision-layout state dicts (``resnet18`` / ``resnet50``
ImageNet checkpoints, or DINO's ``dino_resnet50_pretrain.pth`` for ``resnet50_dino``); ``fc.*`` is not needed.
EfficientNet-B0 (``efficientnet_b0``) takes torchvision-layout ``efficientnet_b0`` state dicts; ``classifier.*`` is not
needed.
"""
from __future__ import annotations

import math
import os
import warnings

import torch

VIT_SHAPES = {
    "vit_small": dict(dim=384, depth=12, heads=6, mlp_dim=1536),
    "vit_base": dict(dim=768, depth=12, heads=12, mlp_dim=3072),
    "vit_large": dict(dim=1024, depth=24, heads=16, mlp_dim=4096),
    # SwiGLU FFN: mlp_dim is the hidden width H of w3(silu(x1) * x2), [x1 | x2] = w12(x) (2 H wide)
    "vit_giant": dict(dim=1536, depth=40, heads=24, mlp_dim=4096, ffn="swiglu"),
}
# DINO v1 is released as ViT-S and ViT-B only; ViT-L and ViT-g exist for DINOv2 (with and without registers)
DINO_V1_TYPES = ("vit_small", "vit_base")


def vit_ffn(backbone_type: str) -> str:
    """"mlp" (fc2(GELU(fc1(x)))) or "swiglu" (w3(silu(x1) * x2)), the FFN of every block of ``backbone_type``."""
    return VIT_SHAPES[backbone_type].get("ffn", "mlp")


def check_backbone_type(backbone: str, backbone_type: str) -> None:
    """Raises ValueError for a ``backbone_type`` outside VIT_SHAPES or one that ``backbone`` is not released at."""
    if backbone_type not in VIT_SHAPES:
        raise ValueError(f"backbone_type '{backbone_type}' is not supported ({', '.join(VIT_SHAPES)})")
    if backbone == "dino" and backbone_type not in DINO_V1_TYPES:
        raise ValueError(f"backbone 'dino' has no '{backbone_type}' (DINO is released as {' and '.join(DINO_V1_TYPES)}); "
                         f"pass backbone='dinov2' or backbone='dinov2_reg'")


def synthetic_dino_state_dict(dim, depth, mlp_dim, patch_size, pretrain_grid, seed=1, attn_std=0.09):
    g = torch.Generator().manual_seed(seed)

    def n(*shape, std):
        return torch.randn(*shape, generator=g) * std

    sd = {
        "cls_token": n(1, 1, dim, std=0.02),
        "pos_embed": n(1, 1 + pretrain_grid**2, dim, std=0.02),
        "patch_embed.proj.weight": n(dim, 3, patch_size, patch_size, std=0.05),
        "patch_embed.proj.bias": n(dim, std=0.02),
        "norm.weight": 1.0 + n(dim, std=0.05),
        "norm.bias": n(dim, std=0.02),
    }
    for i in range(depth):
        b = f"blocks.{i}."
        sd[b + "norm1.weight"] = 1.0 + n(dim, std=0.05)
        sd[b + "norm1.bias"] = n(dim, std=0.02)
        sd[b + "attn.qkv.weight"] = n(3 * dim, dim, std=attn_std)
        sd[b + "attn.qkv.bias"] = n(3 * dim, std=0.02)
        sd[b + "attn.proj.weight"] = n(dim, dim, std=0.02)
        sd[b + "attn.proj.bias"] = n(dim, std=0.02)
        sd[b + "norm2.weight"] = 1.0 + n(dim, std=0.05)
        sd[b + "norm2.bias"] = n(dim, std=0.02)
        sd[b + "mlp.fc1.weight"] = n(mlp_dim, dim, std=0.04)
        sd[b + "mlp.fc1.bias"] = n(mlp_dim, std=0.02)
        sd[b + "mlp.fc2.weight"] = n(dim, mlp_dim, std=0.02)
        sd[b + "mlp.fc2.bias"] = n(dim, std=0.02)
    return sd


# DINOv2 is released at patch 14 only, pre-trained at 518 x 518 (a 37 x 37 position-embedding grid)
DINOV2_PATCH, DINOV2_PRETRAIN_GRID = 14, 37


def synthetic_swiglu_state_dict(dim, depth, hidden, seed=1, attn_std=0.09, device="cpu"):
    """Seeded DINOv2 ViT-g-layout weights with a SwiGLU FFN of hidden width ``hidden``: the DINOv2 layout at patch 14 /
    grid 37 with ``mlp.w12`` (2 hidden x dim) / ``mlp.w3`` (dim x hidden) for ``mlp.fc1`` / ``mlp.fc2``, LayerScale
    gammas and the (unused) ``mask_token``.  Every tensor is drawn on ``device`` from one generator there, so a full
    ViT-g/14 (4.5 GB in fp32) never passes through host memory when ``device`` is a GPU."""
    g = torch.Generator(device=device).manual_seed(seed)

    def n(*shape, std):
        return torch.randn(*shape, generator=g, device=device) * std

    def u(*shape):
        return 0.1 + 0.9 * torch.rand(*shape, generator=g, device=device)

    sd = {
        "cls_token": n(1, 1, dim, std=0.02),
        "pos_embed": n(1, 1 + DINOV2_PRETRAIN_GRID**2, dim, std=0.02),
        "patch_embed.proj.weight": n(dim, 3, DINOV2_PATCH, DINOV2_PATCH, std=0.05),
        "patch_embed.proj.bias": n(dim, std=0.02),
        "norm.weight": 1.0 + n(dim, std=0.05),
        "norm.bias": n(dim, std=0.02),
        "mask_token": torch.zeros(1, dim, device=device),
    }
    for i in range(depth):
        b = f"blocks.{i}."
        sd[b + "norm1.weight"] = 1.0 + n(dim, std=0.05)
        sd[b + "norm1.bias"] = n(dim, std=0.02)
        sd[b + "attn.qkv.weight"] = n(3 * dim, dim, std=attn_std)
        sd[b + "attn.qkv.bias"] = n(3 * dim, std=0.02)
        sd[b + "attn.proj.weight"] = n(dim, dim, std=0.02)
        sd[b + "attn.proj.bias"] = n(dim, std=0.02)
        sd[b + "ls1.gamma"] = u(dim)
        sd[b + "norm2.weight"] = 1.0 + n(dim, std=0.05)
        sd[b + "norm2.bias"] = n(dim, std=0.02)
        sd[b + "mlp.w12.weight"] = n(2 * hidden, dim, std=0.04)
        sd[b + "mlp.w12.bias"] = n(2 * hidden, std=0.02)
        sd[b + "mlp.w3.weight"] = n(dim, hidden, std=0.02)
        sd[b + "mlp.w3.bias"] = n(dim, std=0.02)
        sd[b + "ls2.gamma"] = u(dim)
    return sd


def synthetic_dinov2_state_dict(dim, depth, mlp_dim, seed=1, attn_std=0.09, ffn="mlp", device="cpu"):
    """Seeded DINOv2-layout weights: the DINO layout at patch 14 / grid 37 plus ``blocks.N.ls{1,2}.gamma`` and the
    (unused) ``mask_token``.  The LayerScale gammas vary per channel and are drawn independently for ls1 and ls2, so a
    missing or swapped LayerScale changes the tokens far beyond the parity tolerance.  ``ffn="swiglu"`` gives ViT-g's
    layout (synthetic_swiglu_state_dict, drawn on ``device``)."""
    if ffn == "swiglu":
        return synthetic_swiglu_state_dict(dim, depth, mlp_dim, seed, attn_std, device)
    sd = synthetic_dino_state_dict(dim, depth, mlp_dim, DINOV2_PATCH, DINOV2_PRETRAIN_GRID, seed, attn_std)
    g = torch.Generator().manual_seed(seed + 1)
    for i in range(depth):
        sd[f"blocks.{i}.ls1.gamma"] = 0.1 + 0.9 * torch.rand(dim, generator=g)
        sd[f"blocks.{i}.ls2.gamma"] = 0.1 + 0.9 * torch.rand(dim, generator=g)
    sd["mask_token"] = torch.zeros(1, dim)
    return sd


# Every released DINOv2 *_reg checkpoint has 4 register tokens
DINOV2_REGISTERS = 4
# std of the seeded register tokens, that of cls_token and pos_embed.  The final LayerNorm and every block's norm1 see
# only a register's direction, so its scale barely sets how much the patch tokens attend to it; what it sets is how
# much an added pos[0] turns it: at 0.02 that moves the ViT-S/14 tokens at 224 by about 0.1 rel-L2, as much as zeroing
# (0.1) or dropping (0.08) the registers, while at std 1 the same pos[0] moves them by less than 5e-3.
DINOV2_REGISTER_STD = 0.02


def synthetic_dinov2_reg_state_dict(dim, depth, mlp_dim, seed=1, attn_std=0.09, registers=DINOV2_REGISTERS,
                                    ffn="mlp", device="cpu"):
    """Seeded DINOv2-with-registers weights: ``synthetic_dinov2_state_dict`` plus ``register_tokens`` (1, R, dim), drawn
    from their own generator (seed + 2) with std DINOV2_REGISTER_STD."""
    sd = synthetic_dinov2_state_dict(dim, depth, mlp_dim, seed, attn_std, ffn, device)
    g = torch.Generator().manual_seed(seed + 2)
    sd["register_tokens"] = (torch.randn(1, registers, dim, generator=g) * DINOV2_REGISTER_STD).to(device)
    return sd


_FFN_NAME = {"mlp": "GELU MLP", "swiglu": "SwiGLU FFN"}


def _vit_size(dim: int, depth: int, ffn: str = None) -> str:
    """Names a ViT size; with ``ffn``, a size whose FFN differs is named by its shape and FFN."""
    name = next((k for k, v in VIT_SHAPES.items() if (v["dim"], v["depth"]) == (dim, depth)
                 and (ffn is None or vit_ffn(k) == ffn)), None)
    kind = "" if ffn is None else f", {_FFN_NAME[ffn]}"
    return f"{name} (D = {dim}, {depth} blocks{kind})" if name else f"D = {dim} with {depth} blocks{kind}"


def check_backbone_family(sd: dict, backbone: str, backbone_type: str = None) -> dict:
    """Checks that a ViT state dict belongs to ``backbone`` ("dino": DINO v1, "dinov2": DINOv2 without registers,
    "dinov2_reg": DINOv2 with register tokens) and, when ``backbone_type`` is given, has its width and depth; returns it
    with the keys the backbone does not use dropped (DINOv2's ``mask_token``).  Raises ValueError on a checkpoint of
    another family or size."""
    sd = {k.replace("module.", "").replace("backbone.", ""): v for k, v in sd.items()}
    if backbone_type is not None:
        shp = VIT_SHAPES[backbone_type]
        dim = int(sd["patch_embed.proj.weight"].shape[0])
        depth = len({k.split(".")[1] for k in sd if k.startswith("blocks.")})
        if (dim, depth) != (shp["dim"], shp["depth"]):
            raise ValueError(f"backbone_type '{backbone_type}' needs a {_vit_size(shp['dim'], shp['depth'])} checkpoint; "
                             f"got {_vit_size(dim, depth)}")
        ffn = "swiglu" if "blocks.0.mlp.w12.weight" in sd else "mlp"
        if ffn != vit_ffn(backbone_type):
            want = _vit_size(shp["dim"], shp["depth"], vit_ffn(backbone_type))
            raise ValueError(f"backbone_type '{backbone_type}' needs a {want} checkpoint; "
                             f"got {_vit_size(dim, depth, ffn)}")
    has_reg = "register_tokens" in sd
    has_ls = "blocks.0.ls1.gamma" in sd
    patch = int(sd["patch_embed.proj.weight"].shape[-1])
    if backbone in ("dinov2", "dinov2_reg"):
        if not has_ls or patch != DINOV2_PATCH:
            raise ValueError(f"backbone '{backbone}' needs a DINOv2 checkpoint (LayerScale 'ls1.gamma' and a 14x14 patch "
                             f"conv); got one with{'' if has_ls else 'out'} LayerScale and a {patch}x{patch} patch conv")
        if backbone == "dinov2" and has_reg:
            raise ValueError("backbone 'dinov2' got a checkpoint with register tokens (DINOv2 *_reg): pass "
                             "backbone='dinov2_reg'")
        if backbone == "dinov2_reg" and not has_reg:
            raise ValueError("backbone 'dinov2_reg' needs a checkpoint with register tokens ('register_tokens'): pass "
                             "backbone='dinov2' for the DINOv2 checkpoints without them")
        return {k: v for k, v in sd.items() if k != "mask_token"}
    if has_ls or has_reg or "mask_token" in sd:
        raise ValueError("backbone 'dino' got a DINOv2 checkpoint (LayerScale gammas / mask_token / register tokens): "
                         "pass backbone='dinov2' or backbone='dinov2_reg'")
    return sd


def load_dino_state_dict(backbone_type: str, patch_size: int, pretrained_weights=None, seed: int = 1,
                         backbone: str = "dino", device="cpu"):
    """DINO (``backbone="dino"``), DINOv2 (``"dinov2"``) or DINOv2 with registers (``"dinov2_reg"``; both always patch
    14) weights, from ``pretrained_weights`` / ``$WVN_DINO_WEIGHTS`` or seeded.  A checkpoint is checked against the
    family (check_backbone_family).  Seeded ViT-g weights are drawn on ``device``; the others on the host."""
    check_backbone_type(backbone, backbone_type)
    shp = VIT_SHAPES[backbone_type]
    path = pretrained_weights or os.environ.get("WVN_DINO_WEIGHTS")
    if path:
        sd = torch.load(path, map_location="cpu", weights_only=False)  # DINO full checkpoints pickle argparse objects
        if "state_dict" in sd:
            sd = sd["state_dict"]
        if "teacher" in sd:
            sd = sd["teacher"]
        return check_backbone_family(sd, backbone, backbone_type)
    warnings.warn(f"no {backbone.upper()} checkpoint given (pretrained_weights / $WVN_DINO_WEIGHTS): using seeded random "
                  f"{backbone.upper()}-style weights — fine for parity and throughput work, not for real traversability")
    kw = dict(ffn="swiglu", device=device) if vit_ffn(backbone_type) == "swiglu" else {}
    if backbone == "dinov2":
        return synthetic_dinov2_state_dict(shp["dim"], shp["depth"], shp["mlp_dim"], seed, **kw)
    if backbone == "dinov2_reg":
        return synthetic_dinov2_reg_state_dict(shp["dim"], shp["depth"], shp["mlp_dim"], seed, **kw)
    return synthetic_dino_state_dict(shp["dim"], shp["depth"], shp["mlp_dim"], patch_size, 224 // patch_size, seed)


def synthetic_stego_head(dim_in: int, code_dim: int = 90, n_clusters: int = 32, n_classes: int = 27, seed: int = 3):
    g = torch.Generator().manual_seed(seed)

    def n(*shape, std):
        return torch.randn(*shape, generator=g) * std

    return {
        "cluster1.0.weight": n(code_dim, dim_in, std=0.05), "cluster1.0.bias": n(code_dim, std=0.05),
        "cluster2.0.weight": n(dim_in, dim_in, std=0.05), "cluster2.0.bias": n(dim_in, std=0.05),
        "cluster2.2.weight": n(code_dim, dim_in, std=0.05), "cluster2.2.bias": n(code_dim, std=0.05),
        "cluster_probe.clusters": n(n_clusters, code_dim, std=1.0),
        "linear_probe.weight": n(n_classes, code_dim, std=0.3), "linear_probe.bias": n(n_classes, std=0.1),
    }


# Column layout of the stacked STEGO head output (see wvn_vit_stego_head in include/wvn_b200.h)
HEAD_CODE_COL, HEAD_CLUSTER_COL, HEAD_LINEAR_COL, HEAD_OUT = 0, 128, 192, 256


def fold_stego_head(hd: dict) -> dict:
    """Stack code / cluster-probe / linear-probe into the two affine maps the CUDA head applies:
        out = head_a(t) + head_b(relu(hidden(t)))
    rows [0,90): code = cluster1(t) + cluster2.2(relu(cluster2.0(t)));
    rows [128,128+K): normalize(clusters) @ code  (cluster-probe logits up to a positive per-pixel scale);
    rows [192,192+C): linear_probe(code).
    Exact algebra in fp32 on the host (init-time), so no bf16 rounding of the code sits between
    the head and its probes."""
    w1, b1 = hd["cluster1.0.weight"].float(), hd["cluster1.0.bias"].float()
    w2, b2 = hd["cluster2.2.weight"].float(), hd["cluster2.2.bias"].float()
    cn = torch.nn.functional.normalize(hd["cluster_probe.clusters"].float(), dim=1)
    wl, bl = hd["linear_probe.weight"].float(), hd["linear_probe.bias"].float()
    code_dim, dim_in = w1.shape
    K, C = cn.shape[0], wl.shape[0]
    assert code_dim <= 128 and K <= 64 and C <= 64, "head layout supports code<=128, clusters<=64, classes<=64"
    a_w = torch.zeros(HEAD_OUT, dim_in)
    b_w = torch.zeros(HEAD_OUT, dim_in)
    a_b = torch.zeros(HEAD_OUT)
    a_w[:code_dim], b_w[:code_dim], a_b[:code_dim] = w1, w2, b1 + b2
    a_w[HEAD_CLUSTER_COL : HEAD_CLUSTER_COL + K] = cn @ w1
    b_w[HEAD_CLUSTER_COL : HEAD_CLUSTER_COL + K] = cn @ w2
    a_b[HEAD_CLUSTER_COL : HEAD_CLUSTER_COL + K] = cn @ (b1 + b2)
    a_w[HEAD_LINEAR_COL : HEAD_LINEAR_COL + C] = wl @ w1
    b_w[HEAD_LINEAR_COL : HEAD_LINEAR_COL + C] = wl @ w2
    a_b[HEAD_LINEAR_COL : HEAD_LINEAR_COL + C] = wl @ (b1 + b2) + bl
    return {"head_a.weight": a_w, "head_a.bias": a_b, "hidden.weight": hd["cluster2.0.weight"].float(),
            "hidden.bias": hd["cluster2.0.bias"].float(), "head_b.weight": b_w}


# --------------------------------------------------------------------------------------------
# torchvision ResNets
# --------------------------------------------------------------------------------------------
RESNET_MODELS = {"resnet18": 18, "resnet50": 50, "resnet50_dino": 50}
RESNET_BLOCKS = {18: (2, 2, 2, 2), 50: (3, 4, 6, 3)}
RESNET_BN_EPS = 1e-5
RESNET_RESIDUAL_GAMMA = 0.2


def resnet_convs(depth: int):
    """(conv, batch norm, in, out, kernel, stride) of every conv of the torchvision ResNet trunk, in forward order.
    The downsample conv of a stage's first block comes before the block's own convs."""
    convs = [("conv1", "bn1", 3, 64, 7, 2)]
    bottleneck = depth == 50
    cin = 64
    for L, n in enumerate(RESNET_BLOCKS[depth], start=1):
        planes = 64 << (L - 1)
        cout = planes * 4 if bottleneck else planes
        for blk in range(n):
            p = f"layer{L}.{blk}."
            stride = 2 if blk == 0 and L > 1 else 1
            if blk == 0 and (stride != 1 or cin != cout):
                convs.append((p + "downsample.0", p + "downsample.1", cin, cout, 1, stride))
            if bottleneck:
                # torchvision >= 0.13 (ResNet v1.5): the stride sits in the 3 x 3 conv
                convs += [(p + "conv1", p + "bn1", cin, planes, 1, 1), (p + "conv2", p + "bn2", planes, planes, 3, stride),
                          (p + "conv3", p + "bn3", planes, cout, 1, 1)]
            else:
                convs += [(p + "conv1", p + "bn1", cin, planes, 3, stride), (p + "conv2", p + "bn2", planes, cout, 3, 1)]
            cin = cout
    return convs


def _resnet_calibrate(sd: dict, depth: int, img: torch.Tensor):
    """Runs the trunk in training-mode batch norm on ``img`` and stores each batch norm's batch statistics as its running
    statistics (momentum 1, each layer seeing the already calibrated layers before it)."""
    import torch.nn.functional as F

    def cbr(x, conv, bn, stride, k, relu=True, res=None):
        x = F.conv2d(x, sd[conv + ".weight"], stride=stride, padding=k // 2)
        mean, var = x.mean((0, 2, 3)), x.var((0, 2, 3), unbiased=False)
        sd[bn + ".running_mean"], sd[bn + ".running_var"] = mean, var
        x = F.batch_norm(x, mean, var, sd[bn + ".weight"], sd[bn + ".bias"], False, 0.0, RESNET_BN_EPS)
        if res is not None:
            x = x + res
        return F.relu(x) if relu else x

    x = (img - torch.tensor([0.485, 0.456, 0.406])[:, None, None]) / torch.tensor([0.229, 0.224, 0.225])[:, None, None]
    x = F.max_pool2d(cbr(x, "conv1", "bn1", 2, 7), 3, 2, 1)
    for L, n in enumerate(RESNET_BLOCKS[depth], start=1):
        for blk in range(n):
            p = f"layer{L}.{blk}."
            stride = 2 if blk == 0 and L > 1 else 1
            res = x
            if p + "downsample.0.weight" in sd:
                res = cbr(x, p + "downsample.0", p + "downsample.1", stride, 1, relu=False)
            if depth == 50:
                y = cbr(x, p + "conv1", p + "bn1", 1, 1)
                y = cbr(y, p + "conv2", p + "bn2", stride, 3)
                x = cbr(y, p + "conv3", p + "bn3", 1, 1, res=res)
            else:
                y = cbr(x, p + "conv1", p + "bn1", stride, 3)
                x = cbr(y, p + "conv2", p + "bn2", 1, 3, res=res)


def synthetic_resnet_state_dict(depth: int, seed: int = 1):
    """Seeded torchvision-layout ResNet weights (no ``fc``).  Convs are Kaiming-normal (fan_out, as torchvision
    initialises them), batch-norm affine parameters are drawn around (1, 0), and the running statistics are calibrated
    on four seeded 128 x 128 images, so every tap keeps an RMS of order 1 at any input size instead of growing through
    the residual sums as it does with identity statistics."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    with torch.no_grad():
        for conv, bn, cin, cout, k, _ in resnet_convs(depth):
            sd[conv + ".weight"] = torch.randn(cout, cin, k, k, generator=g) * math.sqrt(2.0 / (cout * k * k))
            # the batch norm closing a residual branch starts small (torchvision's zero_init_residual takes it to 0):
            # each block adds a correction to its input instead of replacing it.  With gamma 1 a random calibrated
            # trunk amplifies any perturbation about 1.2x per conv, so bf16 activations would end 47% off fp32 at
            # ResNet-50's trunk output; at 0.2 they end 3.8% off (DESIGN.md §3.9)
            last = bn.endswith(".bn3" if depth == 50 else ".bn2")
            sd[bn + ".weight"] = (RESNET_RESIDUAL_GAMMA if last else 1.0) * (1.0 + 0.2 * torch.randn(cout, generator=g))
            sd[bn + ".bias"] = 0.2 * torch.randn(cout, generator=g)
            sd[bn + ".running_mean"] = torch.zeros(cout)
            sd[bn + ".running_var"] = torch.ones(cout)
            sd[bn + ".num_batches_tracked"] = torch.tensor(0)
        _resnet_calibrate(sd, depth, torch.rand(4, 3, 128, 128, generator=g))
    return sd


def check_resnet_family(sd: dict, model_type: str) -> dict:
    """Checks that a torchvision-layout state dict is a ``model_type`` ResNet and returns the trunk's tensors (the
    reference loads with ``strict=False``, so a missing ``fc.*`` is fine).  Raises ValueError on another family."""
    if model_type not in RESNET_MODELS:
        raise ValueError(f"model_type '{model_type}' is not supported (resnet18, resnet50, resnet50_dino)")
    depth = RESNET_MODELS[model_type]
    sd = {k.replace("module.", ""): v for k, v in sd.items()}
    missing, bad = [], []
    for conv, bn, cin, cout, k, _ in resnet_convs(depth):
        w = sd.get(conv + ".weight")
        if w is None:
            missing.append(conv + ".weight")
        elif tuple(w.shape) != (cout, cin, k, k):
            bad.append(f"{conv}.weight {tuple(w.shape)} != {(cout, cin, k, k)}")
        for leaf in ("weight", "bias", "running_mean", "running_var"):
            if bn + "." + leaf not in sd:
                missing.append(bn + "." + leaf)
    if missing or bad:
        detail = "; ".join((bad + [f"missing {m}" for m in missing])[:3])
        raise ValueError(f"model_type '{model_type}' needs a torchvision ResNet-{depth} state dict; got another ({detail})")
    keep = {c + ".weight" for c, *_ in resnet_convs(depth)}
    keep |= {b + "." + leaf for _, b, *_ in resnet_convs(depth) for leaf in ("weight", "bias", "running_mean", "running_var")}
    return {k: v for k, v in sd.items() if k in keep}


def load_resnet_state_dict(model_type: str, pretrained_weights=None, seed: int = 1):
    """ResNet weights for ``model_type`` from ``pretrained_weights`` / ``$WVN_RESNET_WEIGHTS`` (checked by
    check_resnet_family), or seeded (synthetic_resnet_state_dict) with a warning."""
    if model_type not in RESNET_MODELS:
        raise ValueError(f"model_type '{model_type}' is not supported (resnet18, resnet50, resnet50_dino)")
    path = pretrained_weights or os.environ.get("WVN_RESNET_WEIGHTS")
    if path:
        sd = torch.load(path, map_location="cpu", weights_only=False)
        if "state_dict" in sd:
            sd = sd["state_dict"]
        return check_resnet_family(sd, model_type)
    warnings.warn(f"no {model_type} checkpoint given (pretrained_weights / $WVN_RESNET_WEIGHTS): using seeded random "
                  f"weights with calibrated batch-norm statistics — fine for parity and throughput work, not for real "
                  f"traversability")
    return synthetic_resnet_state_dict(RESNET_MODELS[model_type], seed)


def fold_resnet_bn(sd: dict, depth: int) -> dict:
    """Eval-mode batch norm folded into the conv before it, in at least fp32 (fp64 stays fp64):
    w' = w * gamma / sqrt(var + eps) per output channel, b' = beta - mean * gamma / sqrt(var + eps).
    Returns {conv name: (w', b')} with the downsample conv named ``layer{L}.0.downsample``."""
    out = {}
    for conv, bn, *_ in resnet_convs(depth):
        w = sd[conv + ".weight"]
        dt = torch.promote_types(w.dtype, torch.float32)
        gamma, beta, mean, var = (sd[bn + "." + k].to(dt) for k in ("weight", "bias", "running_mean", "running_var"))
        scale = gamma / torch.sqrt(var + RESNET_BN_EPS)
        out[conv.replace("downsample.0", "downsample")] = (w.to(dt) * scale[:, None, None, None], beta - mean * scale)
    return out


# --------------------------------------------------------------------------------------------
# torchvision EfficientNet-B0
# --------------------------------------------------------------------------------------------
EFFNET_MODELS = ("efficientnet_b0",)
# (expand ratio, kernel, stride, output channels, blocks) of the seven stages
EFFNET_B0_STAGES = ((1, 3, 1, 16, 1), (6, 3, 2, 24, 2), (6, 5, 2, 40, 2), (6, 3, 2, 80, 3), (6, 5, 1, 112, 3),
                    (6, 5, 2, 192, 4), (6, 3, 1, 320, 1))
EFFNET_BN_EPS = 1e-5
EFFNET_RESIDUAL_GAMMA = 0.2


def efficientnet_b0_blocks():
    """(prefix, in, expanded, out, kernel, stride, squeeze) of every MBConv block, prefix ``features.{s}.{i}.block.``."""
    blocks, cin = [], 32
    for s, (ratio, k, stride, cout, n) in enumerate(EFFNET_B0_STAGES, start=1):
        for i in range(n):
            blocks.append((f"features.{s}.{i}.block.", cin, cin * ratio, cout, k, stride if i == 0 else 1,
                           max(1, cin // 4)))
            cin = cout
    return blocks


def efficientnet_b0_layers():
    """Every parameterised layer of the B0 trunk in forward order: ("conv", module, out, in per group, kernel) for a
    conv + batch norm pair (conv ``{module}.0``, batch norm ``{module}.1``; depthwise convs have 1 input per group) and
    ("se", module, expanded, squeeze) for a squeeze-excitation (``{module}.fc1``, ``{module}.fc2``)."""
    layers = [("conv", "features.0", 32, 3, 3)]
    for p, cin, cexp, cout, k, _, sq in efficientnet_b0_blocks():
        j = 0
        if cexp != cin:
            layers.append(("conv", p + "0", cexp, cin, 1))
            j = 1
        layers += [("conv", p + str(j), cexp, 1, k), ("se", p + str(j + 1), cexp, sq),
                   ("conv", p + str(j + 2), cout, cexp, 1)]
    layers.append(("conv", "features.8", 1280, 320, 1))
    return layers


def _effnet_forward(sd: dict, x: torch.Tensor, calibrate: bool):
    """The B0 trunk on a normalised image in eval-mode batch norm, or with ``calibrate`` in training-mode batch norm,
    each batch norm's batch statistics stored as its running statistics (the layers before it already calibrated)."""
    import torch.nn.functional as F

    def cbn(x, m, stride=1, groups=1, act=True):
        w = sd[m + ".0.weight"]
        x = F.conv2d(x, w, stride=stride, padding=(w.shape[-1] - 1) // 2, groups=groups)
        bn = m + ".1."
        if calibrate:
            sd[bn + "running_mean"], sd[bn + "running_var"] = x.mean((0, 2, 3)), x.var((0, 2, 3), unbiased=False)
        x = F.batch_norm(x, sd[bn + "running_mean"], sd[bn + "running_var"], sd[bn + "weight"], sd[bn + "bias"], False,
                         0.0, EFFNET_BN_EPS)
        return F.silu(x) if act else x

    x = cbn(x, "features.0", stride=2)
    for p, cin, cexp, cout, k, stride, _ in efficientnet_b0_blocks():
        j = 0
        y = x
        if cexp != cin:
            y = cbn(y, p + "0")
            j = 1
        y = cbn(y, p + str(j), stride=stride, groups=cexp)
        se = p + str(j + 1)
        g = F.silu(F.conv2d(y.mean((2, 3), keepdim=True), sd[se + ".fc1.weight"], sd[se + ".fc1.bias"]))
        y = y * torch.sigmoid(F.conv2d(g, sd[se + ".fc2.weight"], sd[se + ".fc2.bias"]))
        y = cbn(y, p + str(j + 2), act=False)
        x = x + y if stride == 1 and cin == cout else y
    return cbn(x, "features.8")


def synthetic_efficientnet_b0_state_dict(seed: int = 1):
    """Seeded torchvision-layout EfficientNet-B0 weights (no ``classifier``).  Convs are Kaiming-normal (fan_out, as
    torchvision initialises them), batch-norm affine parameters are drawn around (1, 0) (around (0.2, 0) for the
    project conv of a residual block, so that each such block adds a correction to its input, see
    RESNET_RESIDUAL_GAMMA), the squeeze-excitation's biases around 0, and the running statistics are calibrated on four
    seeded 128 x 128 images, so that every tap keeps an RMS of order 1 through the 16 blocks."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    residual = {p + str(2 if cexp == cin else 3) for p, cin, cexp, cout, _, stride, _ in efficientnet_b0_blocks()
                if stride == 1 and cin == cout}
    with torch.no_grad():
        for kind, m, cout, cin, *rest in efficientnet_b0_layers():
            if kind == "se":
                sq = cin
                sd[m + ".fc1.weight"] = torch.randn(sq, cout, 1, 1, generator=g) * math.sqrt(2.0 / sq)
                sd[m + ".fc1.bias"] = 0.2 * torch.randn(sq, generator=g)
                sd[m + ".fc2.weight"] = torch.randn(cout, sq, 1, 1, generator=g) * math.sqrt(2.0 / cout)
                sd[m + ".fc2.bias"] = 0.2 * torch.randn(cout, generator=g)
                continue
            k = rest[0]
            fan_out = cout * k * k if cin > 1 or m == "features.0" else k * k
            sd[m + ".0.weight"] = torch.randn(cout, cin, k, k, generator=g) * math.sqrt(2.0 / fan_out)
            gamma = EFFNET_RESIDUAL_GAMMA if m in residual else 1.0
            sd[m + ".1.weight"] = gamma * (1.0 + 0.2 * torch.randn(cout, generator=g))
            sd[m + ".1.bias"] = 0.2 * torch.randn(cout, generator=g)
            sd[m + ".1.running_mean"] = torch.zeros(cout)
            sd[m + ".1.running_var"] = torch.ones(cout)
            sd[m + ".1.num_batches_tracked"] = torch.tensor(0)
        img = torch.rand(4, 3, 128, 128, generator=g)
        x = (img - torch.tensor([0.485, 0.456, 0.406])[:, None, None]) / torch.tensor([0.229, 0.224, 0.225])[:, None, None]
        _effnet_forward(sd, x, calibrate=True)
    return sd


def _effnet_param_shapes():
    shapes = {}
    for kind, m, cout, cin, *rest in efficientnet_b0_layers():
        if kind == "se":
            sq = cin
            shapes.update({m + ".fc1.weight": (sq, cout, 1, 1), m + ".fc1.bias": (sq,), m + ".fc2.weight": (cout, sq, 1, 1),
                           m + ".fc2.bias": (cout,)})
        else:
            shapes[m + ".0.weight"] = (cout, cin, rest[0], rest[0])
            shapes.update({m + ".1." + leaf: (cout,) for leaf in ("weight", "bias", "running_mean", "running_var")})
    return shapes


def check_efficientnet_family(sd: dict, model_type: str) -> dict:
    """Checks that a torchvision-layout state dict is an EfficientNet-B0 and returns the trunk's tensors
    (``classifier.*`` and ``num_batches_tracked`` are dropped).  Raises ValueError naming what it got instead."""
    if model_type not in EFFNET_MODELS:
        raise ValueError(f"model_type '{model_type}' is not supported (efficientnet_b0)")
    sd = {k.replace("module.", ""): v for k, v in sd.items()}
    shapes = _effnet_param_shapes()
    missing = [k for k in shapes if k not in sd]
    bad = [f"{k} {tuple(sd[k].shape)} != {shapes[k]}" for k in shapes if k in sd and tuple(sd[k].shape) != shapes[k]]
    if missing or bad:
        if "conv1.weight" in sd and "features.0.0.weight" not in sd:
            got = "a ResNet state dict"
        elif "features.0.0.weight" in sd and tuple(sd["features.0.0.weight"].shape) != shapes["features.0.0.weight"]:
            stem = sd["features.0.0.weight"].shape[0]
            got = {48: "an EfficientNet-B4 state dict", 64: "an EfficientNet-B7 state dict"}.get(
                stem, f"an EfficientNet with a {stem}-channel stem")
        else:
            got = "another"
        detail = "; ".join((bad + [f"missing {m}" for m in missing])[:3])
        raise ValueError(f"model_type '{model_type}' needs a torchvision EfficientNet-B0 state dict; got {got} ({detail})")
    return {k: sd[k] for k in shapes}


def load_efficientnet_state_dict(model_type: str, pretrained_weights=None, pretrained: bool = True, seed: int = 1):
    """EfficientNet-B0 weights from ``pretrained_weights`` / ``$WVN_EFFICIENTNET_WEIGHTS`` (a torchvision
    ``efficientnet_b0`` checkpoint, checked by check_efficientnet_family).  Without a checkpoint, ``pretrained=False``
    gives seeded weights (synthetic_efficientnet_b0_state_dict, with a warning), as torchvision's ``pretrained=False``
    gives random ones; ``pretrained=True`` asks for torchvision's ImageNet weights, which are only ever read from a
    checkpoint here, so it raises ValueError instead of quietly running random weights."""
    if model_type not in EFFNET_MODELS:
        raise ValueError(f"model_type '{model_type}' is not supported (efficientnet_b0)")
    path = pretrained_weights or os.environ.get("WVN_EFFICIENTNET_WEIGHTS")
    if path:
        sd = torch.load(path, map_location="cpu", weights_only=False)
        if "state_dict" in sd:
            sd = sd["state_dict"]
        return check_efficientnet_family(sd, model_type)
    if pretrained:
        raise ValueError(f"model_type '{model_type}' with pretrained=True needs torchvision's ImageNet checkpoint "
                         f"(state_dict, pretrained_weights or $WVN_EFFICIENTNET_WEIGHTS): downloading it is outside the "
                         f"H100 hot path; pass pretrained=False for seeded weights")
    warnings.warn(f"no {model_type} checkpoint given and pretrained=False: using seeded random weights with calibrated "
                  f"batch-norm statistics — fine for parity and throughput work, not for real traversability")
    return synthetic_efficientnet_b0_state_dict(seed)


def fold_efficientnet_bn(sd: dict) -> dict:
    """Eval-mode batch norm folded into the conv before it, in at least fp32 (fp64 stays fp64), as fold_resnet_bn.
    Returns {module: (w', b')} for every conv + batch norm pair (stem ``features.0``, head ``features.8``) and
    {``{module}.fc1`` / ``{module}.fc2``: (w [out, in], b)} for the squeeze-excitations."""
    out = {}
    for kind, m, *_ in efficientnet_b0_layers():
        if kind == "se":
            for fc in ("fc1", "fc2"):
                w = sd[f"{m}.{fc}.weight"]
                dt = torch.promote_types(w.dtype, torch.float32)
                out[f"{m}.{fc}"] = (w.to(dt)[:, :, 0, 0], sd[f"{m}.{fc}.bias"].to(dt))
            continue
        w = sd[m + ".0.weight"]
        dt = torch.promote_types(w.dtype, torch.float32)
        gamma, beta, mean, var = (sd[m + ".1." + k].to(dt) for k in ("weight", "bias", "running_mean", "running_var"))
        scale = gamma / torch.sqrt(var + EFFNET_BN_EPS)
        out[m] = (w.to(dt) * scale[:, None, None, None], beta - mean * scale)
    return out
