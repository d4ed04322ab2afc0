"""ORACLE (test infrastructure only) — restatement of the STEGO segmentation head and probes.

The arithmetic lives in the external ``stego`` package (``stego.stego.Stego``), absent from
the reference repository; call sites: ``feature_extractor/stego_interface.py:43,91-100,107-109``.
Restated from the public STEGO code [EXTERNAL-RECALLED, SURVEY.md §8 a4]:

* ``segmentation_head``: ``cluster1 = Conv2d(C, dim, 1)``; ``cluster2 = Conv2d(C, C, 1) -> ReLU ->
  Conv2d(C, dim, 1)``; ``code = cluster1(feats) + cluster2(feats)``   (dim = 90 in WVN)
* ``get_code(img)``: ``(code(img) + code(img.flip(3)).flip(3)) / 2`` (horizontal-flip TTA)
* ``postprocess``: ``code = F.interpolate(code, img.shape[-2:], 'bilinear', align_corners=False)``;
  cluster probe = argmax_n <normalize(code), normalize(clusters_n)>; linear probe =
  argmax(Conv2d(dim, n_classes, 1)(code)); CRF off (WVN default ``run_crf=False``).
  Per-image k-means (``run_clustering=True``, WVN's default: feature_extractor.py:47-53): ``image_kmeans`` below.
* ``StegoInterface.inference`` then upsamples code bilinear(align_corners=True) to (H, H) and the
  predictions 'nearest' to (H, H) as int.

PARITY STATUS: the head / probe arithmetic is "parity unpinned" (no upstream weights or golden outputs exist in
the reference); the reference's own wrapper around it (transform, (H, H) interpolation rules, int cast, return order)
IS pinned: tests/golden/stego_wrapper.pt is produced by running the reference's StegoInterface.inference around a shim
model built from the functions below (make_golden.py).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def synthetic_head(dim_in: int, code_dim: int = 90, n_clusters: int = 32, n_classes: int = 27, seed: int = 3) -> dict:
    g = torch.Generator().manual_seed(seed)

    def n(*shape, std):
        return torch.randn(*shape, generator=g) * std

    return {
        "cluster1.0.weight": n(code_dim, dim_in, std=0.05),
        "cluster1.0.bias": n(code_dim, std=0.05),
        "cluster2.0.weight": n(dim_in, dim_in, std=0.05),
        "cluster2.0.bias": n(dim_in, std=0.05),
        "cluster2.2.weight": n(code_dim, dim_in, std=0.05),
        "cluster2.2.bias": n(code_dim, std=0.05),
        "cluster_probe.clusters": n(n_clusters, code_dim, std=1.0),
        "linear_probe.weight": n(n_classes, code_dim, std=0.3),
        "linear_probe.bias": n(n_classes, std=0.1),
    }


@torch.no_grad()
def head_code(feats: torch.Tensor, hd: dict) -> torch.Tensor:
    """feats: (B, C, h, w) -> code (B, dim, h, w)."""
    def conv(x, w, b):
        return F.conv2d(x, w[:, :, None, None], b)

    c1 = conv(feats, hd["cluster1.0.weight"], hd["cluster1.0.bias"])
    h = F.relu(conv(feats, hd["cluster2.0.weight"], hd["cluster2.0.bias"]))
    c2 = conv(h, hd["cluster2.2.weight"], hd["cluster2.2.bias"])
    return c1 + c2


@torch.no_grad()
def postprocess(code: torch.Tensor, out_hw: tuple[int, int], hd: dict):
    """Returns (cluster_pred, linear_pred), each (B, H, W) long, computed the upstream way:
    upsample the code first, then run the probes per pixel."""
    code = F.interpolate(code, out_hw, mode="bilinear", align_corners=False)
    normed_clusters = F.normalize(hd["cluster_probe.clusters"], dim=1)
    normed_features = F.normalize(code, dim=1)
    inner = torch.einsum("bchw,nc->bnhw", normed_features, normed_clusters)
    cluster_pred = inner.argmax(1)
    lin = F.conv2d(code, hd["linear_probe.weight"][:, :, None, None], hd["linear_probe.bias"])
    linear_pred = lin.argmax(1)
    return cluster_pred, linear_pred


@torch.no_grad()
def image_kmeans(code: torch.Tensor, n_clusters: int, iters: int = 10) -> torch.Tensor:
    """Per-image k-means of the code, ``Stego.postprocess(image_clustering=True)`` with ``n_image_clusters`` clusters
    (call site: stego_interface.py:43,91-100).  [EXTERNAL-RECALLED]: the upstream routine is not in the reference repository and
    pins nothing (its initialisation is random); restated as plain Lloyd iterations — Euclidean distance, ``iters``
    iterations, initial centroids = the codes of ``n_clusters`` patches evenly spaced over the token sequence
    (index ``(2k+1) P / (2K)``), an empty cluster keeps its centroid — over the code at patch resolution.
    code: (B, C, h, w) -> centroids (B, K, C)."""
    B, C, h, w = code.shape
    x = code.flatten(2).transpose(1, 2)                                   # (B, P, C)
    P = h * w
    idx = ((2 * torch.arange(n_clusters, device=code.device) + 1) * P) // (2 * n_clusters)
    cent = x[:, idx].clone()                                              # (B, K, C)
    for _ in range(iters):
        score = x @ cent.transpose(1, 2) - 0.5 * (cent**2).sum(-1)[:, None, :]   # argmax == argmin of the distance
        assign = score.argmax(-1)                                         # (B, P), first maximum wins
        one_hot = torch.nn.functional.one_hot(assign, n_clusters).to(x.dtype)    # (B, P, K)
        cnt = one_hot.sum(1)                                              # (B, K)
        sums = one_hot.transpose(1, 2) @ x                                # (B, K, C)
        cent = torch.where(cnt[..., None] > 0, sums / cnt[..., None].clamp_min(1), cent)
    return cent


@torch.no_grad()
def kmeans_predict(code: torch.Tensor, cent: torch.Tensor, out_hw: tuple[int, int]) -> torch.Tensor:
    """``postprocess``'s order of operations with the per-image centroids: upsample the code
    (bilinear, align_corners=False), then every pixel takes its nearest centroid.  -> (B, H, W) long."""
    up = F.interpolate(code, out_hw, mode="bilinear", align_corners=False)
    score = torch.einsum("bchw,bkc->bkhw", up, cent) - 0.5 * (cent**2).sum(-1)[:, :, None, None]
    return score.argmax(1)


@torch.no_grad()
def stego_inference(feats: torch.Tensor, feats_flipped: torch.Tensor | None, hd: dict, img_hw: tuple[int, int],
                    out_h: int | None = None, n_image_clusters: int = 0, kmeans_iters: int = 10):
    """feats: backbone map of the transformed image; feats_flipped: backbone map of its horizontal
    flip (None disables the flip TTA).  ``img_hw``: size of the TRANSFORMED image (what ``postprocess`` upsamples the
    code to, stego_interface.py:91-100); ``out_h``: height H of the ORIGINAL image — the wrapper's final outputs are
    (H, H) (stego_interface.py:104-109); defaults to img_hw[0] (no resize in the transform).
    ``n_image_clusters`` > 0 = WVN's ``run_clustering=True``.
    Returns (code_up (B,dim,H,H), cluster (B,H,H), linear (B,H,H))."""
    code = head_code(feats, hd)
    if feats_flipped is not None:
        code = (code + head_code(feats_flipped, hd).flip(dims=[3])) / 2
    H = img_hw[0] if out_h is None else out_h
    cluster, linear = postprocess(code, img_hw, hd)
    if n_image_clusters > 0:  # run_clustering=True: the cluster prediction comes from the per-image k-means
        cluster = kmeans_predict(code, image_kmeans(code, n_image_clusters, kmeans_iters), img_hw)
    code_up = F.interpolate(code, (H, H), mode="bilinear", align_corners=True)
    cluster = F.interpolate(cluster[None].float(), (H, H), mode="nearest").int()[0]
    linear = F.interpolate(linear[None].float(), (H, H), mode="nearest").int()[0]
    return code_up, cluster, linear
