"""TEST INFRASTRUCTURE ONLY (see oracle/__init__.py) — numpy restatement of STEGO's dense CRF, the refinement behind
``StegoInterface(run_crf=True)`` (stego_interface.py:25, 94-100: ``Stego.postprocess(use_crf_cluster=...,
use_crf_linear=...)``).

RESTATED [EXTERNAL-RECALLED]: ``Stego.postprocess`` and ``dense_crf`` live in the un-vendored ``stego`` package, the
model in ``pydensecrf`` (Krähenbühl's densecrf).  Neither is installed, so this file is the definition the CUDA kernels
(csrc/dense_crf.cu) are held to.  What it commits to:

* Inputs.  The per-patch logits are upsampled bilinearly (align_corners=False) to the S x S transformed image.  Linear:
  the class logits.  Cluster: ``2 <normalize(code_px), normalize(c_k)>``, the code normalised per pixel after
  upsampling (F.normalize, eps 1e-12).  ``log_softmax`` followed by densecrf's softmax is the softmax of the logits.
* Image.  ``np.array(to_pil_image(unnorm(img)))[:, :, ::-1]``: the transformed image x = (v - mean) / std is
  un-normalised (x * std + mean), multiplied by 255 and truncated, all in float32 without fused multiply-adds, then read
  as BGR.  v is the fp32 input, or byte / 255 for camera frames.
* Unary.  ``U = -log(clip(softmax(logits), 1e-5, 1))`` (pydensecrf ``unary_from_softmax``).
* Model.  ``addPairwiseGaussian(sxy=1, compat=3)``: features (x, y) / 1; ``addPairwiseBilateral(sxy=67, srgb=3,
  compat=4)``: features (x/67, y/67, b/3, g/3, r/3), x the column and y the row, each a float32 division.  Potts
  compatibility, NORMALIZE_SYMMETRIC: ``norm = 1 / sqrt(K(1) + 1e-20)`` per pixel.
* Mean field, 10 iterations: ``Q0 = softmax(-U)``; ``Q = softmax(-U + sum_k w_k norm_k K_k(norm_k Q))``.
* K_k is the permutohedral-lattice Gaussian filter (Adams, Baek & Davis 2010) as densecrf builds it, in float32:
  - elevation: ``scale[i] = float(1 / sqrt((i+2)(i+1)) * float(sqrt(2/3) (d+1)))``; with ``cf_j = f_j scale_j``,
    ``E[j] = sum_{i>=j} cf_i - j cf_{j-1}`` accumulated from j = d down to 1 (``E[j] = sm - j*cf; sm += cf``) and
    ``E[0] = sm``;
  - remainder-0 point: ``v = E[i] * float(1/(d+1))``; the nearer of ``ceil(v)(d+1)`` and ``floor(v)(d+1)``, the floor
    on a tie (``up - E < E - down`` picks up);
  - rank: ``rank[i]`` counts the coordinates j with ``E[j]-rem0[j]`` above coordinate i's (ties go to the later index);
    plus ``sum(rem0) / (d+1)``, wrapped into [0, d] while moving rem0 by +-(d+1);
  - barycentric weights: for i = 0..d, ``v = (E[i]-rem0[i]) / (d+1)`` is added to ``b[d-rank[i]]`` and subtracted from
    ``b[d-rank[i]+1]``, then ``b[0] += 1 + b[d+1]`` (in double, rounded once to float);
  - vertex r (0..d) of a pixel has key ``key_i = rem0_i + (r if rank_i <= d-r else r-(d+1))`` for i < d (the last
    coordinate is implied) and weight ``b[r]``;
  - key layout: each coordinate biased by 2^(bits-1) in ``bits`` bits (16 for d = 2, 11 for d = 5), coordinate i at bit
    ``bits * i``, the frame above ``bits * d``; vertices are numbered in ascending packed-key order;
  - splat: each vertex sums ``w * value`` over its pixels; blur: for j = 0..d in that order,
    ``v' = v + 0.5 (v[n1] + v[n2])`` with ``n1 = key - 1, n1[j] = key[j] + d`` and ``n2 = key + 1, n2[j] = key[j] - d``
    (for j = d every coordinate moves by -1 / +1), a missing neighbour counting 0; slice: ``sum_r b[r] v[vertex r]``
    times ``1 / (1 + 2^-d)``.
Parity against pydensecrf is unpinned: neither package is available, so every detail above is recalled, not checked.
"""
from __future__ import annotations

import numpy as np

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
POS_XY_STD, POS_W = 1.0, 3.0
BI_XY_STD, BI_RGB_STD, BI_W = 67.0, 3.0, 4.0
MAX_ITER = 10
CLIP = 1e-5
KEY_BITS = {2: 16, 5: 11}


def crf_image_bytes(v: np.ndarray) -> np.ndarray:
    """v (3,H,W) float32 input in [0,1] (camera bytes: byte / 255 in float32) -> (H,W,3) uint8 BGR, the image
    ``dense_crf`` hands to the bilateral kernel."""
    v = v.astype(np.float32)
    m = np.asarray(IMAGENET_MEAN, np.float32)[:, None, None]
    s = np.asarray(IMAGENET_STD, np.float32)[:, None, None]
    x = (v - m) / s                       # torchvision Normalize
    u = x * s + m                         # STEGO UnNormalize
    b = np.clip(np.trunc(u * np.float32(255.0)), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(b.transpose(1, 2, 0)[:, :, ::-1])


def u8_to_float(img_u8_hwc: np.ndarray) -> np.ndarray:
    """(H,W,3) uint8 RGB -> (3,H,W) float32 byte / 255 (torchvision ToTensor)."""
    return (img_u8_hwc.astype(np.float32) / np.float32(255.0)).transpose(2, 0, 1)


def spatial_features(h: int, w: int) -> np.ndarray:
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    return np.stack([xs.ravel() / np.float32(POS_XY_STD), ys.ravel() / np.float32(POS_XY_STD)], 1)


def bilateral_features(bgr: np.ndarray) -> np.ndarray:
    h, w, _ = bgr.shape
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    c = bgr.reshape(-1, 3).astype(np.float32) / np.float32(BI_RGB_STD)
    return np.concatenate([np.stack([xs.ravel(), ys.ravel()], 1) / np.float32(BI_XY_STD), c], 1)


def scale_factors(d: int) -> np.ndarray:
    inv_std = float(np.float32(np.sqrt(2.0 / 3.0) * (d + 1)))
    return np.array([1.0 / np.sqrt(float((i + 2) * (i + 1))) * inv_std for i in range(d)], np.float64).astype(np.float32)


def pack_keys(keys: np.ndarray, d: int, frame: int = 0) -> np.ndarray:
    """keys (n, d) int -> packed uint64 in the layout above."""
    bits = KEY_BITS[d]
    out = np.full(keys.shape[0], np.uint64(frame) << np.uint64(bits * d), np.uint64)
    for i in range(d):
        out |= (keys[:, i].astype(np.int64) + (1 << (bits - 1))).astype(np.uint64) << np.uint64(bits * i)
    return out


def unpack_keys(packed: np.ndarray, d: int) -> np.ndarray:
    bits = KEY_BITS[d]
    mask = np.uint64((1 << bits) - 1)
    return np.stack([((packed >> np.uint64(bits * i)) & mask).astype(np.int64) - (1 << (bits - 1)) for i in range(d)], 1)


class Lattice:
    """Permutohedral lattice of features (N, d) float32.  Attributes: ``keys`` (M, d) int64 and ``packed`` (M,) uint64
    in vertex order, ``counts`` (M,) pixel-vertex incidences per vertex, ``offsets`` (N, d+1) vertex of each pixel's
    r-th vertex, ``bary`` (N, d+1) float32 weights, ``nbr`` (d+1, M, 2) blur neighbours (-1: none)."""

    def __init__(self, feat: np.ndarray):
        feat = np.asarray(feat, np.float32)
        N, d = feat.shape
        self.d, self.N = d, N
        sf = scale_factors(d)
        cf = feat * sf[None, :]
        E = np.zeros((N, d + 1), np.float32)
        sm = np.zeros(N, np.float32)
        for j in range(d, 0, -1):
            E[:, j] = sm - np.float32(j) * cf[:, j - 1]
            sm = sm + cf[:, j - 1]
        E[:, 0] = sm
        down, up = np.float32(1.0) / np.float32(d + 1), np.float32(d + 1)
        v = E * down
        hi, lo = np.ceil(v) * up, np.floor(v) * up
        rem0 = np.where(hi - E < E - lo, hi, lo).astype(np.int64)
        total = rem0.sum(1) // (d + 1)
        diff = E - rem0.astype(np.float32)
        rank = np.zeros((N, d + 1), np.int64)
        for i in range(d):
            for j in range(i + 1, d + 1):
                lt = diff[:, i] < diff[:, j]
                rank[:, i] += lt
                rank[:, j] += ~lt
        rank += total[:, None]
        neg, big = rank < 0, rank > d
        rank = np.where(neg, rank + d + 1, np.where(big, rank - d - 1, rank))
        rem0 = np.where(neg, rem0 + d + 1, np.where(big, rem0 - d - 1, rem0))
        bary = np.zeros((N, d + 2), np.float32)
        rows = np.arange(N)
        for i in range(d + 1):
            vi = (E[:, i] - rem0[:, i].astype(np.float32)) * down
            bary[rows, d - rank[:, i]] += vi
            bary[rows, d - rank[:, i] + 1] -= vi
        bary[:, 0] = (bary[:, 0].astype(np.float64) + (1.0 + bary[:, d + 1].astype(np.float64))).astype(np.float32)
        self.bary = bary[:, : d + 1]
        r = np.arange(d + 1)
        canon = np.where(rank[:, None, :d] <= d - r[None, :, None], r[None, :, None], r[None, :, None] - (d + 1))
        ekeys = (rem0[:, None, :d] + canon).reshape(-1, d)                  # (N*(d+1), d): entry p*(d+1)+r
        packed = pack_keys(ekeys, d)
        self.packed, inv, self.counts = np.unique(packed, return_inverse=True, return_counts=True)
        self.offsets = inv.reshape(N, d + 1)
        self.keys = unpack_keys(self.packed, d)
        self.M = self.packed.shape[0]
        self.rem0, self.rank, self.elevated = rem0, rank, E
        nbr = np.empty((d + 1, self.M, 2), np.int64)
        for j in range(d + 1):
            n1, n2 = self.keys - 1, self.keys + 1
            if j < d:
                n1[:, j] = self.keys[:, j] + d
                n2[:, j] = self.keys[:, j] - d
            for s, nk in enumerate((n1, n2)):
                pk = pack_keys(nk, d)
                idx = np.minimum(np.searchsorted(self.packed, pk), self.M - 1)
                nbr[j, :, s] = np.where(self.packed[idx] == pk, idx, -1)
        self.nbr = nbr

    def splat_matrix(self):
        import scipy.sparse as sp
        rows = self.offsets.ravel()
        cols = np.repeat(np.arange(self.N), self.d + 1)
        return sp.csr_matrix((self.bary.ravel().astype(np.float64), (rows, cols)), shape=(self.M, self.N))

    def filter(self, values: np.ndarray, blur=(0.5, 1.0, 0.5)) -> np.ndarray:
        """values (N, V) -> the lattice Gaussian (splat, blur, slice) of every column, in float64."""
        Sm = self.splat_matrix()
        v = np.asarray(Sm @ np.asarray(values, np.float64).reshape(self.N, -1))
        for j in range(self.d + 1):
            pad = np.vstack([np.zeros((1, v.shape[1])), v])
            v = blur[1] * v + blur[0] * pad[self.nbr[j, :, 0] + 1] + blur[2] * pad[self.nbr[j, :, 1] + 1]
        alpha = 1.0 / (1.0 + 2.0 ** (-self.d))
        return alpha * np.asarray(Sm.T @ v)


def softmax(x: np.ndarray, axis: int = -1) -> np.ndarray:
    e = np.exp(x - x.max(axis, keepdims=True))
    return e / e.sum(axis, keepdims=True)


def unary_from_logits(logits: np.ndarray, clip: float = CLIP) -> np.ndarray:
    """logits (N, K) -> U (N, K) float32."""
    p = softmax(np.asarray(logits, np.float32).astype(np.float64)).astype(np.float32)
    return (-np.log(np.clip(p, np.float32(clip), np.float32(1.0)))).astype(np.float32)


def mean_field(U: np.ndarray, bgr: np.ndarray, iters: int = MAX_ITER, bilateral: bool = True, blur=(0.5, 1.0, 0.5)):
    """U (N, K), bgr (H, W, 3) uint8 -> Q (N, K) float64 after ``iters`` mean-field updates."""
    h, w, _ = bgr.shape
    kernels = [(Lattice(spatial_features(h, w)), POS_W)]
    if bilateral:
        kernels.append((Lattice(bilateral_features(bgr)), BI_W))
    norms = [1.0 / np.sqrt(lat.filter(np.ones((h * w, 1)), blur)[:, 0] + 1e-20) for lat, _ in kernels]
    U = np.asarray(U, np.float64)
    Q = softmax(-U)
    for _ in range(iters):
        t = -U
        for (lat, wk), n in zip(kernels, norms):
            t = t + wk * n[:, None] * lat.filter(n[:, None] * Q, blur)
        Q = softmax(t)
    return Q


def dense_crf(logits: np.ndarray, bgr: np.ndarray, iters: int = MAX_ITER) -> np.ndarray:
    """STEGO's ``dense_crf``: logits (K, H, W) at image size, bgr (H, W, 3) uint8 -> Q (K, H, W)."""
    K, h, w = logits.shape
    U = unary_from_logits(logits.reshape(K, -1).T)
    return mean_field(U, bgr, iters).T.reshape(K, h, w)


def head_logits(head, batch: int, npad: int, grid: int, size: int, col0: int, classes: int, code_col: int = 0,
                code_dim: int = 0, alpha: float = 2.0):
    """The CRF's input logits from the STEGO head output [batch*npad, ld] (torch, patch p at row 1 + p of each frame):
    (batch, classes, size, size) float32.  code_dim = 0: the linear probe's columns; otherwise the cluster probe,
    ``alpha * <normalize(code_px), normalize(c_k)>`` with the code upsampled before it is normalised."""
    import torch
    import torch.nn.functional as F

    rows = head.view(batch, npad, -1)[:, 1 : 1 + grid * grid].float()

    def up(c0, n):
        g = rows[:, :, c0 : c0 + n].transpose(1, 2).reshape(batch, n, grid, grid)
        return F.interpolate(g, (size, size), mode="bilinear", align_corners=False)

    z = up(col0, classes)
    if code_dim:
        nrm = up(code_col, code_dim).norm(dim=1, keepdim=True).clamp_min(1e-12)
        z = alpha * z / nrm
    return z
