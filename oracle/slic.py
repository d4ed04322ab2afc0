"""TEST INFRASTRUCTURE ONLY (see oracle/__init__.py) — numpy restatement of the SLIC superpixel segmentation behind
``FeatureExtractor(segmentation_type="slic")`` (feature_extractor.py:88-95 ``Slic(num_components=100, compactness=10)``,
:221-225 ``segment_slic``: ``slic.iterate(np.uint8(img * 255))``).

The routine itself lives in the un-vendored ``fast-slic`` C++ package (setup.py:29, unpinned, not installed here; its
source is not in the reference repository and it pins no numbers) -> [EXTERNAL-RECALLED]: restated as the published SLIC
algorithm (Achanta et al.) in the all-integer form fast-slic / gSLIC use — 8-bit sRGB -> CIELAB through lookup tables,
a regular grid of ``num_components`` centres, 10 rounds of {assign every pixel to the nearest of the 3x3 neighbouring
grid cells' centres under  d = |dLab|^2 * S^2 + |dxy|^2 * (compactness * Q)^2 ;  move every centre to the rounded
mean of its pixels}.  fast-slic's sub-sampled centre update and its connectivity enforcement are NOT restated.
Parity unpinned against fast-slic; what the tests hold is (1) this file == the CUDA kernel bit for bit (everything is
integer arithmetic, so there is no tolerance), (2) the SLIC contract: labels in [0, K), every pixel labelled, every
segment within 2 S of its centre, boundaries following colour edges.
"""
from __future__ import annotations

import numpy as np

Q_SHIFT = 6          # Lab is carried in 1/64 units: L in [0, 6400]
T_BITS = 12          # linear RGB and X/Xn, Y/Yn, Z/Zn are carried in 12 bits


def lab_tables():
    """(G [256] sRGB byte -> 12-bit linear, M [3,3] 12-bit fixed-point RGB->XYZ/white, F [4096] f(t) * 4096)."""
    v = np.arange(256, dtype=np.float64) / 255.0
    lin = np.where(v <= 0.04045, v / 12.92, ((v + 0.055) / 1.055) ** 2.4)
    G = np.rint(4095.0 * lin).astype(np.int32)
    M = np.array([[0.4124564, 0.3575761, 0.1804375], [0.2126729, 0.7151522, 0.0721750], [0.0193339, 0.1191920, 0.9503041]])
    Mi = np.rint(4096.0 * M / M.sum(1, keepdims=True)).astype(np.int32)
    t = np.arange(4096, dtype=np.float64) / 4095.0
    f = np.where(t > (6.0 / 29.0) ** 3, np.cbrt(t), t / (3.0 * (6.0 / 29.0) ** 2) + 4.0 / 29.0)
    F = np.rint(4096.0 * f).astype(np.int32)
    return G, Mi, F


def rgb8_to_lab(img_u8: np.ndarray) -> np.ndarray:
    """img_u8 (H,W,3) uint8 -> (H,W,3) int32 Lab in 1/64 units."""
    G, Mi, F = lab_tables()
    lin = G[img_u8.astype(np.int64)]                                     # (H,W,3)
    t = np.minimum(4095, (lin @ Mi.T.astype(np.int64) + 2048) >> T_BITS)  # (H,W,3): X/Xn, Y/Yn, Z/Zn
    fx, fy, fz = F[t[..., 0]], F[t[..., 1]], F[t[..., 2]]
    L = (116 * fy - 65536) >> Q_SHIFT
    a = (500 * (fx - fy)) >> Q_SHIFT
    b = (200 * (fy - fz)) >> Q_SHIFT
    return np.stack([L, a, b], -1).astype(np.int32)


def grid_geometry(H: int, W: int, num_components: int):
    """-> (S, nx, ny): grid interval and the number of grid cells per axis; K = nx * ny clusters."""
    S = max(1, int(np.rint(np.sqrt(H * W / float(num_components)))))
    return S, max(1, int(np.rint(W / S))), max(1, int(np.rint(H / S)))


def float_image_to_u8(img: np.ndarray) -> np.ndarray:
    """``np.uint8(img * 255)`` of the reference: float32 product, truncation. img (3,H,W) float32 in [0,1] -> (H,W,3)."""
    return (np.transpose(img, (1, 2, 0)).astype(np.float32) * np.float32(255.0)).astype(np.uint8)


def slic(img_u8: np.ndarray, num_components: int = 100, compactness: float = 10.0, iters: int = 10):
    """img_u8 (H,W,3) uint8 -> (labels (H,W) int64 in [0, K), centres (K,5) int64 = L,a,b,x,y)."""
    H, W, _ = img_u8.shape
    lab = rgb8_to_lab(img_u8).astype(np.int64)
    S, nx, ny = grid_geometry(H, W, num_components)
    K = nx * ny
    S2 = S * S
    M2 = int(np.rint((compactness * (1 << Q_SHIFT)) ** 2))
    gx0 = ((2 * np.arange(nx) + 1) * W) // (2 * nx)
    gy0 = ((2 * np.arange(ny) + 1) * H) // (2 * ny)
    cy, cx = np.meshgrid(gy0, gx0, indexing="ij")
    cent = np.concatenate([lab[cy.ravel(), cx.ravel()], cx.reshape(-1, 1), cy.reshape(-1, 1)], 1).astype(np.int64)  # (K,5)
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    pgx = np.minimum(nx - 1, (xs * nx) // W)
    pgy = np.minimum(ny - 1, (ys * ny) // H)
    labels = None
    for _ in range(iters):
        best = np.full((H, W), np.iinfo(np.int64).max, dtype=np.int64)
        labels = np.zeros((H, W), dtype=np.int64)
        for dy in (-1, 0, 1):          # candidate order = increasing cluster id, first minimum wins
            for dx in (-1, 0, 1):
                qx, qy = pgx + dx, pgy + dy
                ok = (qx >= 0) & (qx < nx) & (qy >= 0) & (qy < ny)
                k = np.where(ok, qy * nx + qx, 0)
                c = cent[k]                                               # (H,W,5)
                dc = ((lab - c[..., :3]) ** 2).sum(-1)
                ds = (xs - c[..., 3]) ** 2 + (ys - c[..., 4]) ** 2
                d = np.where(ok, dc * S2 + ds * M2, np.iinfo(np.int64).max)
                take = d < best
                best = np.where(take, d, best)
                labels = np.where(take, k, labels)
        flat = labels.ravel()
        cnt = np.bincount(flat, minlength=K).astype(np.int64)
        feats = np.concatenate([lab.reshape(-1, 3), xs.reshape(-1, 1), ys.reshape(-1, 1)], 1)
        sums = np.zeros((K, 5), dtype=np.int64)
        for j in range(5):
            np.add.at(sums[:, j], flat, feats[:, j])
        new = (2 * sums + cnt[:, None]) // np.maximum(2 * cnt[:, None], 1)   # round half up (floor division)
        cent = np.where(cnt[:, None] > 0, new, cent)
    return labels, cent


def compact_labels(labels: np.ndarray) -> np.ndarray:
    """Labels renumbered 0..S-1 in ascending order (clusters that lost all their pixels leave no gap)."""
    u, inv = np.unique(labels, return_inverse=True)
    return inv.reshape(labels.shape).astype(np.int64)


def synthetic_image(h: int, w: int, seed: int = 0) -> np.ndarray:
    """(3,h,w) float32 in [0,1]: smooth colour fields, a few hard-edged patches and mild noise."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.stack([(np.sin(xx / 37.0 + seed) + 1) / 2, (np.cos(yy / 53.0) + 1) / 2, ((xx + yy) % 97) / 97.0], 0)
    for _ in range(6):
        y0, x0 = rng.integers(0, h - 8), rng.integers(0, w - 8)
        hh, ww = rng.integers(8, max(9, h // 3)), rng.integers(8, max(9, w // 3))
        img[:, y0 : y0 + hh, x0 : x0 + ww] = rng.random(3)[:, None, None]
    return np.clip(img + rng.normal(0, 0.03, img.shape), 0, 1).astype(np.float32)
