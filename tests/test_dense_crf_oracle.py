"""oracle/dense_crf.py, the definition of STEGO's dense CRF: lattice invariants, the lattice filter against the exact
Gaussian, the byte-image round trip, mean field on a two-region image and the golden."""
import os

import numpy as np
import torch

from oracle import dense_crf as dc
from oracle.slic import synthetic_image

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dense_crf.pt")


def _features(h=20, w=24, seed=0):
    return [dc.spatial_features(h, w), dc.bilateral_features(dc.crf_image_bytes(synthetic_image(h, w, seed)))]


def test_splat_weights_sum_to_one_and_constants_filter_to_themselves_times_k1():
    for feat in _features():
        lat = dc.Lattice(feat)
        assert np.all(lat.bary >= -1e-6)
        assert np.abs(lat.bary.astype(np.float64).sum(1) - 1).max() <= 4e-7
        assert lat.counts.sum() == feat.shape[0] * (lat.d + 1)
        ones = lat.filter(np.ones((feat.shape[0], 1)))[:, 0]
        c = np.full((feat.shape[0], 3), 2.5)
        assert np.allclose(lat.filter(c), 2.5 * ones[:, None], rtol=1e-12)


def test_spatial_filter_tracks_the_exact_gaussian():
    """On a 16 x 16 pixel grid the spatial lattice filter (unit spacing, sxy = 1) stays within a factor of two below
    the exact Gaussian sum exp(-|f_i - f_j|^2 / 2) @ x and never above it, for non-negative x.  The bilateral lattice is
    far coarser relative to isolated colour features and is held to the GPU kernels, not to the exact Gaussian."""
    rng = np.random.default_rng(0)
    feat = dc.spatial_features(16, 16)
    lat = dc.Lattice(feat)
    x = rng.random((feat.shape[0], 2))
    f = feat.astype(np.float64)
    G = np.exp(-((f[:, None] - f[None]) ** 2).sum(-1) / 2)
    ratio = lat.filter(x) / (G @ x)
    assert ratio.min() >= 0.5 and ratio.max() <= 1.0, (ratio.min(), ratio.max())


def test_byte_image_round_trip():
    """Every byte survives normalise -> unnormalise -> x255 -> truncate except where float32 rounding lands just below
    the integer; those pixels end exactly one lower."""
    v = np.arange(256, dtype=np.float32) / np.float32(255)
    img = np.broadcast_to(v, (3, 1, 256)).copy()
    b = dc.crf_image_bytes(img)[0, :, ::-1].T.astype(np.int64)    # (3, 256) RGB
    d = np.arange(256)[None] - b
    assert set(np.unique(d)) <= {0, 1} and (d == 0).mean() > 0.5
    u8 = np.broadcast_to(np.arange(256, dtype=np.uint8)[:, None], (256, 3))[None]      # (1, 256, 3) camera bytes
    assert np.array_equal(dc.crf_image_bytes(dc.u8_to_float(u8)), dc.crf_image_bytes(img))


def test_mean_field_moves_labels_to_the_region_boundary():
    """Two flat colour regions split at column 20; the unaries favour the correct side only weakly and with noise, so
    the per-pixel argmax is often wrong.  The CRF's labels follow the colour edge."""
    h, w = 24, 40
    img = np.zeros((3, h, w), np.float32)
    img[:, :, :20] = np.array([0.8, 0.2, 0.1], np.float32)[:, None, None]
    img[:, :, 20:] = np.array([0.1, 0.3, 0.9], np.float32)[:, None, None]
    truth = (np.arange(w)[None, :] >= 20).repeat(h, 0)
    rng = np.random.default_rng(3)
    logits = np.stack([np.where(truth, -0.4, 0.4), np.where(truth, 0.4, -0.4)]) + rng.normal(0, 1.0, (2, h, w))
    plain = logits.argmax(0)
    q = dc.dense_crf(logits.astype(np.float32), dc.crf_image_bytes(img))
    assert (plain == truth).mean() < 0.8
    assert (q.argmax(0) == truth).mean() > 0.99


def test_golden():
    g = torch.load(GOLDEN)
    bgr = dc.crf_image_bytes(g["img"].numpy())
    assert np.array_equal(bgr, g["bgr"].numpy())
    for name, feat in (("spatial", dc.spatial_features(24, 20)), ("bilateral", dc.bilateral_features(bgr))):
        lat = dc.Lattice(feat)
        assert np.array_equal(lat.packed.view(np.int64), g[name + "_keys"].numpy())
        assert np.array_equal(lat.counts, g[name + "_counts"].numpy())
    assert np.allclose(dc.dense_crf(g["logits"].numpy(), bgr), g["q"].numpy(), rtol=0, atol=1e-12)
