"""STEGO's dense CRF on the GPU (csrc/dense_crf.cu) against its definition, oracle/dense_crf.py: the lattice exactly,
one filter pass against float64, ten mean-field iterations, determinism, negative controls and StegoInterface /
FeatureExtractor with ``run_crf=True``."""
import numpy as np
import pytest
import torch

from oracle import dense_crf as dc
from oracle.slic import synthetic_image

pytestmark = pytest.mark.gpu

# |Q_gpu - Q_oracle| after 10 iterations: fp32 lattice sums and __expf against float64 (measured on an H100: at most
# 2.7e-5 at every geometry below)
Q_TOL = 2e-4
HEAD_COLS, CODE, CLUSTER, LINEAR = 256, 0, 128, 192


def _image(B, S, u8, seed=0):
    imgs = np.stack([synthetic_image(S, S, seed + b) for b in range(B)])
    if u8:
        t = torch.from_numpy((imgs.transpose(0, 2, 3, 1) * 255).astype(np.uint8))
        ref = [dc.u8_to_float(t[b].numpy()) for b in range(B)]
    else:
        t = torch.from_numpy(imgs)
        ref = list(imgs)
    return t.cuda(), [dc.crf_image_bytes(r) for r in ref]


def _head(B, S, K, seed=0, linear_std=1.5):
    g = S // 8
    npad = (1 + g * g + 7) // 8 * 8
    gen = torch.Generator().manual_seed(seed)
    head = torch.zeros(B * npad, HEAD_COLS)
    rows = head.view(B, npad, HEAD_COLS)[:, 1 : 1 + g * g]
    rows[..., CODE : CODE + 90] = torch.randn(B, g * g, 90, generator=gen)
    rows[..., CLUSTER : CLUSTER + K] = 4.0 * torch.randn(B, g * g, K, generator=gen)
    rows[..., LINEAR : LINEAR + K] = linear_std * torch.randn(B, g * g, K, generator=gen)
    return head.cuda(), npad, g


def _oracle_q(head, B, npad, g, S, K, bgrs, cluster, clip=dc.CLIP, **kw):
    z = dc.head_logits(head.cpu(), B, npad, g, S, CLUSTER if cluster else LINEAR, K, CODE, 90 if cluster else 0)
    return np.stack([dc.mean_field(dc.unary_from_logits(z[b].reshape(K, -1).T.numpy(), clip), bgrs[b], **kw)
                     for b in range(B)])


def _agreement(q, ref):
    """Label agreement over pixels whose oracle top-2 gap exceeds the Q tolerance, and max |dQ|."""
    s = np.sort(ref, -1)
    clear = (s[..., -1] - s[..., -2]) > Q_TOL
    agree = (q.argmax(-1) == ref.argmax(-1))[clear].mean()
    return agree, np.abs(q - ref).max()


@pytest.mark.parametrize("S,u8", [(64, False), (64, True), (224, False)])
def test_lattice_matches_oracle(S, u8):
    from wild_visual_navigation_b200 import ops

    img, bgrs = _image(1, S, u8)
    crf = ops.DenseCrf(S, 32, chunk=1)
    crf.build(img)
    for which, feat in ((0, dc.spatial_features(S, S)), (1, dc.bilateral_features(bgrs[0]))):
        lat = dc.Lattice(feat)
        got = crf.lattice(which)
        keys = got["keys"].cpu().numpy().view(np.uint64)
        assert keys.shape[0] == lat.M
        assert np.array_equal(keys, lat.packed)
        assert np.array_equal(got["counts"].cpu().numpy(), lat.counts)
        assert np.array_equal(got["offsets"].cpu().numpy(), lat.offsets)
        assert np.array_equal(got["bary"].cpu().numpy(), lat.bary)


def test_filter_matches_float64():
    """One unnormalised filter pass against float64 on the same lattice.  Every weight and input is non-negative, so
    each output is a sum of positive terms: at most ``c`` pixel terms in a splat run, 3 operations per blur pass and
    d+1 slice terms, each rounding once.  |error| <= (c + 3 (d+1) + (d+1) + 2) u * filter(x), u = 2^-24."""
    from wild_visual_navigation_b200 import ops

    S = 64
    img, bgrs = _image(1, S, False, seed=3)
    crf = ops.DenseCrf(S, 32, chunk=1)
    crf.build(img)
    x = torch.rand(S * S, 27, generator=torch.Generator().manual_seed(1))
    for which, feat in ((0, dc.spatial_features(S, S)), (1, dc.bilateral_features(bgrs[0]))):
        lat = dc.Lattice(feat)
        ref = lat.filter(x.numpy().astype(np.float64))
        got = crf.filter(which, x.cuda()).cpu().numpy().astype(np.float64)
        bound = (lat.counts.max() + 4 * (lat.d + 1) + 2) * 2.0**-24 * ref
        assert np.all(np.abs(got - ref) <= bound), np.max(np.abs(got - ref) / ref)


@pytest.mark.parametrize("B,S,K,u8", [(1, 64, 27, False), (3, 64, 32, True), (3, 64, 27, False), (1, 224, 32, False),
                                      (1, 224, 27, True)])
def test_mean_field_matches_oracle(B, S, K, u8):
    from wild_visual_navigation_b200 import ops

    img, bgrs = _image(B, S, u8, seed=B)
    head, npad, g = _head(B, S, K, seed=K)
    crf = ops.DenseCrf(S, K, chunk=2)
    for cluster in (True, False):
        lab, q = crf.run(img, head, npad, g, CLUSTER if cluster else LINEAR, K, CODE, 90 if cluster else 0,
                         2.0 if cluster else 1.0, want_q=True)
        q = q.cpu().numpy().reshape(B, S * S, K)
        ref = _oracle_q(head, B, npad, g, S, K, bgrs, cluster)
        agree, dq = _agreement(q, ref)
        print(f"B={B} S={S} K={K} u8={u8} cluster={cluster}: max |dQ| {dq:.2e}, clear-label agreement {agree:.5f}")
        assert dq <= Q_TOL and agree >= 0.999
        assert torch.equal(lab.view(B, -1).cpu(), torch.from_numpy(q.argmax(-1)))


def test_runs_are_bit_identical_and_negative_controls_fail():
    from wild_visual_navigation_b200 import ops

    B, S, K = 2, 64, 27
    img, bgrs = _image(B, S, False, seed=7)
    # logits wide enough that many probabilities fall below the 1e-5 clip
    head, npad, g = _head(B, S, K, seed=5, linear_std=6.0)
    crf = ops.DenseCrf(S, K, chunk=1)
    l1, q1 = crf.run(img, head, npad, g, LINEAR, K, want_q=True)
    l2, q2 = crf.run(img, head, npad, g, LINEAR, K, want_q=True)
    assert torch.equal(l1, l2) and torch.equal(q1, q2)
    q = q1.cpu().numpy().astype(np.float64)
    good = _oracle_q(head, B, npad, g, S, K, bgrs, False)
    assert np.abs(q - good).max() <= Q_TOL
    # the clip bounds the unary at -log(1e-5) = 11.5: without it the smallest Q fall by many orders of magnitude, which
    # the log of Q shows and its absolute value does not
    logq = np.log(np.maximum(q, 1e-38))
    assert np.abs(logq - np.log(np.maximum(good, 1e-38))).max() <= 0.1
    bad = _oracle_q(head, B, npad, g, S, K, bgrs, False, clip=1e-30)
    assert np.abs(logq - np.log(np.maximum(bad, 1e-38))).max() > 1.0
    for kw in (dict(bilateral=False), dict(blur=(0.25, 1.0, 0.25))):
        bad = _oracle_q(head, B, npad, g, S, K, bgrs, False, **kw)
        assert np.abs(q - bad).max() > Q_TOL, kw


def test_stego_interface_run_crf_and_graph_capture():
    from oracle.dino_vit import ViTConfig, synthetic_state_dict
    from oracle.stego_head import synthetic_head
    from wild_visual_navigation_b200.feature_extractor import FeatureExtractor, StegoInterface

    S = 224
    cfg = ViTConfig.from_name("vit_small", 8, S)
    sd, hd = synthetic_state_dict(cfg, seed=6), synthetic_head(384, 90, 32, 27, seed=3)
    with pytest.raises(ValueError, match="run_clustering"):
        StegoInterface("cuda", input_size=S, run_crf=True, run_clustering=True, head_state_dict=hd, backbone_state_dict=sd)
    st = StegoInterface("cuda", input_size=S, run_crf=True, head_state_dict=hd, backbone_state_dict=sd, max_batch=2)
    img = torch.from_numpy(np.stack([synthetic_image(S, S, s) for s in (1, 2)])).cuda()
    lin, clu = st.inference(img)
    B, npad, g = 2, st._geom[2], st._geom[3]
    bgrs = [dc.crf_image_bytes(i) for i in img.cpu().numpy()]
    for pred, cluster, K in ((clu, True, 32), (lin, False, 27)):
        ref = _oracle_q(st._head_out, B, npad, g, S, K, bgrs, cluster)
        s = np.sort(ref, -1)
        clear = (s[..., -1] - s[..., -2]) > Q_TOL
        agree = (pred[0].view(B, -1).cpu().numpy() == ref.argmax(-1))[clear].mean()
        assert pred.shape == (1, B, S, S) and pred.dtype == torch.int32 and agree >= 0.999, agree

    fe = FeatureExtractor("cuda", segmentation_type="stego", feature_type="stego", input_size=S, state_dict=sd,
                          head_state_dict=hd, flip_tta=False, max_batch=2, run_crf=True, run_clustering=False)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            ref = fe.extract_batch(img)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fe.extract_batch(img)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out["seg"], ref["seg"])
