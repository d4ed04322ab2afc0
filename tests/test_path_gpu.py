"""GPU parity tests of the assembled hot path against the oracle (CPU restatement of the
reference, oracle/) and against the golden fixtures produced by the reference's own code.

Stated tolerances (north star: "within a stated fp tolerance"; reference arithmetic is fp32,
the tensor-core path uses bf16 operands with fp32 accumulation):
  ViT patch tokens          rel-L2 <= 2e-2 and mean cosine >= 0.999 vs the fp32 oracle
  dense features            same (bilinear upsampling is fp32 on both sides)
  STEGO code                rel-L2 <= 3e-2; segment ids >= 98 % pixel agreement (ties flip)
  pooled segment features   1e-4 abs when fed identical tokens (pure fp32 reduction reorder)
  centers / adjacency       exact edge set and order; centers 1e-4 (known-answer asset fixture)
  trav / conf maps          abs <= 2e-2 when fed identical tokens
  train step (fp32 kernels) 2e-5 rel on losses / grads / updated params vs the reference-made golden
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


@pytest.fixture(scope="module", autouse=True)
def _fp32_reference_math():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


def _to(sd, dev):
    return {k: v.to(dev) for k, v in sd.items()}


@pytest.fixture(scope="module")
def vit448():
    from oracle.dino_vit import ViTConfig, synthetic_state_dict
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    cfg = ViTConfig.from_name("vit_small", 8, 448)
    sd = synthetic_state_dict(cfg, seed=1)
    di = DinoInterface("cuda", input_size=448, backbone_type="vit_small", patch_size=8, state_dict=sd, max_batch=4, chunk=2)
    return cfg, sd, di


def test_vit_tokens_parity_448(vit448):
    from oracle.dino_vit import vit_tokens
    from oracle.wvn_path import wvn_transform

    cfg, sd, di = vit448
    img = torch.rand(3, 3, 448, 448, generator=torch.Generator().manual_seed(0)).cuda()
    got = di.inference_tokens(img)
    ref = vit_tokens(wvn_transform(img, 448), _to(sd, "cuda"), cfg)
    torch.cuda.synchronize()
    assert got.shape == ref.shape == (3, 3136, 384)
    cos = torch.nn.functional.cosine_similarity(got, ref, dim=-1)
    print("vit448 rel_l2", rel_l2(got, ref), "cos min/mean", cos.min().item(), cos.mean().item())
    assert torch.isfinite(got).all()
    assert rel_l2(got, ref) <= 2e-2
    assert cos.mean() >= 0.999 and cos.min() >= 0.99
    # frames are independent: same frame alone gives the same tokens (chunking / batching invariance)
    alone = di.inference_tokens(img[2:3])
    assert torch.equal(alone[0], got[2])


def test_vit_base_tokens_parity_512():
    """BASELINE.json config 5's model family: DINO ViT-B/8 (D 768, 12 heads) on a 64x64 token grid (512 px; 518 floors
    to the same grid), single frame, against the fp32 oracle."""
    from oracle.dino_vit import ViTConfig, synthetic_state_dict, vit_tokens
    from oracle.wvn_path import wvn_transform
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    cfg = ViTConfig.from_name("vit_base", 8, 512)
    # qkv std scaled by 1/sqrt(2) against the ViT-S fixtures so that the attention logits keep a realistic spread
    # (std ~3, max ~20) at D = 768; at the default std they are ~6 / 40 — a near one-hot softmax in which the bf16
    # rounding of q.k alone moves the weights by > 10 %, which says nothing about the kernels
    sd = synthetic_state_dict(cfg, seed=2, attn_std=0.09 / 2 ** 0.5)
    di = DinoInterface("cuda", input_size=512, backbone_type="vit_base", patch_size=8, state_dict=sd, max_batch=2)
    img = torch.rand(2, 3, 512, 512, generator=torch.Generator().manual_seed(1)).cuda()
    got = di.inference_tokens(img)
    ref = vit_tokens(wvn_transform(img, 512), _to(sd, "cuda"), cfg)
    assert got.shape == ref.shape == (2, 4096, 768)
    cos = torch.nn.functional.cosine_similarity(got, ref, dim=-1)
    print("vit-b 512 rel_l2", rel_l2(got, ref), "cos min/mean", cos.min().item(), cos.mean().item())
    assert rel_l2(got, ref) <= 2e-2 and cos.mean() >= 0.999 and cos.min() >= 0.99


@pytest.mark.parametrize("attn_std", [0.09 / 2 ** 0.5, 0.09])
def test_vit_base_logit_spread_conditioning_and_debug_mode(attn_std, monkeypatch):
    """ViT-B/8 at a realistic attention-logit spread (qkv std 0.064: logits std ~3) and at the DEFAULT std of the
    fixtures (0.09 at D = 768: logits std ~6, max ~40 — near one-hot rows).  What tolerance really holds is a statement
    about the NETWORK's conditioning, measured here with the fp32 oracle itself: round only the weights to bf16, keep
    every operation in fp32, and look at how far the tokens move.  At the realistic spread that is ~1e-2 and the
    tensor-core path stays <= 2e-2; at the default std the exact-arithmetic oracle already moves by > 1e-1 under that
    2^-9 weight perturbation (each block's 0.2 % activation error becomes a ~0.1 logit error in the next block), so no
    bf16-operand implementation can hold 2e-2 there — the tensor-core path is required to stay within 2x that
    conditioning figure.  The parity-debug mode ($WVN_VIT_PRECISE=1: fp32 QKV projections + fp32 SIMT attention,
    SURVEY.md §7) removes the attention kernel's own roundings (q, k, v, P in bf16): its error must not exceed the
    tensor-core path's, which separates a kernel defect from conditioning."""
    from oracle.dino_vit import ViTConfig, synthetic_state_dict, vit_tokens
    from oracle.wvn_path import wvn_transform
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    cfg = ViTConfig.from_name("vit_base", 8, 256)   # 32 x 32 tokens keep the fp32 oracle quick; the effect is per logit
    sd = synthetic_state_dict(cfg, seed=2, attn_std=attn_std)
    img = torch.rand(1, 3, 256, 256, generator=torch.Generator().manual_seed(1)).cuda()
    timg = wvn_transform(img, 256)
    ref = vit_tokens(timg, _to(sd, "cuda"), cfg)
    sd_bf = {k: (v.bfloat16().float() if v.dim() >= 2 and "pos_embed" not in k and "cls" not in k else v) for k, v in sd.items()}
    cond = rel_l2(vit_tokens(timg, _to(sd_bf, "cuda"), cfg), ref)
    res = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("WVN_VIT_PRECISE", mode)
        di = DinoInterface("cuda", input_size=256, backbone_type="vit_base", patch_size=8, state_dict=sd, max_batch=1)
        got = di.inference_tokens(img)
        res[mode] = rel_l2(got, ref)
        del di
    print(f"vit-b attn_std={attn_std:.3f}: fp32 oracle with bf16-rounded weights moves by {cond:.3e}; tensor-core path rel_l2 "
          f"{res['0']:.3e}; precise-attention mode {res['1']:.3e}")
    assert res["0"] <= max(2e-2, 2.0 * cond)
    assert res["1"] <= res["0"] * 1.1 + 1e-3


def test_beats_eager_gpu_reference_path():
    """North star: "end-to-end frames/s at 1 GPU that beats the reference's own GPU PyTorch path on the same H100".
    The oracle IS that path (eager fp32 PyTorch in the reference's order of operations); it is timed here on the GPU
    for the backbone + per-pixel inference of 448x448 frames next to the product.  Prints both; asserts >= 5x."""
    import time

    from oracle import pipeline, wvn_path
    from oracle.dino_vit import ViTConfig, synthetic_state_dict
    from wild_visual_navigation_b200 import TraversabilityInference, get_model
    from wild_visual_navigation_b200.feature_extractor import DinoInterface
    from wild_visual_navigation_b200.utils import ConfidenceGenerator

    cfg = ViTConfig.from_name("vit_small", 8, 448)
    sd = synthetic_state_dict(cfg, seed=1)
    B = 8
    di = DinoInterface("cuda", input_size=448, backbone_type="vit_small", patch_size=8, state_dict=sd, max_batch=B)
    torch.manual_seed(42)
    model = get_model({"name": "SimpleMLP", "simple_mlp_cfg": {"input_size": 384, "hidden_sizes": [256, 32, 1],
                                                               "reconstruction": True}}).cuda()
    cg = ConfidenceGenerator(std_factor=0.5, method="latest_measurement").cuda()
    ti = TraversabilityInference(di, model, cg)
    img = torch.rand(B, 3, 448, 448, generator=torch.Generator().manual_seed(0)).cuda()
    sdc = _to(sd, "cuda")
    mlp_sd = {k: v.detach().clone() for k, v in model.state_dict().items()}

    def eager(frames):
        for b in range(frames):
            f = pipeline.frame_features(img[b : b + 1], sdc, cfg, None)
            wvn_path.pixel_inference(f["dense"], mlp_sd, cg.mean.data, cg.std.data, 0.5)

    def ours():
        ti.predict(img)

    def timed(fn, *a):
        fn(*a)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(*a)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    t_eager = timed(eager, 2) / 2
    t_ours = timed(ours) / B
    print(f"eager fp32 PyTorch on this GPU: {1 / t_eager:.1f} frames/s ({t_eager * 1e3:.1f} ms/frame);  "
          f"wvn-b200 (ViT + per-pixel MLP, B={B}): {1 / t_ours:.1f} frames/s;  speed-up {t_eager / t_ours:.1f}x")
    assert t_eager / t_ours >= 5.0


def test_dino_interface_dense_with_resize():
    """Non-square input that needs the NEAREST resize + center crop, vit_small/8 at 224."""
    from oracle.dino_vit import ViTConfig, synthetic_state_dict
    from oracle.wvn_path import dino_inference
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    cfg = ViTConfig.from_name("vit_small", 8, 224)
    sd = synthetic_state_dict(cfg, seed=4)
    di = DinoInterface("cuda", input_size=224, backbone_type="vit_small", patch_size=8, state_dict=sd, max_batch=2)
    img = torch.rand(2, 3, 270, 360, generator=torch.Generator().manual_seed(5)).cuda()
    got = di.inference(img)
    ref = dino_inference(img, _to(sd, "cuda"), cfg)
    assert got.shape == ref.shape == (2, 384, 270, 270)
    print("dense rel_l2", rel_l2(got, ref))
    assert rel_l2(got, ref) <= 2e-2


def test_uint8_hwc_ingest_matches_float_path_and_oracle():
    """SURVEY.md §8f rank 1: camera frames (B,H,W,3) uint8 straight into the patch loader == ros_image_to_torch
    (ToTensor / 255) + resize_image (NEAREST + center crop) + the float interface — bit-identical tokens — and
    within the ViT tolerance of the oracle run on the reference's own chain of steps."""
    from oracle.dino_vit import ViTConfig, synthetic_state_dict, vit_tokens
    from oracle.wvn_path import ros_image_to_float, resize_image, wvn_transform
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    cfg = ViTConfig.from_name("vit_small", 8, 224)
    sd = synthetic_state_dict(cfg, seed=4)
    di = DinoInterface("cuda", input_size=224, backbone_type="vit_small", patch_size=8, state_dict=sd, max_batch=3, chunk=2)
    u8 = torch.randint(0, 256, (3, 300, 404, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(6)).cuda()
    tok_u8 = di.inference_tokens(u8)
    img = ros_image_to_float(u8)                       # what the node hands to the feature extractor ...
    tok_f = di.inference_tokens(img)
    assert torch.equal(tok_u8, tok_f)
    small = resize_image(img, 224)                     # ... after ImageProjector.resize_image
    assert torch.equal(di.inference_tokens(small), tok_u8)
    ref = vit_tokens(wvn_transform(small, 224), _to(sd, "cuda"), cfg)
    assert rel_l2(tok_u8, ref) <= 2e-2


def test_golden_dino_wrapper_oracle_matches_reference(golden_dir):
    """The oracle's wrapper semantics == the reference's own DinoInterface.inference code (golden)."""
    from oracle.dino_vit import ViTConfig, synthetic_state_dict
    from oracle.wvn_path import dino_inference

    g = torch.load(os.path.join(golden_dir, "dino_wrapper.pt"))
    cfg = ViTConfig(**g["cfg"])
    sd = synthetic_state_dict(cfg, seed=g["vit_seed"], attn_std=g["attn_std"])
    assert (dino_inference(g["img"], sd, cfg) - g["out"]).abs().max() < 1e-5
    assert (dino_inference(g["img2"], sd, cfg) - g["out2"]).abs().max() < 1e-5


@pytest.mark.parametrize("flip_tta,hw", [(False, (224, 224)), (True, (224, 224)), (True, (270, 360))])
def test_stego_head_and_segments(flip_tta, hw):
    from oracle.dino_vit import ViTConfig, synthetic_state_dict, vit_feature_map
    from oracle.stego_head import stego_inference, synthetic_head
    from oracle.wvn_path import wvn_transform
    from wild_visual_navigation_b200.feature_extractor import StegoInterface

    cfg = ViTConfig.from_name("vit_small", 8, 224)
    sd = synthetic_state_dict(cfg, seed=6)
    hd = synthetic_head(384, 90, 32, 27, seed=3)
    si = StegoInterface("cuda", input_size=224, backbone_type="vit_small", patch_size=8, head_state_dict=hd,
                        backbone_state_dict=sd, flip_tta=flip_tta, max_batch=2)
    H, W = hw  # (270, 360): the transform resizes (NEAREST) + crops; outputs are (H, H) (stego_interface.py:104-109)
    img = torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(7)).cuda()
    lin, clu = si.inference(img)
    sdc, hdc = _to(sd, "cuda"), _to(hd, "cuda")
    timg = wvn_transform(img, 224)
    feats = vit_feature_map(timg, sdc, cfg)
    feats_f = vit_feature_map(timg.flip(dims=[3]), sdc, cfg) if flip_tta else None
    code_ref, clu_ref, lin_ref = stego_inference(feats, feats_f, hdc, (224, 224), out_h=H)
    assert clu.shape == (1, 2, H, H) and clu.dtype == torch.int32
    agree_c = (clu[0] == clu_ref).float().mean().item()
    agree_l = (lin[0] == lin_ref).float().mean().item()
    code = si.features
    print("stego code rel_l2", rel_l2(code, code_ref), "cluster agree", agree_c, "linear agree", agree_l)
    assert rel_l2(code, code_ref) <= 3e-2
    assert agree_c >= 0.98 and agree_l >= 0.98


def test_feature_extractor_extract_contract_vs_oracle(golden_dir):
    """``FeatureExtractor.extract`` (stego segmentation + stego features, the reference's supported pairing): the
    returned tuple has the contract the reference's own extract produces (extract_stego.pt: edges (2,E) int64, feat
    (S,90), seg (H,W), center (S,2), dense (1,90,H,H)) and its values match the oracle chain — which test_oracle.py
    holds to that same reference golden — at ViT-S/8 224."""
    from oracle import stego_head, wvn_path
    from oracle.dino_vit import ViTConfig, synthetic_state_dict, vit_feature_map
    from wild_visual_navigation_b200.feature_extractor import FeatureExtractor

    ref = torch.load(os.path.join(golden_dir, "extract_stego.pt"))
    cfg = ViTConfig.from_name("vit_small", 8, 224)
    sd = synthetic_state_dict(cfg, seed=6)
    hd = stego_head.synthetic_head(384, 90, 32, 27, seed=3)
    fe = FeatureExtractor("cuda", segmentation_type="stego", feature_type="stego", input_size=224, state_dict=sd,
                          head_state_dict=hd, flip_tta=True, run_clustering=False, max_batch=2)
    img = torch.rand(1, 3, 224, 224, generator=torch.Generator().manual_seed(8)).cuda()
    edges, feat, seg, center, dense = fe.extract(img, return_dense_features=True)
    assert fe.feature_dim == 90 and fe.feature_type == "stego" and fe.segmentation_type == "stego"
    S = int(seg.max()) + 1
    assert edges.dtype == ref["edges"].dtype and edges.shape[0] == 2 and feat.shape == (S, 90) and center.shape == (S, 2)
    assert seg.shape == (224, 224) and dense.shape == (1, 90, 224, 224)
    sdc, hdc = _to(sd, "cuda"), _to(hd, "cuda")
    t = wvn_path.wvn_transform(img, 224)
    f, ff = vit_feature_map(t, sdc, cfg), vit_feature_map(t.flip(dims=[3]), sdc, cfg)
    code_up, cluster, _ = stego_head.stego_inference(f, ff, hdc, (224, 224))
    seg_ref = wvn_path.relabel(cluster[0].long())
    agree = (seg == seg_ref).float().mean().item()
    print("extract: segment agreement", agree, "dense rel_l2", rel_l2(dense, code_up))
    assert agree >= 0.98 and rel_l2(dense, code_up) <= 3e-2
    # on OUR segmentation the pooled features / centers / edges must equal the reference's definitions exactly
    feat_ref = wvn_path.sparsify_features(dense, seg)
    assert (feat - feat_ref).abs().max() <= 2e-3 * feat_ref.abs().max()
    assert (center - wvn_path.centers(seg[None, None])).abs().max() < 1e-3
    assert torch.equal(edges, wvn_path.adjacency_list(seg[None, None]).T)


def test_stego_kmeans_kernel_vs_oracle_on_identical_code():
    """csrc/stego_kmeans.cu against oracle/stego_head.py:image_kmeans on the SAME fp32 code (only the summation order
    differs): centroids to 1e-3 relative, per-patch nearest-centroid scores to 1e-2 of their range, and the per-pixel
    labels of the upsampled code (wvn_logits_argmax on those scores vs kmeans_predict) on >= 99.5 % of the pixels."""
    from oracle import stego_head
    from wild_visual_navigation_b200 import ops
    from wild_visual_navigation_b200.feature_extractor.weights import HEAD_CLUSTER_COL, HEAD_CODE_COL

    g = torch.Generator(device="cuda").manual_seed(3)
    B, gr, npad, ld, K = 3, 28, 896, 256, 20
    P = gr * gr
    rows = torch.zeros(B * npad, ld, device="cuda")
    # a smooth field + noise, so that clusters are spatially coherent like a real code map
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, gr, device="cuda"), torch.linspace(-1, 1, gr, device="cuda"), indexing="ij")
    basis = torch.stack([yy, xx, yy * xx, yy**2, xx**2, torch.sin(3 * yy), torch.cos(3 * xx), torch.ones_like(yy)], -1)
    mix = torch.randn(B, 8, 90, device="cuda", generator=g)
    code = (basis.reshape(1, P, 8) @ mix) * 2.0 + 0.3 * torch.randn(B, P, 90, device="cuda", generator=g)
    rows.view(B, npad, ld)[:, 1 : 1 + P, HEAD_CODE_COL : HEAD_CODE_COL + 90] = code
    cent = torch.empty(B, K, 90, device="cuda")
    ops.stego_kmeans(rows, B, npad, P, HEAD_CODE_COL, 90, HEAD_CLUSTER_COL, K, 10, centroids_out=cent)
    code_map = code.transpose(1, 2).reshape(B, 90, gr, gr)
    cent_ref = stego_head.image_kmeans(code_map, K, 10)
    print("k-means centroids rel_l2", rel_l2(cent, cent_ref))
    assert rel_l2(cent, cent_ref) <= 1e-3
    score = rows.view(B, npad, ld)[:, 1 : 1 + P, HEAD_CLUSTER_COL : HEAD_CLUSTER_COL + K]
    score_ref = code @ cent_ref.transpose(1, 2) - 0.5 * (cent_ref**2).sum(-1)[:, None, :]
    assert (score - score_ref).abs().max() <= 1e-2 * (score_ref.max() - score_ref.min())
    seg = ops.logits_argmax(rows, HEAD_CLUSTER_COL, K, B, npad, gr, gr, 224, 224)
    seg_ref = stego_head.kmeans_predict(code_map, cent_ref, (224, 224))
    agree = (seg == seg_ref).float().mean().item()
    print("k-means per-pixel labels agreement", agree)
    assert agree >= 0.995


@pytest.mark.parametrize("flip_tta", [False, True])
def test_stego_per_image_kmeans_default(flip_tta):
    """run_clustering=True / n_image_clusters=20 — what WVN actually runs for stego segmentation
    (feature_extractor.py:47-53; the ROS node does not override it).  Lloyd iterations amplify input perturbations
    (a boundary patch that changes cluster moves two centroids, which move more patches ...), so the segments are held
    to the oracle's clustering of OUR code (bf16 tensor-core head, rel-L2 ~1e-2 from the fp32 code): >= 98 % of the
    pixels; against the oracle's clustering of ITS OWN fp32 code the agreement is only reported."""
    from oracle import stego_head, wvn_path
    from oracle.dino_vit import ViTConfig, synthetic_state_dict, vit_feature_map
    from wild_visual_navigation_b200.feature_extractor import FeatureExtractor

    cfg = ViTConfig.from_name("vit_small", 8, 224)
    sd = synthetic_state_dict(cfg, seed=6)
    hd = stego_head.synthetic_head(384, 90, 32, 27, seed=3)
    fe = FeatureExtractor("cuda", segmentation_type="stego", feature_type="stego", input_size=224, state_dict=sd,
                          head_state_dict=hd, flip_tta=flip_tta, max_batch=2)           # defaults: run_clustering=True, K=20
    assert fe._stego._cfg.run_clustering and fe.max_segments == 20
    img = torch.rand(2, 3, 224, 224, generator=torch.Generator().manual_seed(8)).cuda()
    r = fe.extract_batch(img)
    code_ours = r["tokens"].transpose(1, 2).reshape(2, 90, 28, 28)             # our (B, P, 90) code as a map
    cluster_same = stego_head.kmeans_predict(code_ours, stego_head.image_kmeans(code_ours, 20, 10), (224, 224))
    sdc, hdc = _to(sd, "cuda"), _to(hd, "cuda")
    t = wvn_path.wvn_transform(img, 224)
    f = vit_feature_map(t, sdc, cfg)
    ff = vit_feature_map(t.flip(dims=[3]), sdc, cfg) if flip_tta else None
    code_ref, cluster_own, _ = stego_head.stego_inference(f, ff, hdc, (224, 224), n_image_clusters=20, kmeans_iters=10)
    for b in range(2):
        agree = (r["seg"][b] == wvn_path.relabel(cluster_same[b])).float().mean().item()
        agree_own = (r["seg"][b] == wvn_path.relabel(cluster_own[b].long())).float().mean().item()
        print(f"k-means segments (flip_tta={flip_tta}) frame {b}: agreement {agree:.4f} on our code, {agree_own:.4f} vs the "
              f"oracle's own fp32 code; segments {int(r['n_segments'][b])}")
        assert agree >= 0.98
        assert 1 <= int(r["n_segments"][b]) <= 20


def test_segment_known_answer_asset(golden_dir):
    """Reference's shipped fixture: centers(seg.pt) == center.pt, adjacency == graph.pt edge_index."""
    from wild_visual_navigation_b200.feature_extractor import SegmentExtractor

    z = np.load(os.path.join(golden_dir, "segments.npz"))
    se = SegmentExtractor()
    for seg_key, edges_key, cen_key in (("asset_seg", "asset_ref_edges", "asset_centers"),
                                        ("syn_seg", "syn_edges", "syn_centers")):
        seg = torch.from_numpy(z[seg_key].astype(np.int64)).cuda()[None, None]
        edges = se.adjacency_list(seg).cpu().numpy()
        cen = se.centers(seg).cpu().numpy()
        assert np.array_equal(edges, z[edges_key]), (edges[:5], z[edges_key][:5])
        assert np.abs(cen - z[cen_key]).max() < 1e-4
    ei = z["asset_edge_index"]
    assert set(map(tuple, ei.T.tolist())) == set(map(tuple, se.adjacency_list(
        torch.from_numpy(z["asset_seg"].astype(np.int64)).cuda()[None, None]).cpu().tolist()))


def test_segment_pooling_vs_oracle(golden_dir):
    from oracle.wvn_path import sparsify_features
    from wild_visual_navigation_b200 import ops

    z = np.load(os.path.join(golden_dir, "segments.npz"))
    seg = torch.from_numpy(z["asset_seg"].astype(np.int64)).cuda()
    tok = torch.randn(1, 56 * 56, 384, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    r = ops.segment_reduce(seg[None], 100, tokens=tok, grid=(56, 56), want_centers=True, want_edges=True)
    dense = torch.nn.functional.interpolate(tok.reshape(1, 56, 56, 384).permute(0, 3, 1, 2), (448, 448),
                                            mode="bilinear", align_corners=True)
    ref = sparsify_features(dense, seg)
    assert (r["feat"][0] - ref).abs().max() < 1e-4
    # relabel (feature_extractor.py:245-246): drop a third of the labels, then compact to 0..S-1
    from oracle.wvn_path import relabel as relabel_ref
    s3 = seg.clone()
    s3[s3 % 3 == 0] += 1
    want = relabel_ref(s3)
    s3 = s3[None].contiguous()
    counts = ops.relabel(s3, 128)
    assert torch.equal(s3[0], want) and int(counts[0]) == int(want.max()) + 1


@pytest.mark.parametrize("mode", ["fused", "unfused"])
def test_pixel_inference_vs_oracle(vit448, mode, monkeypatch):
    """fused = algebraically restructured per-pixel head (pixel_head.cu); unfused = interp + 3 GEMMs."""
    from oracle.wvn_path import pixel_inference

    monkeypatch.setenv("WVN_PIXEL_HEAD", mode)
    from wild_visual_navigation_b200 import ConfidenceGenerator, SimpleMLP, TraversabilityInference

    cfg, sd, di = vit448
    torch.manual_seed(42)
    model = SimpleMLP(384, [256, 32, 1], True).cuda()
    # move the weights away from init so the outputs are not trivially ~0.5
    with torch.no_grad():
        model.flat_params.mul_(3.0)
    cg = ConfidenceGenerator(std_factor=0.5, method="latest_measurement").cuda()
    tok = torch.randn(2, 3136, 384, device="cuda", generator=torch.Generator(device="cuda").manual_seed(8))
    # centre the confidence interval on this input's reco-loss distribution so the map is not saturated
    from oracle.wvn_path import mlp_forward
    with torch.no_grad():
        xs = tok[0, ::7]
        lr = ((mlp_forward(xs, {k: v.detach() for k, v in model.state_dict().items()})[:, 1:] - xs) ** 2).mean(1)
        cg.mean[0], cg.std[0] = lr.mean() - 0.5 * lr.std(), lr.std()
    ti = TraversabilityInference(di, model, cg)
    trav, conf = ti.predict_from_tokens(tok, 448)
    msd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    for b in range(2):
        dense = torch.nn.functional.interpolate(tok[b : b + 1].reshape(1, 56, 56, 384).permute(0, 3, 1, 2), (448, 448),
                                                mode="bilinear", align_corners=True)
        t_ref, c_ref = pixel_inference(dense, msd, cg.mean.data, cg.std.data, 0.5)
        dt, dc = (trav[b] - t_ref).abs().max().item(), (conf[b] - c_ref).abs().max().item()
        print(f"pixel inference [{mode}] max abs diff trav/conf", dt, dc, "conf range", c_ref.min().item(), c_ref.max().item())
        assert dt <= 2e-2 and dc <= 3e-2
        assert 0.02 < c_ref.float().mean() < 0.98  # the test is not saturated


def test_relabel_and_pooling_vs_reference_golden(golden_dir):
    """CUDA relabel + segment pooling against the outputs of the reference's own segment_stego relabel loop and
    sparsify_features (sparsify.pt).  Pooling is fed tokens at full resolution (grid == image), so the fused
    weights-by-linearity path must reproduce the per-pixel means exactly (1e-5)."""
    from wild_visual_navigation_b200 import ops

    g = torch.load(os.path.join(golden_dir, "sparsify.pt"))
    raw = g["raw_clusters"][0].cuda().long().contiguous()         # (1, H, W) arbitrary cluster ids
    counts = ops.relabel(raw, 27)
    assert int(counts[0]) == 5 and torch.equal(raw.cpu(), g["relabelled"][0])
    dense = g["dense"].cuda()                                       # (1, D, H, W): use it as a token grid of the same size
    _, D, H, W = dense.shape
    tokens = dense[0].permute(1, 2, 0).reshape(1, H * W, D).contiguous()
    r = ops.segment_reduce(raw, 8, tokens=tokens, grid=(H, W), want_centers=False, want_edges=False)
    assert (r["feat"][0, :5].cpu() - g["feat"]).abs().max() < 1e-5


def test_supervision_label_pooling_vs_reference_golden(golden_dir):
    """SURVEY.md §8f rank 3: the pooled labels of the CUDA reduction == MissionNode.update_supervision_signal
    (the reference's own method, executed by make_golden.py), batched and with ids outside [0, smax) ignored."""
    from wild_visual_navigation_b200 import ops

    g = torch.load(os.path.join(golden_dir, "supervision.pt"))
    seg, mask = g["seg"].cuda(), g["mask"].cuda()
    S = int(seg.max()) + 1
    seg2 = seg.clone()
    seg2[:3] = -1                                   # frame 1: a few ignored pixels (random-pixel mode marks them -1)
    y, valid = ops.pool_supervision(torch.stack([seg, seg2]), torch.stack([mask, mask]), S + 3)
    assert (y[0, :S].cpu() - g["signal"]).abs().max() < 1e-6
    assert torch.equal(valid[0, :S].cpu(), g["valid"])
    assert (y[:, S:] == 0).all() and not valid[:, S:].any()
    from oracle.wvn_path import update_supervision_signal
    keep = seg2 >= 0
    m2 = mask.clone()
    m2[:, ~keep] = float("nan")
    ref2, v2 = update_supervision_signal(m2.cpu(), seg.cpu())
    assert (y[1, :S].cpu() - ref2).abs().max() < 1e-6 and torch.equal(valid[1, :S].cpu(), v2)
    # single-channel (H, W) mask form
    y1, _ = ops.pool_supervision(seg[None], mask[0][None], S)
    ref1, _ = update_supervision_signal(mask[:1].cpu(), seg.cpu())
    assert (y1[0].cpu() - ref1).abs().max() < 1e-6


def test_train_step_vs_reference_golden(golden_dir):
    """3 Adam steps on the reference-generated fixture (reference SimpleMLP + TraversabilityLoss + Adam)."""
    from wild_visual_navigation_b200 import ops

    g = torch.load(os.path.join(golden_dir, "mlp_train.pt"))
    D, (h1, h2, _) = g["dim"], g["hidden"]
    keys = ["layers.0.weight", "layers.0.bias", "layers.2.weight", "layers.2.bias", "layers.4.weight", "layers.4.bias"]
    flat = torch.cat([g["init_state_dict"][k].reshape(-1) for k in keys]).cuda()
    tr = ops.MlpTrainer(flat, D, h1, h2, max_rows=128)
    x, y, yv = g["x"].cuda(), g["y"].cuda(), g["y_valid"].cuda()
    for s, want in enumerate(g["steps"]):
        conf = tr.step(x, y, yv)
        m = tr.metrics.tolist()
        gflat = torch.cat([want["grads"][k].reshape(-1) for k in keys]).cuda()
        pflat = torch.cat([want["state_dict"][k].reshape(-1) for k in keys]).cuda()
        print(f"step {s}: loss {m[0]:.7f} vs {want['loss_total']:.7f}; grad rel {rel_l2(tr.grads[:-1], gflat):.2e}; "
              f"param rel {rel_l2(tr.params, pflat):.2e}")
        assert abs(m[0] - want["loss_total"]) <= 2e-5 * max(1, abs(want["loss_total"]))
        assert abs(m[1] - want["loss_trav"]) <= 2e-5 and abs(m[2] - want["loss_reco"]) <= 2e-5
        assert abs(m[3] - want["loss_trav_confidence"]) <= 2e-5
        assert abs(m[4] - want["cg_mean"].item()) <= 1e-5 and abs(m[5] - want["cg_std"].item()) <= 1e-5
        assert (conf.cpu() - want["confidence"]).abs().max() <= 1e-4
        assert rel_l2(tr.grads[:-1], gflat) <= 2e-5
        assert rel_l2(tr.params, pflat) <= 2e-5
    # forward with the trained weights == reference forward (in-place sigmoid on column 0)
    pred = ops.mlp_forward_f32(tr.params, g["xq"].cuda(), D, h1, h2)
    assert (pred.cpu() - g["pred"]).abs().max() <= 1e-5


def test_train_step_full_size_vs_oracle():
    from oracle.wvn_path import mlp_init, synthetic_supervision, train_step
    from wild_visual_navigation_b200 import TraversabilityEstimator
    from wild_visual_navigation_b200.traversability_estimator import MissionNode

    te = TraversabilityEstimator(device="cuda", min_samples_for_training=1)
    sd = mlp_init(384, (256, 32), seed=42)
    for k, v in te._model.state_dict().items():
        assert torch.equal(v.cpu(), sd[k]), k  # same seeded init as the reference
    g = torch.Generator().manual_seed(12)
    for i in range(8):
        x = torch.randn(100, 384, generator=g)
        y, yv = synthetic_supervision(100, seed=20 + i)
        te.add_mission_node(MissionNode(x.cuda(), y.cuda(), yv.cuda()))
    opt_state = None
    for step in range(3):
        import random
        st = random.getstate()
        graph = te.make_batch(8)
        random.setstate(st)
        graph = te.make_batch(8)  # deterministic replay of the same sample
        xs, ys, yvs = graph.x.cpu(), graph.y.cpu(), graph.y_valid.cpu()
        te.train_on_batch(graph)
        m = te._trainer.metrics.tolist()
        sd, opt_state, ref = train_step(sd, opt_state, xs, ys, yvs, lr=1e-3)
        got = torch.cat([v.reshape(-1) for v in te._model.state_dict().values()]).cpu()
        want = torch.cat([v.reshape(-1) for v in sd.values()])
        print(f"full-size step {step}: loss {m[0]:.7f} vs {ref['loss_total']:.7f}, param rel {rel_l2(got, want):.2e}")
        assert abs(m[0] - ref["loss_total"]) <= 3e-5 * max(1.0, abs(ref["loss_total"]))
        assert rel_l2(got, want) <= 3e-5
    out = te.train()
    assert set(out) == {"mission_graph_num_valid_node", "loss_total", "loss_trav", "loss_reco"}


def test_checkpoint_roundtrip(tmp_path):
    from wild_visual_navigation_b200 import TraversabilityEstimator
    from wild_visual_navigation_b200.traversability_estimator import MissionNode

    te = TraversabilityEstimator(device="cuda", min_samples_for_training=0)
    x = torch.randn(64, 384, device="cuda")
    yv = torch.rand(64, device="cuda") < 0.3
    y = torch.where(yv, torch.rand(64, device="cuda"), torch.zeros(64, device="cuda"))
    te.add_mission_node(MissionNode(x, y, yv))
    te.train()
    te.save_checkpoint(str(tmp_path), "ck.pt")
    ck = torch.load(os.path.join(tmp_path, "ck.pt"))
    assert set(ck) == {"step", "model_state_dict", "optimizer_state_dict", "traversability_loss_state_dict", "loss"}
    assert list(ck["model_state_dict"]) == ["layers.0.weight", "layers.0.bias", "layers.2.weight", "layers.2.bias",
                                            "layers.4.weight", "layers.4.bias"]
    assert "_confidence_generator.mean" in ck["traversability_loss_state_dict"]
    # a stock torch Adam accepts the optimizer state
    ref_model = torch.nn.Sequential(torch.nn.Linear(384, 256), torch.nn.ReLU(), torch.nn.Linear(256, 32),
                                    torch.nn.ReLU(), torch.nn.Linear(32, 385)).cuda()
    torch.optim.Adam(ref_model.parameters(), lr=1e-3).load_state_dict(ck["optimizer_state_dict"])
    te2 = TraversabilityEstimator(device="cuda", min_samples_for_training=0)
    te2.load_checkpoint(os.path.join(tmp_path, "ck.pt"))
    assert torch.equal(te2._model.flat_params, te._model.flat_params)
    assert te2.step == te.step
