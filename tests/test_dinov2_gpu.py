"""DINOv2 (ViT-S/14, ViT-B/14) on the sm_90a path, against the fp32 oracle and float64 kernel references.

  tokens                    rel-L2 <= 2e-2 and mean cosine >= 0.999 vs the fp32 oracle (as for DINO)
  uint8 camera ingest       bit-identical to the float path; flip TTA bit-identical to the flipped image
  GEMM K tail               element by element (tests/test_kernel_edges_gpu.py's bounds and sentinels) at K = 588
                            (3 * 14 * 14), 65 and 130, with NaN in the pad columns of both operands
  attention                 every row at n_valid 257 (224 / 14) and 1370 (518 / 14)
  FeatureExtractor          every segmentation type with DINOv2 features vs the oracle chain
  per-pixel trav / conf     <= 2e-2 abs vs oracle.wvn_path.pixel_inference on the same tokens, grid 32 and 16
"""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_edges_gpu import (ACT_GELU, ACT_NONE, EPI_BF16, EPI_F32, EPI_PATCH, EPI_RESID,  # noqa: E402
                                   assert_owned_and_untouched, assert_within, attn_bound, attn_inputs, attn_ref,
                                   check_gemm, gemm_ref, sentinel)

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


def _attn_std(backbone_type):
    # ViT-B at the DINO-like qkv scale (DESIGN.md §5): torch's default std makes random ViT-B ill-conditioned in bf16
    return 0.09 if backbone_type == "vit_small" else 0.09 / 2 ** 0.5


def _v2(backbone_type, image_size, seed=1):
    from oracle.dinov2_vit import dinov2_config, synthetic_dinov2_state_dict

    cfg = dinov2_config(backbone_type, image_size)
    return cfg, synthetic_dinov2_state_dict(cfg, seed=seed, attn_std=_attn_std(backbone_type))


# ------------------------------------------------------------------------------------------------ tokens
@pytest.mark.parametrize("backbone_type,image_size,B,chunk", [("vit_small", 448, 1, 0), ("vit_small", 448, 8, 4),
                                                              ("vit_small", 224, 2, 0), ("vit_small", 518, 1, 0),
                                                              ("vit_base", 448, 1, 0)])
def test_dinov2_tokens_vs_oracle(backbone_type, image_size, B, chunk):
    from oracle.dinov2_vit import dinov2_tokens
    from oracle.wvn_path import wvn_transform
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    cfg, sd = _v2(backbone_type, image_size, seed=image_size + B)
    # patch_size=8 as the ROS default passes it with dinov2: the backbone still runs at patch 14
    di = DinoInterface("cuda", backbone="dinov2", input_size=image_size, backbone_type=backbone_type, patch_size=8,
                       state_dict=sd, max_batch=B, chunk=chunk)
    assert di.vit_patch_size == 8 and di.backbone == "dinov2" and di.grid == image_size // 14
    assert di.feature_dim == cfg.dim
    img = torch.rand(B, 3, image_size, image_size, generator=torch.Generator().manual_seed(B)).cuda()
    got = di.inference_tokens(img)
    ref = dinov2_tokens(wvn_transform(img, image_size), _to(sd, "cuda"), cfg)
    torch.cuda.synchronize()
    assert got.shape == ref.shape == (B, cfg.grid ** 2, cfg.dim)
    cos = torch.nn.functional.cosine_similarity(got, ref, dim=-1)
    print(f"dinov2 {backbone_type}@{image_size} B={B}: rel_l2 {rel_l2(got, ref):.3e} cos min/mean "
          f"{cos.min().item():.5f}/{cos.mean().item():.6f}")
    assert rel_l2(got, ref) <= 2e-2 and cos.mean() >= 0.999


def test_dinov2_uint8_ingest_and_flip_tta_bit_identical():
    """A 480 x 640 uint8 camera frame gives the tokens of its float image bit for bit (the loader's fused /255, NEAREST
    resize and center crop at patch 14), and the flip pass of the test-time augmentation gives those of the flipped
    transformed image."""
    from oracle.wvn_path import ros_image_to_float
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    _, sd = _v2("vit_small", 448, seed=3)
    di = DinoInterface("cuda", backbone="dinov2", input_size=448, backbone_type="vit_small", state_dict=sd, max_batch=4,
                       chunk=2)
    u8 = torch.randint(0, 256, (2, 480, 640, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(6)).cuda()
    tok_u8 = di.inference_tokens(u8).clone()
    tok_f = di.inference_tokens(ros_image_to_float(u8))
    assert tok_u8.shape == (2, 1024, 384)
    assert torch.equal(tok_u8, tok_f)
    img = torch.rand(2, 3, 448, 448, generator=torch.Generator().manual_seed(7)).cuda()
    both = di._model.forward(img, flip_tta=True).clone()
    assert torch.equal(both[2:], di._model.forward(img.flip(dims=[3])))
    assert torch.equal(both[:2], di._model.forward(img))


def test_feature_extractor_dinov2_is_not_dino_v1():
    """FeatureExtractor(feature_type="dinov2") builds a DINOv2 backbone (grid 16 at 224, patch 14), not DINO v1."""
    from wild_visual_navigation_b200.feature_extractor import FeatureExtractor

    with pytest.warns(UserWarning, match="DINOV2"):
        fe = FeatureExtractor("cuda", segmentation_type="grid", feature_type="dinov2", input_size=224)
    assert fe._dino.backbone == "dinov2" and fe._dino.grid == 16 and fe.feature_dim == 384
    r = fe.extract_batch(torch.rand(1, 3, 224, 224, generator=torch.Generator().manual_seed(1)).cuda())
    assert r["tokens"].shape == (1, 256, 384)
    with pytest.warns(UserWarning, match="DINOV2"):
        fe_b = FeatureExtractor("cuda", segmentation_type="grid", feature_type="dinov2", input_size=224,
                                backbone_type="vit_base")
    assert fe_b.feature_dim == 768 and fe_b._dino._model.dim == 768


# ------------------------------------------------------------------------------------------------ GEMM K tail
def _gemm_k(a, w, K, *, epi, act=ACT_NONE, bias=None, out=None, block_n=0, **kw):
    """wvn_gemm_bf16_ex with an explicit K: a [M, lda >= K], w [N, round_up(K, 8)] (pad columns included)."""
    from ctypes import byref, c_void_p

    from wild_visual_navigation_b200 import _C

    p = lambda t: c_void_p(0 if t is None else t.data_ptr())  # noqa: E731
    args = _C.GemmExArgs()
    args.m, args.n, args.k = a.shape[0], w.shape[0], K
    args.epi, args.act, args.block_n = epi, act, block_n
    args.a, args.lda, args.w, args.bias = p(a), a.stride(0), p(w), p(bias)
    args.out, args.ldo = p(out), out.stride(0)
    if "pos" in kw:
        args.pos = p(kw.pop("pos"))
    for name, val in kw.items():
        setattr(args, name, val)
    _C.check(_C.lib().wvn_gemm_bf16_ex(byref(args), _C.stream()))


def _k_operands(M, N, K, seed, extra_a=0):
    """A [M, K] at pitch round_up(K, 8) + extra_a and W [N, K] at pitch round_up(K, 8), NaN in every pad column: a
    kernel that read past K would turn every output of the row / column into NaN."""
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(seed)
    kp = (K + 7) // 8 * 8
    a = torch.full((M, kp + extra_a), float("nan"), device=dev)
    a[:, :K] = torch.randn(M, K, generator=g, device=dev)
    w = torch.full((N, kp), float("nan"), device=dev)
    w[:, :K] = torch.randn(N, K, generator=g, device=dev) / math.sqrt(K)
    return a.bfloat16(), w.bfloat16(), torch.randn(N, generator=g, device=dev)


PLAIN_K = {"f32": (EPI_F32, ACT_NONE), "bf16": (EPI_BF16, ACT_NONE), "bf16_gelu": (EPI_BF16, ACT_GELU),
           "resid": (EPI_RESID, ACT_NONE)}


@pytest.mark.parametrize("K", [588, 65, 130])
@pytest.mark.parametrize("kind", list(PLAIN_K))
def test_gemm_k_tail_plain_epilogues(kind, K):
    epi, act = PLAIN_K[kind]
    dev = "cuda"
    M, N = 200, 384
    a, w, bias = _k_operands(M, N, K, seed=K + len(kind), extra_a=8)
    dtype = torch.bfloat16 if epi == EPI_BF16 else torch.float32
    rows = M + 64
    init = torch.randn(rows, N, device=dev) if epi == EPI_RESID else sentinel((rows, N), dtype, dev)
    out = init.clone()
    _gemm_k(a, w, K, epi=epi, act=act, bias=bias, out=out)
    torch.cuda.synchronize()
    ref, S = gemm_ref(a[:, :K], w[:, :K], bias)
    if act == ACT_GELU:
        ref = torch.nn.functional.gelu(ref)
    if epi == EPI_RESID:
        base = init[:M].double()
        ref, S = ref + base, S + base.abs()
    owned = torch.zeros(rows, N, dtype=torch.bool, device=dev)
    owned[:M] = True
    assert_owned_and_untouched(out, init, owned, f"k{K}_{kind}")
    check_gemm(out[:M], ref, S, K, f"ktail_{kind}", bf16_out=epi == EPI_BF16, gelu=act == ACT_GELU)


@pytest.mark.parametrize("P", [1024, 256])
def test_gemm_k_tail_patch_embed(P):
    """The DINOv2 patch-embed GEMM as the backbone runs it: K = 588 at pitch 592, scattered to token rows 1 + tok of
    npad-row frames (npad 1152 at grid 32, 384 at grid 16); CLS and padding rows keep their sentinel."""
    dev = "cuda"
    K, D, frames = 588, 384, 3
    npad = (P + 1 + 127) // 128 * 128
    a, w, bias = _k_operands(frames * P, D, K, seed=P)
    g = torch.Generator(device=dev).manual_seed(P + 1)
    pos = torch.randn(1 + P, D, generator=g, device=dev)
    init = sentinel((frames * npad, D), torch.float32, dev)
    out = init.clone()
    _gemm_k(a, w, K, epi=EPI_PATCH, bias=bias, out=out, pos=pos, tokens_in=P, npad=npad)
    torch.cuda.synchronize()
    ref, S = gemm_ref(a[:, :K], w[:, :K], bias)
    pe = pos[1:].double().repeat(frames, 1)
    ref, S = ref + pe, S + pe.abs()
    rows = (torch.arange(frames, device=dev)[:, None] * npad + 1 + torch.arange(P, device=dev)[None, :]).reshape(-1)
    owned = torch.zeros(frames * npad, D, dtype=torch.bool, device=dev)
    owned[rows] = True
    assert_owned_and_untouched(out, init, owned, f"patch{P}")
    check_gemm(out[rows], ref, S, K, "ktail_patch", bf16_out=False)


# ------------------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("H", [6, 12])
@pytest.mark.parametrize("n_valid,npad", [(257, 384), (1370, 1408)])
def test_attention_dinov2_token_counts(n_valid, npad, H):
    """Every query row against float64 at the DINOv2 token counts of 224 (16 x 16 + 1) and 518 (37 x 37 + 1); 257
    leaves a single valid key in the masked last tile.  Without that tile the dominant rows must fail the bound."""
    from wild_visual_navigation_b200 import ops

    dev = "cuda"
    B = max(1, 36 // H)
    q, k, v, sel, t0 = attn_inputs(B, H, n_valid, npad, n_valid + H, dev)
    vt = v.transpose(1, 2).contiguous()
    out = ops.attention(q.view(B, H, npad, 64), k.view(B, H, npad, 64), vt.view(B, H, 64, npad), n_valid, 0.125)
    torch.cuda.synchronize()
    got = out.view(B, npad, H, 64).permute(0, 2, 1, 3).reshape(B * H, npad, 64)
    ref, PV, vmax = attn_ref(q, k, v, n_valid, 0.125)
    bound = attn_bound(ref, PV, vmax)
    assert_within(got, ref, bound, "attention_dinov2")
    dropped, _, _ = attn_ref(q, k, v, n_valid, 0.125, keys_end=t0)
    rows_fail = ((dropped[:, sel] - ref[:, sel]).abs() > bound[:, sel]).any(dim=-1)
    assert bool(rows_fail.all())


# ------------------------------------------------------------------------------------------------ FeatureExtractor
@pytest.mark.parametrize("seg_type", ["slic", "grid", "random", "none", "stego"])
def test_feature_extractor_dinov2_features_vs_oracle(seg_type):
    """Every segmentation type with DINOv2 features at 224 (grid 16): dense features vs the oracle's DINOv2 chain;
    pooled features, centers and edges vs the reference's definitions on the returned segmentation.  With stego
    segmentation, STEGO segments with its own DINO v1 backbone while the features come from a second, DINOv2 handle:
    the segments must match the oracle's STEGO on DINO v1 and the features the oracle's DINOv2."""
    from oracle import stego_head, wvn_path
    from oracle.dino_vit import ViTConfig, synthetic_state_dict, vit_feature_map
    from oracle.dinov2_vit import dinov2_inference
    from wild_visual_navigation_b200.feature_extractor import FeatureExtractor

    cfg, sd = _v2("vit_small", 224, seed=11)
    kw = {}
    if seg_type == "stego":
        cfg1 = ViTConfig.from_name("vit_small", 8, 224)
        sd1 = synthetic_state_dict(cfg1, seed=6)
        hd = stego_head.synthetic_head(384, 90, 32, 27, seed=3)
        kw = dict(stego_state_dict=sd1, head_state_dict=hd, flip_tta=False, run_clustering=False)
    fe = FeatureExtractor("cuda", segmentation_type=seg_type, feature_type="dinov2", input_size=224, state_dict=sd,
                          max_batch=1, **kw)
    assert fe.feature_dim == 384 and fe._dino.backbone == "dinov2" and fe._dino.grid == 16
    img = torch.rand(1, 3, 224, 224, generator=torch.Generator().manual_seed(12)).cuda()
    edges, feat, seg, center, dense = fe.extract(img, return_dense_features=True)
    dense_ref = dinov2_inference(img, _to(sd, "cuda"), cfg)
    assert dense.shape == dense_ref.shape == (1, 384, 224, 224)
    print(f"{seg_type}: dense rel_l2 {rel_l2(dense, dense_ref):.3e}")
    assert rel_l2(dense, dense_ref) <= 2e-2
    if seg_type == "none":
        assert feat.shape == dense.shape and torch.equal(feat, dense)
        assert edges.shape[0] == 2 and center.shape == (224 * 224, 2)
        return
    if seg_type == "random":
        assert edges is None and center is None
        ys, xs = (seg >= 0).nonzero(as_tuple=True)
        ids = seg[ys, xs]
        want = torch.empty_like(feat)
        want[ids] = dense[0, :, ys, xs].T
        assert (feat - want).abs().max() <= 1e-4
        assert rel_l2(feat[ids], dense_ref[0, :, ys, xs].T) <= 2e-2
        return
    S = int(seg.max()) + 1
    assert feat.shape == (S, 384) and center.shape == (S, 2)
    if seg_type == "stego":
        assert fe._dino is not fe._stego._dino
        sdc, hdc = _to(kw["stego_state_dict"], "cuda"), _to(kw["head_state_dict"], "cuda")
        f1 = vit_feature_map(wvn_path.wvn_transform(img, 224), sdc, cfg1)
        _, cluster, _ = stego_head.stego_inference(f1, None, hdc, (224, 224))
        agree = (seg == wvn_path.relabel(cluster[0].long())).float().mean().item()
        print(f"stego segments on DINO v1: agreement {agree:.4f}")
        assert agree >= 0.98
    # on OUR segmentation: pooled features, centers and edges by the reference's definitions
    assert (feat - wvn_path.sparsify_features(dense, seg)).abs().max() <= 2e-3 * feat.abs().max()
    assert rel_l2(feat, wvn_path.sparsify_features(dense_ref, seg)) <= 2e-2
    assert (center - wvn_path.centers(seg[None, None])).abs().max() < 1e-3
    assert torch.equal(edges.T.cpu(), wvn_path.adjacency_list(seg[None, None]).cpu())


# ------------------------------------------------------------------------------------------------ per-pixel maps
@pytest.mark.parametrize("image_size", [448, 224])
def test_pixel_inference_from_dinov2_tokens(image_size):
    """The fused per-pixel head on DINOv2 tokens (grid 32: token window 7; grid 16) vs the oracle's
    pixel_inference on the same tokens, bilinearly upsampled."""
    from oracle.wvn_path import pixel_inference
    from wild_visual_navigation_b200 import ConfidenceGenerator, SimpleMLP, TraversabilityInference
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    _, sd = _v2("vit_small", image_size, seed=5)
    di = DinoInterface("cuda", backbone="dinov2", input_size=image_size, backbone_type="vit_small", state_dict=sd,
                       max_batch=2)
    g = di.grid
    img = torch.rand(2, 3, image_size, image_size, generator=torch.Generator().manual_seed(0)).cuda()
    tokens = di.inference_tokens(img)
    torch.manual_seed(42)
    model = SimpleMLP(384, [256, 32, 1], True).cuda()
    cg = ConfidenceGenerator(0.5, "latest_measurement").cuda()
    with torch.no_grad():
        cg.mean[0], cg.std[0] = 0.3, 0.1
    trav, conf = TraversabilityInference(di, model, cg).predict_from_tokens(tokens, image_size)
    msd = {k: v.detach() for k, v in model.state_dict().items()}
    for b in range(2):
        dense = torch.nn.functional.interpolate(tokens[b:b + 1].reshape(1, g, g, 384).permute(0, 3, 1, 2),
                                                (image_size, image_size), mode="bilinear", align_corners=True)
        t_ref, c_ref = pixel_inference(dense, msd, cg.mean.data, cg.std.data, 0.5)
        dt, dc = (trav[b] - t_ref).abs().max().item(), (conf[b] - c_ref).abs().max().item()
        print(f"{image_size} frame {b}: trav / conf max abs diff {dt:.2e} / {dc:.2e}")
        assert dt <= 2e-2 and dc <= 2e-2
