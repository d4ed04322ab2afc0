"""DINOv2 with register tokens (ViT-S/14-reg, ViT-B/14-reg) on the sm_90a path, against the fp32 oracle and float64
kernel references.  Token rows of a frame: [CLS, reg_0 .. reg_{R-1}, patch_0 ..], so patch p sits in row 1 + R + p.

  tokens                    rel-L2 <= 2e-2 and mean cosine >= 0.999 vs oracle/dinov2_reg_vit.py (as for DINOv2),
                            at R = 4 and at R = 2 (read from the checkpoint's shape)
  interpolation             a handle interpolates its 37 x 37 embeddings exactly as F.interpolate(size=, antialias)
  uint8 camera ingest       bit-identical to the float path; flip TTA bit-identical to the flipped image
  patch-embed epilogue      element by element at registers 1 / 4, K = 588, P = 256 / 1024; CLS, register and padding
                            rows keep their NaN sentinel; registers = 0 is bit-identical to a struct without the field set
  attention                 every row at n_valid / npad 261 / 384, 1029 / 1152 and 1374 / 1408
  per-pixel trav / conf     the backbone's own bf16 tokens == the fp32 tokens' path bit for bit; <= 2e-2 vs the oracle
  FeatureExtractor          every segmentation type with feature_type="dinov2_reg" vs the oracle chain
  creation                  registers with a STEGO head is WVN_STATUS_INVALID; a missing register_tokens is reported
"""
import os
import sys
from ctypes import byref, c_void_p

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_dinov2_gpu import _gemm_k, _k_operands  # noqa: E402
from test_kernel_edges_gpu import (EPI_PATCH, assert_owned_and_untouched, assert_within, attn_bound,  # noqa: E402
                                   attn_inputs, attn_ref, check_gemm, gemm_ref, sentinel)

pytestmark = pytest.mark.gpu

WVN_STATUS_INVALID, WVN_STATUS_STATE = -1, -4


def rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


@pytest.fixture(scope="module", autouse=True)
def _fp32_reference_math():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


def _to(sd, dev):
    return {k: v.to(dev) for k, v in sd.items()}


def _reg(backbone_type, image_size, seed=1):
    from oracle.dinov2_reg_vit import synthetic_dinov2_reg_state_dict
    from oracle.dinov2_vit import dinov2_config

    cfg = dinov2_config(backbone_type, image_size)
    attn_std = 0.09 if backbone_type == "vit_small" else 0.09 / 2 ** 0.5
    return cfg, synthetic_dinov2_reg_state_dict(cfg, seed=seed, attn_std=attn_std)


def _di(sd, image_size, backbone_type="vit_small", **kw):
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    return DinoInterface("cuda", backbone="dinov2_reg", input_size=image_size, backbone_type=backbone_type,
                         patch_size=8, state_dict=sd, **kw)


# ------------------------------------------------------------------------------------------------ tokens
@pytest.mark.parametrize("backbone_type,image_size,B,chunk", [("vit_small", 224, 1, 0), ("vit_small", 448, 1, 0),
                                                              ("vit_small", 518, 1, 0), ("vit_small", 448, 8, 4),
                                                              ("vit_base", 448, 1, 0)])
def test_dinov2_reg_tokens_vs_oracle(backbone_type, image_size, B, chunk):
    from oracle.dinov2_reg_vit import dinov2_reg_tokens
    from oracle.wvn_path import wvn_transform

    cfg, sd = _reg(backbone_type, image_size, seed=image_size + B)
    di = _di(sd, image_size, backbone_type, max_batch=B, chunk=chunk)
    g = image_size // 14
    assert di.vit_patch_size == 8 and di.backbone == "dinov2_reg" and di.grid == g and di.feature_dim == cfg.dim
    assert di._model.registers == 4 and di._model.npad == (1 + 4 + g * g + 127) // 128 * 128
    img = torch.rand(B, 3, image_size, image_size, generator=torch.Generator().manual_seed(B)).cuda()
    got = di.inference_tokens(img)
    ref = dinov2_reg_tokens(wvn_transform(img, image_size), _to(sd, "cuda"), cfg)
    torch.cuda.synchronize()
    assert got.shape == ref.shape == (B, g * g, cfg.dim)
    cos = torch.nn.functional.cosine_similarity(got, ref, dim=-1)
    print(f"dinov2_reg {backbone_type}@{image_size} B={B}: rel_l2 {rel_l2(got, ref):.3e} cos min/mean "
          f"{cos.min().item():.5f}/{cos.mean().item():.6f}")
    assert rel_l2(got, ref) <= 2e-2 and cos.mean() >= 0.999


def test_register_count_read_from_the_checkpoint():
    """R = 2 (not the released 4): the handle takes R from the shape of ``register_tokens`` and the tokens follow the
    oracle; npad at 224 stays 384 (256 + 1 + 2 = 259 tokens)."""
    from oracle.dinov2_reg_vit import dinov2_reg_tokens, synthetic_dinov2_reg_state_dict
    from oracle.dinov2_vit import dinov2_config
    from oracle.wvn_path import wvn_transform

    cfg = dinov2_config("vit_small", 224)
    sd = synthetic_dinov2_reg_state_dict(cfg, seed=21, registers=2)
    di = _di(sd, 224, max_batch=2)
    assert di._model.registers == 2 and di._model.npad == 384
    img = torch.rand(2, 3, 224, 224, generator=torch.Generator().manual_seed(22)).cuda()
    got = di.inference_tokens(img)
    ref = dinov2_reg_tokens(wvn_transform(img, 224), _to(sd, "cuda"), cfg)
    torch.cuda.synchronize()
    cos = torch.nn.functional.cosine_similarity(got, ref, dim=-1)
    print(f"dinov2_reg R=2 @224: rel_l2 {rel_l2(got, ref):.3e} cos mean {cos.mean().item():.6f}")
    assert rel_l2(got, ref) <= 2e-2 and cos.mean() >= 0.999


@pytest.mark.parametrize("image_size", [448, 224])
def test_backbone_uses_the_register_interpolation(image_size):
    """A register handle built from the 37 x 37 pre-training embeddings gives, bit for bit, the tokens of one built
    from embeddings already interpolated by F.interpolate(size=(g, g), bicubic, antialias=True) (which the handle then
    takes as they are).  Built from DINO's +0.1 scale-factor interpolation instead, the tokens differ."""
    import torch.nn.functional as F

    from wild_visual_navigation_b200.ops import interpolate_pos_embed

    _, sd = _reg("vit_small", image_size, seed=31)
    g = image_size // 14
    pe = sd["pos_embed"]
    patch = F.interpolate(pe[:, 1:].reshape(1, 37, 37, 384).permute(0, 3, 1, 2), size=(g, g), mode="bicubic",
                          align_corners=False, antialias=True)
    pe_aa = torch.cat((pe[:, :1], patch.permute(0, 2, 3, 1).reshape(1, g * g, 384)), dim=1)
    img = torch.rand(1, 3, image_size, image_size, generator=torch.Generator().manual_seed(32)).cuda()
    tok = _di(sd, image_size, max_batch=1).inference_tokens(img).clone()
    tok_aa = _di(dict(sd, pos_embed=pe_aa), image_size, max_batch=1).inference_tokens(img).clone()
    tok_v1 = _di(dict(sd, pos_embed=interpolate_pos_embed(pe, g)), image_size, max_batch=1).inference_tokens(img)
    torch.cuda.synchronize()
    assert torch.equal(tok, tok_aa)
    assert not torch.equal(tok, tok_v1)


def test_dinov2_reg_uint8_ingest_and_flip_tta_bit_identical():
    from oracle.wvn_path import ros_image_to_float

    _, sd = _reg("vit_small", 448, seed=3)
    di = _di(sd, 448, max_batch=4, chunk=2)
    u8 = torch.randint(0, 256, (2, 480, 640, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(6)).cuda()
    tok_u8 = di.inference_tokens(u8).clone()
    tok_f = di.inference_tokens(ros_image_to_float(u8))
    assert tok_u8.shape == (2, 1024, 384)
    assert torch.equal(tok_u8, tok_f)
    img = torch.rand(2, 3, 448, 448, generator=torch.Generator().manual_seed(7)).cuda()
    both = di._model.forward(img, flip_tta=True).clone()
    assert torch.equal(both[2:], di._model.forward(img.flip(dims=[3])))
    assert torch.equal(both[:2], di._model.forward(img))


# ------------------------------------------------------------------------------------------------ patch-embed epilogue
@pytest.mark.parametrize("P", [1024, 256])
@pytest.mark.parametrize("registers", [1, 4])
def test_patch_embed_epilogue_with_registers(registers, P):
    """K = 588 at pitch 592; patch p of frame f lands in row f * npad + 1 + R + p with pos[1 + p]; the CLS, register and
    padding rows keep their NaN sentinel bit for bit."""
    dev = "cuda"
    K, D, frames = 588, 384, 3
    npad = (P + 1 + registers + 127) // 128 * 128
    a, w, bias = _k_operands(frames * P, D, K, seed=P + registers)
    pos = torch.randn(1 + P, D, generator=torch.Generator(device=dev).manual_seed(P + 1), device=dev)
    init = sentinel((frames * npad, D), torch.float32, dev)
    out = init.clone()
    _gemm_k(a, w, K, epi=EPI_PATCH, bias=bias, out=out, pos=pos, tokens_in=P, npad=npad, registers=registers)
    torch.cuda.synchronize()
    ref, S = gemm_ref(a[:, :K], w[:, :K], bias)
    pe = pos[1:].double().repeat(frames, 1)
    ref, S = ref + pe, S + pe.abs()
    rows = (torch.arange(frames, device=dev)[:, None] * npad + 1 + registers
            + torch.arange(P, device=dev)[None, :]).reshape(-1)
    owned = torch.zeros(frames * npad, D, dtype=torch.bool, device=dev)
    owned[rows] = True
    assert_owned_and_untouched(out, init, owned, f"patch{P}_reg{registers}")
    check_gemm(out[rows], ref, S, K, f"patch_reg{registers}", bf16_out=False)


def test_patch_embed_registers_zero_is_the_unset_struct():
    dev = "cuda"
    K, D, P, frames = 588, 384, 256, 2
    npad = 384
    a, w, bias = _k_operands(frames * P, D, K, seed=9)
    pos = torch.randn(1 + P, D, generator=torch.Generator(device=dev).manual_seed(10), device=dev)
    out0 = sentinel((frames * npad, D), torch.float32, dev)
    out1 = out0.clone()
    _gemm_k(a, w, K, epi=EPI_PATCH, bias=bias, out=out0, pos=pos, tokens_in=P, npad=npad)
    _gemm_k(a, w, K, epi=EPI_PATCH, bias=bias, out=out1, pos=pos, tokens_in=P, npad=npad, registers=0)
    torch.cuda.synchronize()
    assert torch.equal(out0.view(torch.int32), out1.view(torch.int32))


# ------------------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("H", [6, 12])
@pytest.mark.parametrize("n_valid,npad", [(261, 384), (1029, 1152), (1374, 1408)])
def test_attention_register_token_counts(n_valid, npad, H):
    """Every query row against float64 at the register models' token counts of 224, 448 and 518 (g^2 + 1 + 4); the
    dominant rows put their softmax mass in the masked last tile and must fail the bound without it."""
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
    assert_within(got, ref, bound, "attention_dinov2_reg")
    dropped, _, _ = attn_ref(q, k, v, n_valid, 0.125, keys_end=t0)
    rows_fail = ((dropped[:, sel] - ref[:, sel]).abs() > bound[:, sel]).any(dim=-1)
    assert bool(rows_fail.all())


# ------------------------------------------------------------------------------------------------ per-pixel maps
@pytest.mark.parametrize("image_size,out_size", [(448, 448), (224, 256)])
def test_pixel_inference_from_register_backbone(image_size, out_size):
    """The fused per-pixel head reads the backbone's bf16 tokens from row 1 + R (grid 32, and grid 16 upsampled to 256):
    it equals the head on the fp32 tokens bit for bit (both hand the same bf16 values to the same kernels) and the
    oracle's pixel_inference within 2e-2.  The same tokens shifted by R rows (what a head reading from row 1 would see)
    miss the oracle by far."""
    from oracle.wvn_path import pixel_inference
    from wild_visual_navigation_b200 import ConfidenceGenerator, SimpleMLP, TraversabilityInference

    _, sd = _reg("vit_small", image_size, seed=5)
    di = _di(sd, image_size, max_batch=2)
    g = di.grid
    img = torch.rand(2, 3, image_size, image_size, generator=torch.Generator().manual_seed(0)).cuda()
    tokens = di.inference_tokens(img)
    torch.manual_seed(42)
    model = SimpleMLP(384, [256, 32, 1], True).cuda()
    cg = ConfidenceGenerator(0.5, "latest_measurement").cuda()
    with torch.no_grad():
        cg.mean[0], cg.std[0] = 0.3, 0.1
    mlp = TraversabilityInference(di, model, cg)._mlp
    head = (cg.mean.data, cg.std.data, 0.5)
    trav, conf = mlp.pixels_from_vit(di._model, 2, (out_size, out_size), *head)       # the handle's bf16 tokens
    trav_f, conf_f = mlp.pixels(tokens, (g, g), (out_size, out_size), *head)           # the fp32 tokens, re-cast
    trav_s, conf_s = mlp.pixels(torch.roll(tokens, shifts=4, dims=1), (g, g), (out_size, out_size), *head)
    torch.cuda.synchronize()
    assert torch.equal(trav, trav_f) and torch.equal(conf, conf_f)
    msd = {k: v.detach() for k, v in model.state_dict().items()}
    for b in range(2):
        dense = torch.nn.functional.interpolate(tokens[b:b + 1].reshape(1, g, g, 384).permute(0, 3, 1, 2),
                                                (out_size, out_size), mode="bilinear", align_corners=True)
        t_ref, c_ref = pixel_inference(dense, msd, cg.mean.data, cg.std.data, 0.5)
        dt, dc = (trav[b] - t_ref).abs().max().item(), (conf[b] - c_ref).abs().max().item()
        st, sc = (trav_s[b] - t_ref).abs().max().item(), (conf_s[b] - c_ref).abs().max().item()
        print(f"grid {g} -> {out_size} frame {b}: trav / conf max abs diff {dt:.2e} / {dc:.2e}; shifted by R "
              f"{st:.2e} / {sc:.2e}")
        assert dt <= 2e-2 and dc <= 2e-2
        assert max(st, sc) > 5 * 2e-2


# ------------------------------------------------------------------------------------------------ FeatureExtractor
@pytest.mark.parametrize("seg_type", ["slic", "grid", "random", "none", "stego"])
def test_feature_extractor_dinov2_reg_features_vs_oracle(seg_type):
    """Every segmentation type with register-model features at 224 (grid 16).  With stego segmentation STEGO segments
    on its own DINO v1 handle and the features come from a second, register handle."""
    from oracle import stego_head, wvn_path
    from oracle.dino_vit import ViTConfig, synthetic_state_dict, vit_feature_map
    from oracle.dinov2_reg_vit import dinov2_reg_inference
    from wild_visual_navigation_b200.feature_extractor import FeatureExtractor

    cfg, sd = _reg("vit_small", 224, seed=11)
    kw = {}
    if seg_type == "stego":
        cfg1 = ViTConfig.from_name("vit_small", 8, 224)
        sd1 = synthetic_state_dict(cfg1, seed=6)
        hd = stego_head.synthetic_head(384, 90, 32, 27, seed=3)
        kw = dict(stego_state_dict=sd1, head_state_dict=hd, flip_tta=False, run_clustering=False)
    fe = FeatureExtractor("cuda", segmentation_type=seg_type, feature_type="dinov2_reg", input_size=224,
                          state_dict=sd, max_batch=1, **kw)
    assert fe.feature_dim == 384 and fe._dino.backbone == "dinov2_reg" and fe._dino.grid == 16
    img = torch.rand(1, 3, 224, 224, generator=torch.Generator().manual_seed(12)).cuda()
    edges, feat, seg, center, dense = fe.extract(img, return_dense_features=True)
    dense_ref = dinov2_reg_inference(img, _to(sd, "cuda"), cfg)
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
        assert fe._dino is not fe._stego._dino and fe._stego._dino._model.registers == 0
        sdc, hdc = _to(kw["stego_state_dict"], "cuda"), _to(kw["head_state_dict"], "cuda")
        f1 = vit_feature_map(wvn_path.wvn_transform(img, 224), sdc, cfg1)
        _, cluster, _ = stego_head.stego_inference(f1, None, hdc, (224, 224))
        agree = (seg == wvn_path.relabel(cluster[0].long())).float().mean().item()
        print(f"stego segments on DINO v1: agreement {agree:.4f}")
        assert agree >= 0.98
    assert (feat - wvn_path.sparsify_features(dense, seg)).abs().max() <= 2e-3 * feat.abs().max()
    assert rel_l2(feat, wvn_path.sparsify_features(dense_ref, seg)) <= 2e-2
    assert (center - wvn_path.centers(seg[None, None])).abs().max() < 1e-3
    assert torch.equal(edges.T.cpu(), wvn_path.adjacency_list(seg[None, None]).cpu())


def test_feature_extractor_dinov2_reg_seeded_default():
    from wild_visual_navigation_b200.feature_extractor import FeatureExtractor

    with pytest.warns(UserWarning, match="DINOV2_REG"):
        fe = FeatureExtractor("cuda", segmentation_type="grid", feature_type="dinov2_reg", input_size=224,
                              backbone_type="vit_base")
    assert fe.feature_dim == 768 and fe._dino._model.dim == 768 and fe._dino._model.registers == 4
    r = fe.extract_batch(torch.rand(1, 3, 224, 224, generator=torch.Generator().manual_seed(1)).cuda())
    assert r["tokens"].shape == (1, 256, 768)


# ------------------------------------------------------------------------------------------------ creation checks
def _cfg(registers, head_out):
    from wild_visual_navigation_b200._C import VitConfig

    return VitConfig(224, 14, 384, 12, 6, 1536, 1, 0, 1e-6, head_out, registers)


def test_registers_with_stego_head_is_invalid():
    from wild_visual_navigation_b200 import _C

    h = c_void_p()
    assert _C.lib().wvn_vit_create(byref(_cfg(4, 256)), byref(h)) == WVN_STATUS_INVALID
    assert _C.lib().wvn_vit_create(byref(_cfg(-1, 0)), byref(h)) == WVN_STATUS_INVALID
    assert _C.lib().wvn_vit_create(byref(_cfg(4, 0)), byref(h)) == 0
    _C.lib().wvn_vit_destroy(h)


def test_missing_register_tokens_is_reported(monkeypatch):
    from wild_visual_navigation_b200 import _C, ops

    _, sd = _reg("vit_small", 224, seed=2)
    orig = ops.ViTBackbone._set
    monkeypatch.setattr(ops.ViTBackbone, "_set", lambda self, n, t: None if n == "register_tokens" else orig(self, n, t))
    vit = ops.ViTBackbone(224, 14, 384, 12, 6, 1536, sd, max_batch=1)
    assert vit.registers == 4
    with pytest.raises(_C.WvnError, match="register_tokens"):
        vit.forward(torch.rand(1, 3, 224, 224, device="cuda"))
