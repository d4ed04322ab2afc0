"""DINOv2 ViT-L/14 (``backbone_type="vit_large"``: D = 1024, 24 blocks, 16 heads) on the sm_90a path.

  LayerNorm             the D = 1024 instantiation element by element against float64 with test_vit_io_gpu.py's
                        derived bound: the bf16 block input (both row orders, bit-identical) and the final norm's fp32
                        output (CLS / register / padding rows dropped, reverse order)
  tokens                both variants at 224 and 448, B = 1 and 3, against the fp32 oracle and against a bf16-storage
                        emulation of the sm_90a path (below); bars in TOKEN_BAR
  uint8 camera ingest   bit-identical to the float path
  CUDA graph            a captured forward replays to the eager tokens bit for bit
  HotPathStep           every learner, per-pixel and segment-wise, on STEGO (``stego_backbone_type``), SLIC and grid
                        segmentation, against the same work composed by hand, eager and through capture / replay

The bf16-storage emulation runs the oracle's arithmetic in fp32 with the path's rounding points: the normalised image,
the GEMM weights (LayerScale folded first, in fp32, as the product does), each LayerNorm output that feeds a GEMM,
Q / K / V, the unnormalised softmax weights fed to P V, the attention output and the GELU output are rounded to bf16;
the residual stream, the statistics, the biases and the position embeddings stay fp32.
"""
import os
import sys
import warnings

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_segment_maps_gpu import LEARNERS, _check_against_composed, _check_replay, _img, _labels  # noqa: E402
from test_vit_io_gpu import (LN_CONSTANTS, LN_EPS, assert_bits_equal, assert_guards, assert_within,  # noqa: E402,F401
                             bf16_half_ulp, guarded, ln_reference, ln_rows, ops)

pytestmark = pytest.mark.gpu

D = 1024
ATTN_STD = 0.09 * (384 / D) ** 0.5   # keeps the attention logits' spread of the ViT-S/B tests
# rel-L2 bars of the tokens, set from the bf16 emulation's own distance from the fp32 oracle, measured at most 9.3e-3
# over these cases (DESIGN.md §3.13): that distance against the bf16-storage emulation, 1.5 times it against fp32
TOKEN_BAR = {"fp32": 1.4e-2, "bf16": 1e-2}


@pytest.fixture(scope="module", autouse=True)
def _fp32_reference_math():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


def rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def large_config(image_size):
    from oracle.dino_vit import ViTConfig
    from oracle.dinov2_vit import PATCH, PRETRAIN_GRID
    from wild_visual_navigation_b200.feature_extractor.weights import VIT_SHAPES

    s = VIT_SHAPES["vit_large"]
    return ViTConfig(image_size, PATCH, s["dim"], s["depth"], s["heads"], s["mlp_dim"], PRETRAIN_GRID)


@pytest.fixture(scope="module")
def large_sds():
    from oracle.dinov2_reg_vit import synthetic_dinov2_reg_state_dict

    return {"dinov2": synthetic_dinov2_reg_state_dict(large_config(448), seed=5, attn_std=ATTN_STD),
            "dinov2_reg": synthetic_dinov2_reg_state_dict(large_config(448), seed=6, attn_std=ATTN_STD)}


def _sd(large_sds, variant):
    sd = large_sds[variant]
    return sd if variant == "dinov2_reg" else {k: v for k, v in sd.items() if k != "register_tokens"}


def _di(sd, variant, image_size, **kw):
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    return DinoInterface("cuda", backbone=variant, input_size=image_size, backbone_type="vit_large", patch_size=8,
                         state_dict=sd, **kw)


# ------------------------------------------------------------------------------------------------ LayerNorm
def _ln_params(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return 1 + 0.5 * torch.randn(D, generator=g, device="cuda"), 0.5 * torch.randn(D, generator=g, device="cuda")


def test_layernorm_1024_bf16_per_element(ops):
    """9 frames of the 448 grid (npad 1152): 10368 rows, more than one grid-stride pass of 132 * 64 warps."""
    rows = 9 * 1152
    x = ln_rows(rows, D, seed=D, device="cuda")
    gamma, beta = _ln_params(2)
    outs = {}
    for rev in (0, 1):
        buf, out = guarded(rows * D, torch.bfloat16)
        ops.layernorm(x, gamma, beta, LN_EPS, out=out.view(rows, D), reverse=bool(rev))
        torch.cuda.synchronize()
        assert_guards(buf, f"layernorm D=1024 reverse={rev}")
        outs[rev] = out.view(rows, D).clone()
    assert_bits_equal(outs[1], outs[0], "layernorm D=1024: reverse=1 vs reverse=0")
    got = outs[0]
    ref, bound = ln_reference(x, gamma, beta, LN_EPS)
    assert_within(got, ref, bound + bf16_half_ulp(got), "layernorm bf16 D=1024")
    zero_rows = torch.arange(0, rows, 11, device="cuda")
    zero_rows = zero_rows[(zero_rows // 11) % len(LN_CONSTANTS) == LN_CONSTANTS.index(0.0)]
    assert_bits_equal(got[zero_rows], beta.bfloat16().expand(len(zero_rows), D), "zero rows D=1024")


@pytest.mark.parametrize("B,npad,n_valid,row0", [
    (9, 1152, 1025, 1),    # ViT-L/14 @ 448: CLS dropped
    (23, 384, 261, 5),     # ViT-L/14-reg @ 224: CLS and 4 registers dropped; 8832 rows
])
def test_layernorm_1024_fp32_final_norm(ops, B, npad, n_valid, row0):
    rows = B * npad
    x = ln_rows(rows, D, seed=D + row0, device="cuda")
    gamma, beta = _ln_params(4)
    keep = n_valid - row0
    bbuf, ob = guarded(rows * D, torch.bfloat16)
    fbuf, of = guarded(B * keep * D, torch.float32)
    ops.layernorm(x, gamma, beta, LN_EPS, out=ob.view(rows, D), out_f32=of.view(B * keep, D), npad=npad,
                  n_valid=n_valid, row0=row0, reverse=True)
    torch.cuda.synchronize()
    tag = f"layernorm D=1024 fp32 tokens row0={row0}"
    assert_guards(bbuf, tag)
    assert_guards(fbuf, tag)
    got_b, got_f = ob.view(B, npad, D), of.view(B, keep, D)
    ref, bound = ln_reference(x, gamma, beta, LN_EPS)
    ref, bound = ref.view(B, npad, D)[:, row0:n_valid], bound.view(B, npad, D)[:, row0:n_valid]
    assert_within(got_f, ref, bound, tag)
    assert_bits_equal(got_f.bfloat16(), got_b[:, row0:n_valid], tag + ": bf16(fp32 output) vs bf16 output")


# ------------------------------------------------------------------------------------------------ tokens
def _bf(t):
    return t.bfloat16().float()


@torch.no_grad()
def tokens_bf16_storage(img, sd, cfg):
    """The fp32 oracle with the sm_90a path's bf16 rounding points (module docstring); (B, P, D)."""
    from oracle.wvn_path import wvn_transform
    from wild_visual_navigation_b200.ops import (fold_layerscale, interpolate_pos_embed,
                                                 interpolate_pos_embed_antialias)

    sd = fold_layerscale(sd, cfg.depth)
    reg = sd.get("register_tokens")
    R = 0 if reg is None else reg.shape[1]
    x = F.conv2d(_bf(wvn_transform(img, cfg.image_size)), _bf(sd["patch_embed.proj.weight"]),
                 sd["patch_embed.proj.bias"], stride=cfg.patch_size)
    B, _, gh, gw = x.shape
    interp = interpolate_pos_embed_antialias if R else interpolate_pos_embed
    pos = interp(sd["pos_embed"].float().cpu(), gh).to(img.device)
    x = torch.cat((sd["cls_token"].expand(B, -1, -1), x.flatten(2).transpose(1, 2)), dim=1) + pos
    if R:
        x = torch.cat((x[:, :1], reg.expand(B, -1, -1), x[:, 1:]), dim=1)
    H, C = cfg.heads, cfg.dim
    ln = lambda t, p: F.layer_norm(t, (C,), sd[p + ".weight"], sd[p + ".bias"], cfg.ln_eps)  # noqa: E731
    for i in range(cfg.depth):
        b = f"blocks.{i}."
        qkv = _bf(F.linear(_bf(ln(x, b + "norm1")), _bf(sd[b + "attn.qkv.weight"]), sd[b + "attn.qkv.bias"]))
        q, k, v = qkv.reshape(B, -1, 3, H, 64).permute(2, 0, 3, 1, 4)
        s = (q @ k.transpose(-2, -1)) * 0.125
        e = torch.exp(s - s.amax(-1, keepdim=True))
        o = _bf((_bf(e) @ v) / e.sum(-1, keepdim=True)).transpose(1, 2).reshape(B, -1, C)
        x = x + F.linear(o, _bf(sd[b + "attn.proj.weight"]), sd[b + "attn.proj.bias"])
        h = _bf(F.gelu(F.linear(_bf(ln(x, b + "norm2")), _bf(sd[b + "mlp.fc1.weight"]), sd[b + "mlp.fc1.bias"])))
        x = x + F.linear(h, _bf(sd[b + "mlp.fc2.weight"]), sd[b + "mlp.fc2.bias"])
    return ln(x, "norm")[:, 1 + R:]


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("image_size", [224, 448])
@pytest.mark.parametrize("variant", ["dinov2", "dinov2_reg"])
def test_vit_large_tokens_vs_oracles(large_sds, variant, image_size, B):
    from oracle.dinov2_reg_vit import dinov2_reg_tokens
    from oracle.dinov2_vit import dinov2_tokens
    from oracle.wvn_path import wvn_transform

    sd = _sd(large_sds, variant)
    cfg = large_config(image_size)
    di = _di(sd, variant, image_size, max_batch=B)
    g, R = image_size // 14, 4 if variant == "dinov2_reg" else 0
    assert di.feature_dim == 1024 and di.grid == g and di._model.registers == R
    assert di._model.npad == (1 + R + g * g + 127) // 128 * 128
    img = torch.rand(B, 3, image_size, image_size, generator=torch.Generator().manual_seed(B + image_size)).cuda()
    got = di.inference_tokens(img).clone()
    sdc = {k: v.cuda() for k, v in sd.items()}
    oracle = dinov2_reg_tokens if R else dinov2_tokens
    ref = oracle(wvn_transform(img, image_size), sdc, cfg)
    emu = tokens_bf16_storage(img, sdc, cfg)
    torch.cuda.synchronize()
    assert got.shape == ref.shape == emu.shape == (B, g * g, D)
    d_fp32, d_bf16, d_emu = rel_l2(got, ref), rel_l2(got, emu), rel_l2(emu, ref)
    cos = F.cosine_similarity(got, ref, dim=-1).mean().item()
    print(f"vit_large {variant} @{image_size} B={B}: rel-L2 vs fp32 {d_fp32:.3e}, vs bf16 storage {d_bf16:.3e}; "
          f"bf16 emulation vs fp32 {d_emu:.3e}; mean cosine vs fp32 {cos:.6f}")
    assert d_fp32 <= TOKEN_BAR["fp32"] and d_bf16 <= TOKEN_BAR["bf16"] and cos >= 0.999


@pytest.mark.parametrize("variant", ["dinov2", "dinov2_reg"])
def test_vit_large_uint8_ingest_bit_identical(large_sds, variant):
    from oracle.wvn_path import ros_image_to_float

    di = _di(_sd(large_sds, variant), variant, 448, max_batch=2)
    u8 = torch.randint(0, 256, (2, 480, 640, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(6)).cuda()
    tok_u8 = di.inference_tokens(u8).clone()
    tok_f = di.inference_tokens(ros_image_to_float(u8))
    assert tok_u8.shape == (2, 1024, D)
    assert torch.equal(tok_u8, tok_f)


def test_vit_large_capture_replay_equals_eager(large_sds):
    """The forward allocates nothing and never synchronises with the host: it captures, and a replay on new frames
    gives the eager tokens bit for bit."""
    di = _di(_sd(large_sds, "dinov2_reg"), "dinov2_reg", 448, max_batch=3)
    img0, img1 = (torch.rand(3, 3, 448, 448, generator=torch.Generator().manual_seed(s)).cuda() for s in (1, 2))
    static = img0.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        di.inference_tokens(static)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = di._model.forward(static)
    static.copy_(img1)
    graph.replay()
    got = out.clone()
    want = di.inference_tokens(img1)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ HotPathStep
@pytest.fixture(scope="module")
def stego_head():
    import bench

    return bench.make_weights()[2]   # the ViT-S STEGO head (384-d)


def _hot_path(large_sds, stego_head, variant, model, anomaly, **kw):
    from wild_visual_navigation_b200 import HotPathStep

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return HotPathStep("cuda", _sd(large_sds, variant), stego_head, batch=3, input_size=224, chunk=32,
                           flip_tta=False, run_clustering=True, n_image_clusters=20, model=model,
                           anomaly_detection=anomaly, feature_type=variant, backbone_type="vit_large",
                           stego_backbone_type="vit_small", **kw)


def _check_per_pixel_against_composed(a, b, img, y, yv, exact):
    """Per-pixel maps: b runs the per-pixel head on a's tokens and trains on a's rows."""
    ra = a.step(img, y, yv)
    tb, cb = b.ti.predict_from_tokens(ra["tokens"], b.input_size)
    tb, cb = tb.clone(), (None if cb is None else cb.clone())
    crow = b.te.train_on_padded(ra["feat"], ra["n_segments"], y, yv)
    b.ti.refresh_weights()
    assert ra["trav"].shape == (3, 224, 224) and torch.isfinite(ra["trav"]).all()
    assert (ra["conf"] is None) == (cb is None)
    dt = (ra["trav"] - tb).abs().max().item()
    dc = 0.0 if cb is None else (ra["conf"] - cb).abs().max().item()
    print(f"per-pixel step vs composed: |d| trav {dt:.2e} conf {dc:.2e}")
    if exact:
        assert torch.equal(ra["trav"], tb) and torch.equal(ra["conf"], cb)
    assert dt <= 1e-3 and dc <= 1e-4
    n = int(ra["n_segments"].sum())
    if a.te._anomaly_detection:
        n = int(yv[:n].sum())
    assert torch.isfinite(ra["confidence_rows"][:n]).all()
    assert (ra["confidence_rows"][:n] - crow[:n]).abs().max().item() <= 1e-4


@pytest.mark.parametrize("model,anomaly", LEARNERS)
def test_segment_wise_step_on_stego(large_sds, stego_head, model, anomaly):
    a = _hot_path(large_sds, stego_head, "dinov2", model, anomaly, prediction_per_pixel=False)
    b = _hot_path(large_sds, stego_head, "dinov2", model, anomaly, prediction_per_pixel=False)
    assert a.fe.feature_dim == 1024 and a.fe._dino._model.dim == 1024
    assert a.fe._stego._dino._model.dim == 384 and a.fe._stego._dino is not a.fe._dino
    y, yv = _labels(a, 3)
    p0 = a.te._model.flat_params.clone()
    ra = _check_against_composed(a, b, _img(1), y, yv, exact=model in ("SimpleMLP", "DoubleMLP") and not anomaly)
    assert ra["feat"].shape[1:] == (a.smax, 1024)
    assert not torch.equal(a.te._model.flat_params, p0)


@pytest.mark.parametrize("model,anomaly", [m for m in LEARNERS if m[0] != "SimpleGCN"])
def test_per_pixel_step_on_stego(large_sds, stego_head, model, anomaly):
    a = _hot_path(large_sds, stego_head, "dinov2_reg", model, anomaly)
    b = _hot_path(large_sds, stego_head, "dinov2_reg", model, anomaly)
    y, yv = _labels(a, 4)
    _check_per_pixel_against_composed(a, b, _img(2), y, yv, exact=model == "SimpleMLP" and not anomaly)


@pytest.mark.parametrize("seg_type,model,per_pixel", [("slic", "SimpleMLP", True), ("grid", "SimpleMLP", True),
                                                      ("slic", "SimpleGCN", False), ("grid", "DoubleMLP", False)])
def test_step_on_slic_and_grid(large_sds, stego_head, seg_type, model, per_pixel):
    kw = dict(segmentation_type=seg_type, prediction_per_pixel=per_pixel)
    a = _hot_path(large_sds, stego_head, "dinov2", model, False, **kw)
    b = _hot_path(large_sds, stego_head, "dinov2", model, False, **kw)
    assert a.fe._stego is None
    y, yv = _labels(a, 5)
    if per_pixel:
        _check_per_pixel_against_composed(a, b, _img(3), y, yv, exact=True)
    else:
        _check_against_composed(a, b, _img(3), y, yv, exact=model != "SimpleGCN")


@pytest.mark.parametrize("variant,seg_type,model,per_pixel", [("dinov2_reg", "stego", "SimpleMLP", True),
                                                              ("dinov2", "slic", "SimpleGCN", False)])
def test_capture_replay_equals_eager(large_sds, stego_head, variant, seg_type, model, per_pixel):
    kw = dict(segmentation_type=seg_type, prediction_per_pixel=per_pixel)
    a = _hot_path(large_sds, stego_head, variant, model, False, **kw)
    b = _hot_path(large_sds, stego_head, variant, model, False, **kw)
    y, yv = _labels(a, 9)
    _check_replay(a, b, y, yv)
