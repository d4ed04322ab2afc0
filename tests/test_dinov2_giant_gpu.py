"""DINOv2 ViT-g/14 (``backbone_type="vit_giant"``: D = 1536, 40 blocks, 24 heads, SwiGLU FFN) on the sm_90a path.

  EPI_SWIGLU            the w12 GEMM's fused epilogue element by element against float64 (bound below), M in {1, 63,
                        64, 65, 4097}, N in {256, 8192}, K in {1536, 1000}; 4097 x 8192 runs 2080 tiles on fewer CTAs,
                        so both consumer warpgroups of the ping-pong store tiles.  Negative controls: gate and value
                        halves swapped, and w12 not packed, each rejected by the same check
  LayerNorm             the D = 1536 instantiation against float64 with test_vit_io_gpu.py's derived bound, both modes
  tokens                both variants at 224 and 448, B = 1 and 3, against the fp32 oracle (run on the GPU, TF32 off)
                        and a bf16-storage emulation; bars in TOKEN_BAR
  uint8 camera ingest   bit-identical to the float path; a captured forward replays to the eager tokens bit for bit
  HotPathStep           LinearRnvp (anomaly_detection=True) per-pixel and segment-wise on STEGO (``stego_backbone_type``),
                        SLIC and grid segmentation against the same work composed by hand, eager and captured; SimpleMLP,
                        DoubleMLP and SimpleGCN refuse the 1536-wide rows

EPI_SWIGLU bound.  g and v are the gate and value pre-activations (acc + bias), each within the GEMM bound of
test_kernel_edges_gpu.py, B_g = c K 2^-24 S_g + 2^-23 |g| (and B_v likewise); silu is 1.1-Lipschitz, and __expf /
__fdividef and the product add at most 2^-19 |silu(g) v| (relative).  So
    |got - ref| <= E + 2^-8 (|ref| + E),   E = 1.1 B_g (|v| + B_v) + (|silu(g)| + 1.1 B_g) B_v + 2^-19 |silu(g) v|
with ref = silu(g) v in float64 and the last term the one bf16 rounding of the output.

The bf16-storage emulation is test_dinov2_large_gpu.py's with the SwiGLU FFN: the gated product silu(x1) * x2 of the
fp32 w12 outputs is rounded to bf16 once (where the ViT-L emulation rounds the GELU output).
"""
import os
import sys
import warnings

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_dinov2_giant_oracle import ATTN_STD, D, H, giant_config, giant_state_dict, giant_tokens  # noqa: E402
from test_kernel_edges_gpu import C_ACC, U24, assert_owned_and_untouched, gemm_ex, sentinel  # noqa: E402
from test_kernel_edges_gpu import assert_within as assert_within_f64  # noqa: E402
from test_segment_maps_gpu import _check_against_composed, _check_replay, _img, _labels  # noqa: E402
from test_vit_io_gpu import (LN_CONSTANTS, LN_EPS, assert_bits_equal, assert_guards, assert_within,  # noqa: E402,F401
                             bf16_half_ulp, guarded, ln_reference, ln_rows, ops)

pytestmark = pytest.mark.gpu

EPI_SWIGLU = 7
SILU_LIPSCHITZ = 1.1
# rel-L2 bars of the tokens, set as ViT-L/14's were from the bf16 emulation's own distance from the fp32 oracle,
# measured at most 5.06e-2 over these cases (DESIGN.md §3.14): about that distance against the bf16-storage emulation,
# 1.5 times it against fp32
TOKEN_BAR = {"fp32": 7.6e-2, "bf16": 5.5e-2}


@pytest.fixture(scope="module", autouse=True)
def _fp32_reference_math():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


def rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


# ------------------------------------------------------------------------------------------------ EPI_SWIGLU
def _packed_rows(n):
    from test_dinov2_giant_oracle import packed_rows

    return packed_rows(n).cuda()


def _swiglu_ref(a, w12, bias, K):
    """float64 silu(g) v from the checkpoint-order w12 [gate; value] and its bound (module docstring)."""
    a64, w64 = a.double(), w12.double()
    half = w12.shape[0] // 2
    ref = a64 @ w64.T
    S = a64.abs() @ w64.abs().T
    if bias is not None:
        ref, S = ref + bias.double(), S + bias.double().abs()
    g, v, Sg, Sv = ref[:, :half], ref[:, half:], S[:, :half], S[:, half:]
    bg = C_ACC * K * U24 * Sg + 2.0 ** -23 * g.abs()
    bv = C_ACC * K * U24 * Sv + 2.0 ** -23 * v.abs()
    s = F.silu(g)
    out = s * v
    e = SILU_LIPSCHITZ * bg * (v.abs() + bv) + (s.abs() + SILU_LIPSCHITZ * bg) * bv + 2.0 ** -19 * out.abs()
    return out, e + 2.0 ** -8 * (out.abs() + e)


def _run_swiglu(a, w_packed, bias_packed, M, N, ldo):
    out_buf = sentinel((M, ldo), torch.bfloat16, "cuda")
    before = out_buf.clone()
    gemm_ex(a, w_packed, epi=EPI_SWIGLU, bias=bias_packed, out=out_buf, ldo=ldo, M=M, N=N)
    torch.cuda.synchronize()
    return out_buf, before


def _operands(M, N, K, seed, bias=True):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, generator=g, device="cuda").bfloat16()
    w = (torch.randn(N, K, generator=g, device="cuda") * (2.0 / K**0.5)).bfloat16()
    b = 0.5 * torch.randn(N, generator=g, device="cuda") if bias else None
    return a, w, b


def _pad_k(w, K):
    """W's rows at the GEMM's pitch round_up(K, 8)."""
    ld = (K + 7) // 8 * 8
    if ld == K:
        return w.contiguous()
    out = torch.zeros(w.shape[0], ld, dtype=w.dtype, device=w.device)
    out[:, :K] = w
    return out[:, :K]


@pytest.mark.parametrize("K", [1536, 1000])
@pytest.mark.parametrize("N", [256, 8192])
@pytest.mark.parametrize("M", [1, 63, 64, 65, 4097])
def test_swiglu_epilogue_per_element(M, N, K):
    a, w, b = _operands(M, N, K, seed=M * 7 + N + K, bias=(M != 63))
    perm = _packed_rows(N)
    wp, bp = _pad_k(w[perm], K), (None if b is None else b[perm].contiguous())
    ldo = N // 2 + 8   # a pitched output: the 8 columns past N / 2 must stay untouched
    out, before = _run_swiglu(a, wp, bp, M, N, ldo)
    ref, bound = _swiglu_ref(a, w, b, K)
    owned = torch.zeros(M, ldo, dtype=torch.bool, device="cuda")
    owned[:, :N // 2] = True
    tag = f"swiglu M={M} N={N} K={K}"
    assert_owned_and_untouched(out, before, owned, tag)
    assert_within_f64(out[:, :N // 2], ref, bound, tag)


@pytest.mark.parametrize("control", ["halves_swapped", "unpacked"])
def test_swiglu_negative_controls(control):
    """The same check rejects a w12 whose gate and value halves are swapped, and one the library did not pack."""
    M, N, K = 130, 1024, 1536
    a, w, b = _operands(M, N, K, seed=11)
    half = N // 2
    if control == "halves_swapped":
        swap = torch.cat((torch.arange(half, N), torch.arange(half)))
        perm = swap.cuda()[_packed_rows(N)]
    else:
        perm = torch.arange(N, device="cuda")
    out, _ = _run_swiglu(a, _pad_k(w[perm], K), b[perm].contiguous(), M, N, half)
    ref, bound = _swiglu_ref(a, w, b, K)
    with pytest.raises(AssertionError, match="outside the bound"):
        assert_within_f64(out, ref, bound, f"swiglu control {control}")


def test_swiglu_refuses_bad_arguments():
    from wild_visual_navigation_b200._C import WvnError

    a, w, b = _operands(64, 512, 256, seed=3)
    out = torch.empty(64, 256, dtype=torch.bfloat16, device="cuda")
    for kw in (dict(block_n=128), dict(act=2), dict(ldo=128)):
        with pytest.raises(WvnError, match="SwiGLU"):
            gemm_ex(a, w, epi=EPI_SWIGLU, bias=b, out=out, **kw)


# ------------------------------------------------------------------------------------------------ LayerNorm
def _ln_params(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return 1 + 0.5 * torch.randn(D, generator=g, device="cuda"), 0.5 * torch.randn(D, generator=g, device="cuda")


def test_layernorm_1536_bf16_per_element(ops):
    """9 frames of the 448 grid (npad 1152): 10368 rows, more than one grid-stride pass."""
    rows = 9 * 1152
    x = ln_rows(rows, D, seed=D, device="cuda")
    gamma, beta = _ln_params(2)
    outs = {}
    for rev in (0, 1):
        buf, out = guarded(rows * D, torch.bfloat16)
        ops.layernorm(x, gamma, beta, LN_EPS, out=out.view(rows, D), reverse=bool(rev))
        torch.cuda.synchronize()
        assert_guards(buf, f"layernorm D=1536 reverse={rev}")
        outs[rev] = out.view(rows, D).clone()
    assert_bits_equal(outs[1], outs[0], "layernorm D=1536: reverse=1 vs reverse=0")
    got = outs[0]
    ref, bound = ln_reference(x, gamma, beta, LN_EPS)
    assert_within(got, ref, bound + bf16_half_ulp(got), "layernorm bf16 D=1536")
    zero_rows = torch.arange(0, rows, 11, device="cuda")
    zero_rows = zero_rows[(zero_rows // 11) % len(LN_CONSTANTS) == LN_CONSTANTS.index(0.0)]
    assert_bits_equal(got[zero_rows], beta.bfloat16().expand(len(zero_rows), D), "zero rows D=1536")


@pytest.mark.parametrize("B,npad,n_valid,row0", [
    (9, 1152, 1025, 1),    # ViT-g/14 @ 448: CLS dropped
    (23, 384, 261, 5),     # ViT-g/14-reg @ 224: CLS and 4 registers dropped
])
def test_layernorm_1536_fp32_final_norm(ops, B, npad, n_valid, row0):
    rows = B * npad
    x = ln_rows(rows, D, seed=D + row0, device="cuda")
    gamma, beta = _ln_params(4)
    keep = n_valid - row0
    bbuf, ob = guarded(rows * D, torch.bfloat16)
    fbuf, of = guarded(B * keep * D, torch.float32)
    ops.layernorm(x, gamma, beta, LN_EPS, out=ob.view(rows, D), out_f32=of.view(B * keep, D), npad=npad,
                  n_valid=n_valid, row0=row0, reverse=True)
    torch.cuda.synchronize()
    tag = f"layernorm D=1536 fp32 tokens row0={row0}"
    assert_guards(bbuf, tag)
    assert_guards(fbuf, tag)
    got_b, got_f = ob.view(B, npad, D), of.view(B, keep, D)
    ref, bound = ln_reference(x, gamma, beta, LN_EPS)
    ref, bound = ref.view(B, npad, D)[:, row0:n_valid], bound.view(B, npad, D)[:, row0:n_valid]
    assert_within(got_f, ref, bound, tag)
    assert_bits_equal(got_f.bfloat16(), got_b[:, row0:n_valid], tag + ": bf16(fp32 output) vs bf16 output")


# ------------------------------------------------------------------------------------------------ tokens
@pytest.fixture(scope="module")
def giant_sds():
    """Full-depth seeded ViT-g/14 weights, drawn on the GPU (4.5 GB each in fp32)."""
    return {"dinov2": giant_state_dict(40, seed=5, device="cuda"),
            "dinov2_reg": giant_state_dict(40, seed=6, registers=True, device="cuda")}


def _di(sd, variant, image_size, **kw):
    from wild_visual_navigation_b200.feature_extractor import DinoInterface

    return DinoInterface("cuda", backbone=variant, input_size=image_size, backbone_type="vit_giant", patch_size=8,
                         state_dict=sd, **kw)


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
    Hh, C = cfg.heads, cfg.dim
    ln = lambda t, p: F.layer_norm(t, (C,), sd[p + ".weight"], sd[p + ".bias"], cfg.ln_eps)  # noqa: E731
    for i in range(cfg.depth):
        b = f"blocks.{i}."
        qkv = _bf(F.linear(_bf(ln(x, b + "norm1")), _bf(sd[b + "attn.qkv.weight"]), sd[b + "attn.qkv.bias"]))
        q, k, v = qkv.reshape(B, -1, 3, Hh, 64).permute(2, 0, 3, 1, 4)
        s = (q @ k.transpose(-2, -1)) * 0.125
        e = torch.exp(s - s.amax(-1, keepdim=True))
        o = _bf((_bf(e) @ v) / e.sum(-1, keepdim=True)).transpose(1, 2).reshape(B, -1, C)
        x = x + F.linear(o, _bf(sd[b + "attn.proj.weight"]), sd[b + "attn.proj.bias"])
        x1, x2 = F.linear(_bf(ln(x, b + "norm2")), _bf(sd[b + "mlp.w12.weight"]), sd[b + "mlp.w12.bias"]).chunk(2, -1)
        x = x + F.linear(_bf(F.silu(x1) * x2), _bf(sd[b + "mlp.w3.weight"]), sd[b + "mlp.w3.bias"])
    return ln(x, "norm")[:, 1 + R:]


def _sd(giant_sds, variant):
    return giant_sds[variant]


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("image_size", [224, 448])
@pytest.mark.parametrize("variant", ["dinov2", "dinov2_reg"])
def test_vit_giant_tokens_vs_oracles(giant_sds, variant, image_size, B):
    from oracle.wvn_path import wvn_transform

    sd = _sd(giant_sds, variant)
    cfg = giant_config(image_size)
    di = _di(sd, variant, image_size, max_batch=B)
    g, R = image_size // 14, 4 if variant == "dinov2_reg" else 0
    assert di.feature_dim == D and di.grid == g and di._model.registers == R
    img = torch.rand(B, 3, image_size, image_size, generator=torch.Generator().manual_seed(B + image_size)).cuda()
    got = di.inference_tokens(img).clone()
    ref = giant_tokens(wvn_transform(img, image_size), sd, cfg)
    emu = tokens_bf16_storage(img, sd, cfg)
    torch.cuda.synchronize()
    assert got.shape == ref.shape == emu.shape == (B, g * g, D)
    d_fp32, d_bf16, d_emu = rel_l2(got, ref), rel_l2(got, emu), rel_l2(emu, ref)
    cos = F.cosine_similarity(got, ref, dim=-1).mean().item()
    print(f"vit_giant {variant} @{image_size} B={B}: rel-L2 vs fp32 {d_fp32:.3e}, vs bf16 storage {d_bf16:.3e}; "
          f"bf16 emulation vs fp32 {d_emu:.3e}; mean cosine vs fp32 {cos:.6f}")
    assert d_fp32 <= TOKEN_BAR["fp32"] and d_bf16 <= TOKEN_BAR["bf16"] and cos >= 0.99
    # the GPU is as far from fp32 as the emulation of its rounding points is
    assert abs(d_fp32 - d_emu) <= 0.1 * d_emu


def test_vit_giant_uint8_ingest_and_capture(giant_sds):
    from oracle.wvn_path import ros_image_to_float

    di = _di(_sd(giant_sds, "dinov2_reg"), "dinov2_reg", 448, max_batch=2)
    u8 = torch.randint(0, 256, (2, 480, 640, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(6)).cuda()
    tok_u8 = di.inference_tokens(u8).clone()
    tok_f = di.inference_tokens(ros_image_to_float(u8)).clone()
    assert tok_u8.shape == (2, 1024, D)
    assert torch.equal(tok_u8, tok_f)
    # a captured forward replays to the eager tokens bit for bit
    img0, img1 = (torch.rand(2, 3, 448, 448, generator=torch.Generator().manual_seed(s)).cuda() for s in (1, 2))
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


def _hot_path(giant_sds, stego_head, variant, model, anomaly, **kw):
    from wild_visual_navigation_b200 import HotPathStep

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return HotPathStep("cuda", _sd(giant_sds, variant), stego_head, batch=3, input_size=224, chunk=32,
                           flip_tta=False, run_clustering=True, n_image_clusters=20, model=model,
                           anomaly_detection=anomaly, feature_type=variant, backbone_type="vit_giant",
                           stego_backbone_type="vit_small", **kw)


def _check_per_pixel_against_composed(a, b, img, y, yv):
    """Per-pixel maps: b runs the per-pixel head on a's tokens and trains on a's rows."""
    ra = a.step(img, y, yv)
    tb, cb = b.ti.predict_from_tokens(ra["tokens"], b.input_size)
    tb = tb.clone()
    crow = b.te.train_on_padded(ra["feat"], ra["n_segments"], y, yv)
    b.ti.refresh_weights()
    assert ra["trav"].shape == (3, 224, 224) and torch.isfinite(ra["trav"]).all()
    assert ra["conf"] is None and cb is None
    dt = (ra["trav"] - tb).abs().max().item()
    print(f"per-pixel step vs composed: |d| trav {dt:.2e}")
    assert dt <= 1e-3
    n = int(yv[:int(ra["n_segments"].sum())].sum())
    assert torch.isfinite(ra["confidence_rows"][:n]).all()
    assert (ra["confidence_rows"][:n] - crow[:n]).abs().max().item() <= 1e-4


@pytest.mark.parametrize("seg_type", ["stego", "slic", "grid"])
def test_linear_rnvp_segment_wise(giant_sds, stego_head, seg_type):
    kw = dict(segmentation_type=seg_type, prediction_per_pixel=False)
    a = _hot_path(giant_sds, stego_head, "dinov2", "SimpleMLP", True, **kw)
    b = _hot_path(giant_sds, stego_head, "dinov2", "SimpleMLP", True, **kw)
    assert a.fe.feature_dim == D and a.fe._dino._model.dim == D
    if seg_type == "stego":
        assert a.fe._stego._dino._model.dim == 384
    y, yv = _labels(a, 3)
    p0 = a.te._model.flat_params.clone()
    ra = _check_against_composed(a, b, _img(1), y, yv, exact=False)
    assert ra["feat"].shape[1:] == (a.smax, D)
    assert not torch.equal(a.te._model.flat_params, p0)


@pytest.mark.parametrize("seg_type", ["stego", "slic", "grid"])
def test_linear_rnvp_per_pixel(giant_sds, stego_head, seg_type):
    a = _hot_path(giant_sds, stego_head, "dinov2_reg", "SimpleMLP", True, segmentation_type=seg_type)
    b = _hot_path(giant_sds, stego_head, "dinov2_reg", "SimpleMLP", True, segmentation_type=seg_type)
    y, yv = _labels(a, 4)
    _check_per_pixel_against_composed(a, b, _img(2), y, yv)


@pytest.mark.parametrize("seg_type,per_pixel", [("stego", True), ("slic", False), ("grid", True)])
def test_linear_rnvp_capture_replay_equals_eager(giant_sds, stego_head, seg_type, per_pixel):
    kw = dict(segmentation_type=seg_type, prediction_per_pixel=per_pixel)
    a = _hot_path(giant_sds, stego_head, "dinov2", "SimpleMLP", True, **kw)
    b = _hot_path(giant_sds, stego_head, "dinov2", "SimpleMLP", True, **kw)
    y, yv = _labels(a, 9)
    _check_replay(a, b, y, yv)


@pytest.mark.parametrize("model", ["SimpleMLP", "DoubleMLP", "SimpleGCN"])
def test_narrow_learners_refuse_1536_rows(giant_sds, stego_head, model):
    with pytest.raises(Exception, match="1024"):
        _hot_path(giant_sds, stego_head, "dinov2", model, False, segmentation_type="grid",
                  prediction_per_pixel=model != "SimpleGCN")
