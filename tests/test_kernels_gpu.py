"""GPU parity tests of the individual sm_90a kernels against plain PyTorch fp32 references.

Tolerances (stated per test): bf16 tensor-core kernels are compared with an fp32 reference
evaluated on the SAME bf16-rounded operands, so the only differences are accumulation order and
the bf16 rounding of the output: rel-L2 <= 4e-3 and max-abs <= 2^-7 * scale.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


@pytest.fixture(scope="module")
def ops():
    from wild_visual_navigation_b200 import ops as o

    return o


@pytest.mark.parametrize("M,N,K,bn", [
    (128, 128, 64, 128), (300, 384, 384, 0), (1000, 1152, 384, 192), (777, 1536, 384, 256), (512, 384, 1536, 0),
    (130, 448, 64, 224), (4096, 64, 256, 64), (128 * 150, 384, 192, 128), (25600, 1152, 384, 0), (12800, 1536, 384, 0),
    # odd 128-row block count + row tail, long K (1536), 256- and 128-wide tiles
    (25600 + 128 + 37, 1152, 384, 0), (20000, 384, 1536, 0), (19200, 512, 384, 0), (19000, 640, 128, 128),
])
@pytest.mark.parametrize("out_kind,act", [(0, 0), (0, 1), (0, 2), (1, 0), (2, 0)])
def test_gemm(ops, M, N, K, bn, out_kind, act):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = (torch.randn(M, K, device="cuda", generator=g)).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    ref = a.float() @ w.float().T + bias
    if act == 1:
        ref = torch.relu(ref)
    elif act == 2:
        ref = torch.nn.functional.gelu(ref)
    if out_kind == 2:
        base = torch.randn(M, N, device="cuda", generator=g)
        out = base.clone()
        ops.gemm_bf16(a, w, bias, out_kind=2, out=out, block_n=bn)
        ref = ref + base
    else:
        out = ops.gemm_bf16(a, w, bias, out_kind=out_kind, act=act, block_n=bn)
    torch.cuda.synchronize()
    tol = 6e-3 if out_kind == 0 else 2e-5 * math.sqrt(K) + 1e-4
    assert rel_l2(out.float(), ref) < tol, (rel_l2(out.float(), ref), tol)
    assert torch.isfinite(out.float()).all()


def test_gemm_no_bias_and_repeat(ops):
    a = torch.randn(256, 128, device="cuda").bfloat16()
    w = torch.randn(192, 128, device="cuda").bfloat16()
    r1 = ops.gemm_bf16(a, w, None, out_kind=1)
    r2 = ops.gemm_bf16(a, w, None, out_kind=1)
    torch.cuda.synchronize()
    assert torch.equal(r1, r2)  # deterministic
    assert rel_l2(r1, a.float() @ w.float().T) < 1e-5


@pytest.mark.parametrize("B,H,n_valid", [(1, 1, 128), (2, 3, 200), (1, 6, 3137), (2, 2, 1025)])
def test_attention(ops, B, H, n_valid):
    npad = (n_valid + 127) // 128 * 128
    g = torch.Generator(device="cuda").manual_seed(n_valid)
    q = torch.randn(B, H, npad, 64, device="cuda", generator=g).bfloat16()
    k = (torch.randn(B, H, npad, 64, device="cuda", generator=g) * 1.5).bfloat16()
    v = torch.randn(B, H, npad, 64, device="cuda", generator=g).bfloat16()
    # poison the padding rows of K/V with large finite values: they must be masked out
    k[:, :, n_valid:] = 50.0
    v[:, :, n_valid:] = 1000.0
    out = ops.attention(q, k, v.transpose(2, 3).contiguous(), n_valid, 0.125)
    torch.cuda.synchronize()
    qf, kf, vf = q.float(), k.float()[:, :, :n_valid], v.float()[:, :, :n_valid]
    att = torch.softmax(qf @ kf.transpose(-1, -2) * 0.125, dim=-1)
    ref = (att @ vf).transpose(1, 2).reshape(B, npad, H * 64)
    got = out.float()
    # P is rounded to bf16 before P·V and the output to bf16: rel-L2 <= 1e-2
    assert rel_l2(got[:, :n_valid], ref[:, :n_valid]) < 1e-2, rel_l2(got[:, :n_valid], ref[:, :n_valid])
    assert torch.isfinite(got).all()


def test_attention_peaked_softmax(ops):
    """Large logit spread: the running row maximum grows by more than 2^8 between tiles."""
    B, H, n_valid, npad = 1, 2, 640, 640
    g = torch.Generator(device="cuda").manual_seed(1)
    q = (torch.randn(B, H, npad, 64, device="cuda", generator=g) * 4).bfloat16()
    k = (torch.randn(B, H, npad, 64, device="cuda", generator=g) * 4).bfloat16()
    # make later keys progressively more aligned with the queries
    k = (k.float() + q.float().mean(2, keepdim=True) * torch.linspace(0, 3, npad, device="cuda")[None, None, :, None]).bfloat16()
    v = torch.randn(B, H, npad, 64, device="cuda", generator=g).bfloat16()
    out = ops.attention(q, k, v.transpose(2, 3).contiguous(), n_valid, 0.125).float()
    att = torch.softmax(q.float() @ k.float().transpose(-1, -2) * 0.125, dim=-1)
    ref = (att @ v.float()).transpose(1, 2).reshape(B, npad, H * 64)
    assert rel_l2(out, ref) < 1.5e-2, rel_l2(out, ref)


@pytest.mark.parametrize("dim", [384, 768])
def test_layernorm(ops, dim):
    x = torch.randn(1000, dim, device="cuda") * 3 + 0.5
    gmm = torch.randn(dim, device="cuda")
    bta = torch.randn(dim, device="cuda")
    out = ops.layernorm(x, gmm, bta, 1e-6).float()
    ref = torch.nn.functional.layer_norm(x, (dim,), gmm, bta, 1e-6)
    assert (out - ref).abs().max() < 2 ** -7 * ref.abs().max()
    assert rel_l2(out, ref) < 3e-3


def test_upsample_dense_matches_torch(ops):
    tok = torch.randn(2, 14 * 14, 96, device="cuda")
    out = ops.upsample_dense(tok, 14, 14, 112, 112)
    ref = torch.nn.functional.interpolate(tok.reshape(2, 14, 14, 96).permute(0, 3, 1, 2), (112, 112), mode="bilinear",
                                          align_corners=True)
    assert (out - ref).abs().max() < 1e-5


def test_logits_argmax_pruned_candidates_two_ranges(ops):
    """Spatially smooth logits (1-3 classes can win per interpolation cell -> the candidate-pruned path) for two probe
    ranges resolved in one pass, against torch's upsample + argmax."""
    B, g, npad, Ka, Kb = 3, 28, 896, 32, 27
    gen = torch.Generator(device="cuda").manual_seed(5)
    yy, xx = torch.meshgrid(torch.arange(g, device="cuda").float(), torch.arange(g, device="cuda").float(), indexing="ij")
    def field(K):
        cy = torch.rand(B, K, generator=gen, device="cuda") * g
        cx = torch.rand(B, K, generator=gen, device="cuda") * g
        d = (yy[None, None] - cy[:, :, None, None]) ** 2 + (xx[None, None] - cx[:, :, None, None]) ** 2
        return (-d / 20 + 0.05 * torch.randn(B, K, g, g, generator=gen, device="cuda")).permute(0, 2, 3, 1)  # (B,g,g,K)
    fa, fb = field(Ka), field(Kb)
    logits = torch.zeros(B * npad, 128, device="cuda")
    v = logits.view(B, npad, 128)
    v[:, 1 : 1 + g * g, 8 : 8 + Ka] = fa.reshape(B, g * g, Ka)
    v[:, 1 : 1 + g * g, 64 : 64 + Kb] = fb.reshape(B, g * g, Kb)
    sa, sb = ops.logits_argmax(logits, 8, Ka, B, npad, g, g, 224, 224, col0_b=64, classes_b=Kb)
    for got, f in ((sa, fa), (sb, fb)):
        ref = torch.nn.functional.interpolate(f.permute(0, 3, 1, 2), (224, 224), mode="bilinear", align_corners=False).argmax(1)
        agree = (got == ref).float().mean().item()
        assert agree > 0.9995, agree


def test_logits_argmax_matches_upstream_order(ops):
    """argmax(bilinear_upsample(logits)) == argmax(probe(bilinear_upsample(code)))."""
    B, g, K, npad = 2, 7, 11, 128
    logits = torch.zeros(B * npad, 64, device="cuda")
    grid = torch.randn(B, g * g, K, device="cuda")
    logits.view(B, npad, 64)[:, 1 : 1 + g * g, 8 : 8 + K] = grid
    seg = ops.logits_argmax(logits, 8, K, B, npad, g, g, 56, 56)
    ref = torch.nn.functional.interpolate(grid.reshape(B, g, g, K).permute(0, 3, 1, 2), (56, 56), mode="bilinear",
                                          align_corners=False).argmax(1)
    assert (seg == ref).float().mean() > 0.999
