"""Element-wise edge tests of the wgmma GEMM epilogues and of attention's padded last KV tile, against float64
references computed on the same bf16 operands.

The end-to-end tolerances elsewhere (rel-L2 over 12 ViT layers, absolute error on per-pixel maps) cannot see a wrong
tail row, a wrong last token or a dropped masked KV tile: each moves the result by about 1 / n_valid of its size.
Here every output element is held to its own bound, every element a kernel does not own is checked to be untouched,
and the shapes are chosen to hit the edges: M tails, pitched operands, every tile width (BN 224 is the only one with
the n32 accumulator, 192 uses the n64 one), 1 / 2 / 3 units per CTA of the ping-pong schedule, reverse_m, QKV and
patch-embed scatters around frame boundaries, the fused MLP head across n-chunks, and attention rows whose softmax
mass sits in the masked last tile.

GEMM bound, with ref = A64 @ W64^T + bias and S = |A64| @ |W64|^T + |bias| in float64 (plus the residual base or the
positional embedding where the epilogue adds one):
    fp32 output   |got - ref| <= c * K * 2^-24 * S + 2^-23 * |ref|
    bf16 output   ... + 2^-8 * |ref|        (the output rounding)
    GELU          the accumulator term times 1.13 (max |GELU'|), + 2e-6 (the polynomial)
The first term is the fp32 accumulation over K (c = C_ACC, measured on the H100 and set at about 4x the worst ratio
observed, see DESIGN.md §4); the second covers the fp32 roundings of the bias / positional-embedding / residual
adds, which assumes c * K >= 2 (K >= 64 here).

The checkers themselves are tested on the CPU (no gpu mark): each negative control corrupts a correct result in one
place and asserts that the checker rejects it.
"""
import math
import os
import subprocess
import sys
from ctypes import byref, c_void_p

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Accumulator constant c of the GEMM bound: the worst (|err| - other terms) / (K 2^-24 S) measured over this module's
# fp32-output cases on one H100 80GB HBM3 (700 W) was 0.0175, so c is set at 4x that (DESIGN.md §4).
C_ACC = 0.07
U24 = 2.0 ** -24
GELU_LIPSCHITZ = 1.13
BF16_NAN_BITS = 0x7FC1  # a quiet bf16 NaN used as the sentinel of bf16 outputs

EPI_BF16, EPI_F32, EPI_RESID, EPI_PATCH, EPI_QKV, EPI_MLP_HEAD = 0, 1, 2, 3, 4, 5
ACT_NONE, ACT_RELU, ACT_GELU = 0, 1, 2

# worst ratios seen by this module's checks: tag -> [max |err| / bound, max accumulator ratio]
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst_ratios():
    yield
    if _WORST:
        print("\nworst error / bound per check (accumulator ratio = (|err| - other terms) / (K 2^-24 S)):")
        for tag in sorted(_WORST):
            r, a = _WORST[tag]
            print(f"  {tag:28s} err/bound {r:.4f}" + (f"   accumulator ratio {a:.4f}" if a is not None else ""))


def _record(tag, ratio, acc_ratio=None):
    old = _WORST.get(tag, [0.0, None])
    a = old[1] if acc_ratio is None else max(acc_ratio, old[1] or 0.0)
    _WORST[tag] = [max(old[0], ratio), a]


# ------------------------------------------------------------------------------------------------ checkers
def assert_within(got, ref, bound, tag, acc_scale=None, rest=None):
    """Every element of got (any float dtype) lies within bound of ref (float64).  NaN fails."""
    got = got.double()
    err = (got - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{tag}: {int(bad.sum())} of {bad.numel()} elements outside the bound; first at {idx}: "
                             f"got {got[idx].item():.9g} ref {ref[idx].item():.9g} bound {bound[idx].item():.3g}")
    if err.numel():
        acc_r = None
        if acc_scale is not None:
            acc_r = ((err - rest).clamp_min(0) / acc_scale.clamp_min(1e-300)).max().item()
        _record(tag, (err / bound.clamp_min(1e-300)).max().item(), acc_r)


def gemm_bound(ref, S, K, bf16_out, gelu=False, c=None):
    """The element-wise GEMM bound of the module docstring -> (bound, accumulator scale K 2^-24 S, other terms)."""
    c = C_ACC if c is None else c
    scale = K * U24 * S
    acc = c * scale * (GELU_LIPSCHITZ if gelu else 1.0)
    rest = 2.0 ** -23 * ref.abs()
    if bf16_out:
        rest = rest + 2.0 ** -8 * ref.abs()
    if gelu:
        rest = rest + 2e-6
    return acc + rest, scale, rest


def check_gemm(got, ref, S, K, tag, bf16_out, gelu=False, c=None):
    bound, scale, rest = gemm_bound(ref, S, K, bf16_out, gelu, c)
    assert_within(got, ref, bound, tag, scale * (GELU_LIPSCHITZ if gelu else 1.0), rest)


def gemm_ref(a, w, bias):
    """float64 A @ W^T + bias and |A| @ |W|^T + |bias| on the bf16 operands."""
    a64, w64 = a.double(), w.double()
    ref, S = a64 @ w64.T, a64.abs() @ w64.abs().T
    if bias is not None:
        ref, S = ref + bias.double(), S + bias.double().abs()
    return ref, S


def sentinel(shape, dtype, device):
    if dtype == torch.float32:
        return torch.full(shape, float("nan"), device=device)
    return torch.full(shape, BF16_NAN_BITS, dtype=torch.int16, device=device).view(torch.bfloat16)


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def assert_owned_and_untouched(after, before, owned, tag):
    """Every owned element was written (finite: the sentinel is NaN), every other element is bit-identical."""
    fin = torch.isfinite(after.float())
    miss = owned & ~fin
    if bool(miss.any()):
        idx = tuple(int(i) for i in miss.nonzero()[0])
        raise AssertionError(f"{tag}: {int(miss.sum())} owned elements not written (sentinel / non-finite); first at {idx}")
    changed = (_bits(after) != _bits(before)) & ~owned
    if bool(changed.any()):
        idx = tuple(int(i) for i in changed.nonzero()[0])
        raise AssertionError(f"{tag}: {int(changed.sum())} elements outside the output were modified; first at {idx}")


def bf16_half_ulp(x):
    """Half the spacing of bf16 values above |x| (0 at x == 0)."""
    _, e = torch.frexp(x.double())
    h = torch.ldexp(torch.ones_like(x, dtype=torch.float64), (e - 9).to(torch.int32))
    return torch.where(x == 0, torch.zeros_like(h), h)


def check_gelu_rounding(got, x, tag):
    """For exact pre-activations x: got must be the bf16 rounding of some value within 2e-6 + 2^-23 |gelu(x)| of
    gelu(x) (the polynomial's error and the fp32 arithmetic, nothing else)."""
    ref = torch.nn.functional.gelu(x.double())
    e = 2e-6 + 2.0 ** -23 * ref.abs()
    assert_within(got, ref, e + bf16_half_ulp(got.double()), tag)


def attn_ref(q, k, v, n_valid, scale, keys_end=None):
    """float64 softmax(q k^T scale) v over keys [0, keys_end or n_valid) -> (O, P|V|, max|V|) per (frame*head)."""
    n = n_valid if keys_end is None else keys_end
    q64, k64, v64 = q.double(), k[:, :n].double(), v[:, :n].double()
    O = torch.empty(q.shape, dtype=torch.float64, device=q.device)
    PV = torch.empty_like(O)
    for i in range(q.shape[0]):
        p = torch.softmax(q64[i] @ k64[i].T * scale, dim=-1)
        O[i] = p @ v64[i]
        PV[i] = p @ v64[i].abs()
    vmax = v[:, :n_valid].double().abs().amax(dim=(1, 2))
    return O, PV, vmax


def attn_bound(ref, PV, vmax):
    """|got - ref| <= 2^-7 P|V| (P rounded to bf16) + 2^-8 |ref| (bf16 output) + 1e-6 max|V|."""
    return 2.0 ** -7 * PV + 2.0 ** -8 * ref.abs() + 1e-6 * vmax[:, None, None]


def attn_inputs(B, H, n_valid, npad, seed, device):
    """Random Q / K / V with dominant-tail rows: every 5th query row points along a per-head direction u that the
    keys of the last (masked) KV tile share, so those keys carry ~96 % of the row's softmax mass even at 4096 other
    keys; their values are distinctive.  Padding K / V rows are large and finite and must be masked out.
    Returns q, k, v as [B*H, npad, 64] bf16, the dominant query rows and the first key of the last tile."""
    g = torch.Generator(device=device).manual_seed(seed)
    BH = B * H
    q = torch.randn(BH, npad, 64, generator=g, device=device)
    k = torch.randn(BH, npad, 64, generator=g, device=device)
    v = torch.randn(BH, npad, 64, generator=g, device=device)
    u = torch.randn(BH, 1, 64, generator=g, device=device)
    u = u / u.norm(dim=-1, keepdim=True)
    t0 = (n_valid - 1) // 128 * 128
    sel = torch.arange(0, npad, 5, device=device)
    q[:, sel] = 8 * u + 0.1 * torch.randn(BH, len(sel), 64, generator=g, device=device)
    nt = n_valid - t0
    k[:, t0:n_valid] = 12 * u + 0.1 * torch.randn(BH, nt, 64, generator=g, device=device)
    v[:, t0:n_valid] = 4 + torch.randn(BH, nt, 64, generator=g, device=device)
    k[:, n_valid:] = 50.0
    v[:, n_valid:] = 1000.0
    return q.bfloat16(), k.bfloat16(), v.bfloat16(), sel, t0


def gelu_poly_f32(x, coeffs):
    """The GEMM epilogue's GELU polynomial (gemm_wgmma.cu gelu_erf_fast) in fp32 with an exact exp2: the CPU stand-in
    used to show that the GELU sweep sees a coefficient change."""
    x = x.float()
    t = x.abs().clamp_max(5.5)
    p = torch.full_like(t, coeffs[0]) * t + coeffs[1]
    for c in coeffs[2:]:
        p = p * t + c
    e = torch.exp2(p.double()).float()
    return x.clamp_min(0) - t * e


GELU_COEFFS = [-0.0003865310864, 0.006509808358, -0.05048002675, -0.4613505006, -1.150225043, -1.00010848]


def gelu_sweep_values(device):
    """Every bf16 value in [-12, 12] with |x| >= 2^-12, and 0 (includes +-5.5, its neighbours and values near 1e-3)."""
    b = torch.arange(0, 1 << 16, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).float()
    b = b[torch.isfinite(b) & (b.abs() <= 12) & ((b.abs() >= 2.0 ** -12) | (b == 0))].unique()
    assert 5.5 in b.tolist() and -5.5 in b.tolist()
    return b.to(device)


def mlp_head_ref(y, eps_y, x, feat, trav_col, cg_mean, cg_std, std_factor):
    """Traversability head in float64 from the layer-3 outputs y (any column layout: y[:, :feat] reconstructs x,
    y[:, trav_col] is the logit) and their element-wise error bound eps_y.

    Bounds, derived from the accumulator bound eps_y (u = 2^-24):
      trav:  |d sigmoid / d logit| <= 1/4, so |dtrav| <= eps_logit / 4 + 2^-19 (fast exp and reciprocal);
      loss:  |(d + delta)^2 - d^2| <= 2 |d| eps + eps^2 per column, the fp32 subtraction / square / sum of feat terms
             add (feat + 4) u (|d| + eps)^2, and the division by feat u * loss:
             |dloss| <= [sum_j (2 |d_j| eps_j + eps_j^2) + (feat + 4) u sum_j (|d_j| + eps_j)^2] / feat + u loss;
      conf:  conf = 1 - (clamp(loss, lo, hi) - lo) / (hi - lo) is 1 / (hi - lo)-Lipschitz in loss, lo and hi, and
             lo / hi are computed in fp32 from the fp32 scalars (error <= eta = 8 u (|mean| + std (|f| + 2))):
             |dconf| <= (|dloss| + 2 eta) / (hi - lo) + 4 u.
    Returns dict(trav, loss, conf, *_bound)."""
    d = y[:, :feat] - x[:, :feat].double()
    eps = eps_y[:, :feat]
    loss = (d * d).sum(1) / feat
    u = U24
    dloss = ((2 * d.abs() * eps + eps * eps).sum(1) + (feat + 4) * u * ((d.abs() + eps) ** 2).sum(1)) / feat + u * loss
    out = {"loss": loss, "loss_bound": dloss}
    out.update(trav_ref(y[:, trav_col], eps_y[:, trav_col]))
    out.update(conf_ref(loss, dloss, cg_mean, cg_std, std_factor))
    return out


def trav_ref(logit, eps_logit):
    """mlp_head_ref's trav rule: sigmoid of the float64 logit, bound eps_logit / 4 + 2^-19."""
    return {"trav": torch.sigmoid(logit), "trav_bound": eps_logit / 4 + 2.0 ** -19}


def conf_ref(loss, dloss, cg_mean, cg_std, std_factor):
    """mlp_head_ref's conf rule: conf of the float64 loss and its 1 / (hi - lo)-Lipschitz bound from dloss."""
    u = U24
    mean, sd = float(cg_mean), float(cg_std)
    shifted = mean + sd * std_factor
    lo, hi = max(shifted - sd, 0.0), shifted + sd
    conf = 1 - (loss.clamp(lo, hi) - lo) / (hi - lo)
    eta = 8 * u * (abs(mean) + sd * (abs(std_factor) + 2))
    return {"conf": conf, "conf_bound": (dloss + 2 * eta) / (hi - lo) + 4 * u, "lo": lo, "hi": hi}


# ------------------------------------------------------------------------------------------------ CPU negative controls
def _cpu_gemm_case(M=150, N=128, K=128, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).bfloat16()
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, generator=g)
    got = a.float() @ w.float().T + bias          # a correct fp32 result, computed another way
    ref, S = gemm_ref(a, w, bias)
    return got, ref, S, K


def test_checker_accepts_correct_gemm_results():
    got, ref, S, K = _cpu_gemm_case()
    check_gemm(got, ref, S, K, "cpu_positive_f32", bf16_out=False)
    check_gemm(got.bfloat16(), ref, S, K, "cpu_positive_bf16", bf16_out=True)


def test_checker_rejects_neighbouring_tile_slice():
    got, ref, S, K = _cpu_gemm_case()
    got[64:128, 32:64] = got[0:64, 32:64]
    with pytest.raises(AssertionError, match="outside the bound"):
        check_gemm(got, ref, S, K, "neg", bf16_out=False)


def test_checker_rejects_tail_row_left_at_sentinel():
    got, ref, S, K = _cpu_gemm_case()
    for dtype in (torch.float32, torch.bfloat16):
        buf = sentinel((got.shape[0] + 8, got.shape[1] + 16), dtype, "cpu")
        before = buf.clone()
        M, N = got.shape
        buf[:M, :N] = got.to(dtype)
        owned = torch.zeros(buf.shape, dtype=torch.bool)
        owned[:M, :N] = True
        assert_owned_and_untouched(buf, before, owned, "cpu_positive")
        bad = buf.clone()
        bad[M - 1, :N] = before[M - 1, :N]
        with pytest.raises(AssertionError, match="not written"):
            assert_owned_and_untouched(bad, before, owned, "neg")
        with pytest.raises(AssertionError, match="outside the bound"):
            check_gemm(bad[:M, :N], ref, S, K, "neg", bf16_out=dtype == torch.bfloat16)
        bad = buf.clone()
        bad[M + 3, N + 5] = 0
        with pytest.raises(AssertionError, match="modified"):
            assert_owned_and_untouched(bad, before, owned, "neg")


def test_checker_rejects_four_bf16_ulps():
    got, ref, S, K = _cpu_gemm_case()
    out = got.bfloat16()
    i, j = divmod(int(ref.abs().argmax()), ref.shape[1])
    bits = out.view(torch.int16)
    bits[i, j] += 4                  # sign-magnitude: 4 ulps further from zero for either sign
    with pytest.raises(AssertionError, match="outside the bound"):
        check_gemm(out, ref, S, K, "neg", bf16_out=True)


def _cpu_attention_case():
    B, H, n_valid, npad = 1, 2, 129, 256
    q, k, v, sel, t0 = attn_inputs(B, H, n_valid, npad, 3, "cpu")
    ref, PV, vmax = attn_ref(q, k, v, n_valid, 0.125)
    return q, k, v, sel, t0, n_valid, ref, PV, vmax


def test_attention_checker_accepts_correct_and_rejects_swapped_row():
    q, k, v, sel, t0, n_valid, ref, PV, vmax = _cpu_attention_case()
    got = ref.float().bfloat16()
    bound = attn_bound(ref, PV, vmax)
    assert_within(got, ref, bound, "cpu_positive_attention")
    bad = got.clone()
    bad[:, 7] = got[:, 8]          # one query row replaced by the next one's
    with pytest.raises(AssertionError, match="outside the bound"):
        assert_within(bad, ref, bound, "neg")


def test_attention_checker_rejects_dropped_last_tile():
    q, k, v, sel, t0, n_valid, ref, PV, vmax = _cpu_attention_case()
    assert n_valid - t0 == 1       # a single valid key in the last tile
    dropped, _, _ = attn_ref(q, k, v, n_valid, 0.125, keys_end=t0)
    bound = attn_bound(ref, PV, vmax)
    for r in sel.tolist():
        with pytest.raises(AssertionError, match="outside the bound"):
            assert_within(dropped[:, r].float().bfloat16(), ref[:, r], bound[:, r], "neg")


def test_gelu_sweep_sees_a_changed_polynomial_coefficient():
    x = gelu_sweep_values("cpu")
    check_gelu_rounding(gelu_poly_f32(x, GELU_COEFFS).bfloat16(), x, "cpu_positive_gelu")
    mutated = list(GELU_COEFFS)
    mutated[4] = -1.151225043        # 4th significant digit of the linear coefficient
    with pytest.raises(AssertionError, match="outside the bound"):
        check_gelu_rounding(gelu_poly_f32(x, mutated).bfloat16(), x, "neg")


# ------------------------------------------------------------------------------------------------ GPU driver
def _lib():
    from wild_visual_navigation_b200 import _C

    _C.require_device()
    return _C


def _p(t):
    return c_void_p(0 if t is None else t.data_ptr())


def gemm_ex(a, w, *, epi, act=ACT_NONE, bias=None, out=None, ldo=0, M=None, N=None, block_n=0, reverse_m=0, **kw):
    """wvn_gemm_bf16_ex on torch tensors; a and out may be row-pitched views."""
    _C = _lib()
    args = _C.GemmExArgs()
    args.m = a.shape[0] if M is None else M
    args.n = w.shape[0] if N is None else N
    args.k = w.shape[1]
    args.epi, args.act, args.block_n, args.reverse_m = epi, act, block_n, reverse_m
    args.a, args.lda, args.w, args.bias = _p(a), a.stride(0), _p(w), _p(bias)
    args.out, args.ldo = _p(out), ldo or (out.stride(0) if out is not None else 0)
    for name in ("pos", "q_out", "k_out", "vt_out", "x", "trav", "conf", "loss_reco", "cg_mean", "cg_std"):
        if name in kw:
            setattr(args, name, _p(kw.pop(name)))
    for name, val in kw.items():
        setattr(args, name, val)
    _C.check(_C.lib().wvn_gemm_bf16_ex(byref(args), _C.stream()))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ plain epilogues
PLAIN = {"bf16": (EPI_BF16, ACT_NONE), "bf16_relu": (EPI_BF16, ACT_RELU), "bf16_gelu": (EPI_BF16, ACT_GELU),
         "f32": (EPI_F32, ACT_NONE), "resid": (EPI_RESID, ACT_NONE)}
BLOCK_NS = [64, 128, 192, 224, 256]
# (M, N / BN, K, extra A columns, extra output columns, bias)
SHAPES = {
    "tail1_pitched": (129, 2, 128, 64, 32, True),
    "tail63_nobias": (191, 1, 192, 0, 0, False),
    "small_pitched": (37, 1, 64, 8, 8, True),
}
UNITS = ["tiles1", "tiles_sms+1", "tiles_2sms", "tiles_2sms+5"]


def _plain_case(kind, bn, M, N, K, xa, xo, with_bias, seed):
    epi, act = PLAIN[kind]
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(M, K + xa, generator=g, device=dev).bfloat16()[:, :K]
    w = (torch.randn(N, K, generator=g, device=dev) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, generator=g, device=dev) if with_bias else None
    ldo = N + xo
    rows = M + 64
    dtype = torch.bfloat16 if epi == EPI_BF16 else torch.float32
    init = torch.randn(rows, ldo, generator=g, device=dev) if epi == EPI_RESID else sentinel((rows, ldo), dtype, dev)
    outs = []
    for rm in (0, 1):
        buf = init.clone()
        gemm_ex(a, w, epi=epi, act=act, bias=bias, out=buf, ldo=ldo, M=M, N=N, block_n=bn, reverse_m=rm)
        outs.append(buf)
    torch.cuda.synchronize()
    ref, S = gemm_ref(a, w, bias)
    if act == ACT_RELU:
        ref = ref.clamp_min(0)
    elif act == ACT_GELU:
        ref = torch.nn.functional.gelu(ref)
    if epi == EPI_RESID:
        base = init[:M, :N].double()
        ref, S = ref + base, S + base.abs()
    owned = torch.zeros(rows, ldo, dtype=torch.bool, device=dev)
    owned[:M, :N] = True
    assert_owned_and_untouched(outs[0], init, owned, f"{kind}/bn{bn}")
    check_gemm(outs[0][:M, :N], ref, S, K, f"gemm_{kind}", bf16_out=epi == EPI_BF16, gelu=act == ACT_GELU)
    # each element is one tile's fixed-order k-loop plus at most one add: the walk direction cannot change it
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), f"{kind}/bn{bn}: reverse_m=1 differs from reverse_m=0"


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("bn", BLOCK_NS)
@pytest.mark.parametrize("kind", list(PLAIN))
def test_gemm_epilogue_tails_and_pitches(kind, bn, shape):
    M, nb, K, xa, xo, with_bias = SHAPES[shape]
    _plain_case(kind, bn, M, nb * bn, K, xa, xo, with_bias, seed=M + bn + K)


@pytest.mark.gpu
@pytest.mark.parametrize("units", UNITS)
@pytest.mark.parametrize("bn", BLOCK_NS)
@pytest.mark.parametrize("kind", list(PLAIN))
def test_gemm_epilogue_units_per_cta(kind, bn, units):
    """N = BN, so tiles = m-blocks: CTAs own exactly 1, then 1 or 2, exactly 2, and up to 3 tiles (the ping-pong's
    opening pass, odd counts and the last owner not passing)."""
    sms = _sms()
    M = {"tiles1": 64, "tiles_sms+1": (sms + 1) * 64 - 17, "tiles_2sms": 2 * sms * 64,
         "tiles_2sms+5": (2 * sms + 5) * 64 - 63}[units]
    _plain_case(kind, bn, M, bn, 128, 8, 0, True, seed=bn + M)


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [64, 224, 256])
@pytest.mark.parametrize("act", [ACT_NONE, ACT_RELU, ACT_GELU])
def test_gemm_activation_sweep_one_hot(act, bn):
    """K = 64 with a one-hot W: out[i, n] = act(A[i, n % 64]) with an exact bf16 pre-activation, swept over every bf16
    value in [-12, 12] down to 2^-12 (0, +-5.5 = the polynomial's clamp and its neighbours, values around 1e-3)."""
    dev = "cuda"
    x = gelu_sweep_values(dev)
    M = (x.numel() + 63) // 64
    a = torch.zeros(M * 64, device=dev)
    a[: x.numel()] = x
    a = a.view(M, 64).bfloat16()
    N = {64: 64, 224: 448, 256: 256}[bn]
    w = torch.zeros(N, 64, device=dev)
    w[torch.arange(N), torch.arange(N) % 64] = 1
    w = w.bfloat16()
    out = sentinel((M, N), torch.bfloat16, dev)
    gemm_ex(a, w, epi=EPI_BF16, act=act, out=out, block_n=bn)
    torch.cuda.synchronize()
    pre = a.float()[:, torch.arange(N, device=dev) % 64]
    if act == ACT_NONE:
        assert torch.equal(out.float(), pre)
    elif act == ACT_RELU:
        assert torch.equal(out.float(), pre.clamp_min(0))
    else:
        ref = torch.nn.functional.gelu(pre.double())
        check_gemm(out, ref, pre.double().abs(), 64, "gelu_sweep", bf16_out=True, gelu=True)
        check_gelu_rounding(out, pre, "gelu_sweep_rounding")


# ------------------------------------------------------------------------------------------------ QKV scatter
QKV_CFG = [(384, 6, 0), (768, 12, 0), (384, 6, 64), (768, 12, 128)]   # dim, heads, block_n (0: 192 / 256)
QKV_GEOM = [(128, 3), (192, 2), (896, 1), (3200, 2)]                  # npad, frames


@pytest.mark.gpu
@pytest.mark.parametrize("npad,frames", QKV_GEOM)
@pytest.mark.parametrize("dim,heads,bn", QKV_CFG)
def test_qkv_scatter(dim, heads, bn, npad, frames):
    """Q / K [b*h, npad, 64] and V^T [b*h, 64, npad] element by element, written into frames [1, 1 + frames) of larger
    buffers (as the ViT's sub-range offsets do); the frames around them must stay bit-identical.  The last valid
    token sits alone in its 64-row tile and, like the padding rows after it, carries distinctive values."""
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(npad + dim + bn)
    n_valid = npad - 63
    M, N, K = frames * npad, 3 * dim, dim
    a = torch.randn(frames, npad, K, generator=g, device=dev)
    a[:, n_valid - 1] = 8 * torch.randn(frames, K, generator=g, device=dev) + 2
    a[:, n_valid:] = 0.5 * torch.randn(frames, npad - n_valid, K, generator=g, device=dev) - 3 + \
        torch.arange(npad - n_valid, device=dev)[None, :, None] / 16
    a = a.reshape(M, K).bfloat16()
    w = (torch.randn(N, K, generator=g, device=dev) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, generator=g, device=dev)
    tot = (frames + 2) * heads
    init_qk = sentinel((tot, npad, 64), torch.bfloat16, dev)
    init_vt = sentinel((tot, 64, npad), torch.bfloat16, dev)
    runs = []
    for rm in (0, 1):
        q, k, vt = init_qk.clone(), init_qk.clone(), init_vt.clone()
        gemm_ex(a, w, epi=EPI_QKV, bias=bias, block_n=bn, reverse_m=rm, npad=npad, dim=dim, heads=heads,
                q_out=q[heads:], k_out=k[heads:], vt_out=vt[heads:])
        runs.append((q, k, vt))
    torch.cuda.synchronize()
    ref, S = gemm_ref(a, w, bias)
    ref, S = ref.view(frames, npad, 3, heads, 64), S.view(frames, npad, 3, heads, 64)
    owned_qk = torch.zeros(tot, npad, 64, dtype=torch.bool, device=dev)
    owned_qk[heads:(frames + 1) * heads] = True
    owned_vt = owned_qk.view(tot, 64, npad)  # same frames, same element count per (frame, head)
    q, k, vt = runs[0]
    for name, got, which, owned in (("q", q, 0, owned_qk), ("k", k, 1, owned_qk), ("vt", vt, 2, owned_vt)):
        assert_owned_and_untouched(got, init_vt if name == "vt" else init_qk, owned, f"qkv_{name}")
        r = ref[:, :, which].permute(0, 2, 1, 3)   # frames, heads, npad, 64
        s = S[:, :, which].permute(0, 2, 1, 3)
        if name == "vt":
            r, s = r.transpose(2, 3), s.transpose(2, 3)
        sub = got[heads:(frames + 1) * heads].view(r.shape)
        check_gemm(sub, r, s, K, f"qkv_{name}", bf16_out=True)
    for t0, t1 in zip(runs[0], runs[1]):
        assert torch.equal(_bits(t0), _bits(t1)), "QKV: reverse_m=1 differs from reverse_m=0"


# ------------------------------------------------------------------------------------------------ patch-embed scatter
PATCH_CASES = [(784, 384, 3, 192), (784, 768, 2, 768), (3136, 384, 2, 192), (3136, 768, 1, 192), (4096, 384, 1, 192),
               (4096, 768, 3, 192)]   # patches per frame, dim, frames, K


@pytest.mark.gpu
@pytest.mark.parametrize("P,D,frames,K", PATCH_CASES)
def test_patch_embed_scatter(P, D, frames, K):
    """out[frame*npad + 1 + tok] = A[frame*P + tok] W^T + bias + pos[1 + tok]; P = 784 is not a multiple of 64, so
    tiles straddle frames.  The CLS row and the padding rows [1 + P, npad) of every frame keep their sentinel."""
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(P + D + frames)
    npad = (P + 1 + 127) // 128 * 128
    a = torch.randn(frames * P, K, generator=g, device=dev).bfloat16()
    w = (torch.randn(D, K, generator=g, device=dev) / math.sqrt(K)).bfloat16()
    bias = torch.randn(D, generator=g, device=dev)
    pos = torch.randn(1 + P, D, generator=g, device=dev)
    init = sentinel((frames * npad, D), torch.float32, dev)
    outs = []
    for rm in (0, 1):
        out = init.clone()
        gemm_ex(a, w, epi=EPI_PATCH, bias=bias, out=out, reverse_m=rm, pos=pos, tokens_in=P, npad=npad)
        outs.append(out)
    torch.cuda.synchronize()
    ref, S = gemm_ref(a, w, bias)
    pe = pos[1:].double().repeat(frames, 1)
    ref, S = ref + pe, S + pe.abs()
    rows = (torch.arange(frames, device=dev)[:, None] * npad + 1 + torch.arange(P, device=dev)[None, :]).reshape(-1)
    owned = torch.zeros(frames * npad, D, dtype=torch.bool, device=dev)
    owned[rows] = True
    assert_owned_and_untouched(outs[0], init, owned, "patch")
    check_gemm(outs[0][rows], ref, S, K, "patch", bf16_out=False)
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), "patch: reverse_m=1 differs from reverse_m=0"


# ------------------------------------------------------------------------------------------------ fused MLP head
def _mlp_cg(feat, seed, dev, std_factor=0.5):
    """ConfidenceGenerator scalars that put lo / hi at the 20 % / 80 % quantiles of the loss of _mlp_head_data's
    row distribution (estimated on 4096 rows), so that rows clamp at lo, at hi and fall between."""
    a, w, b, x = _mlp_head_data(4096, feat, seed + 1, dev)
    y = gemm_ref(a, w, b)[0]
    loss = ((y[:, :feat] - x[:, :feat].double()) ** 2).mean(1)
    q20, q80 = torch.quantile(loss, 0.2).item(), torch.quantile(loss, 0.8).item()
    sd = (q80 - q20) / 2
    mean = (q20 + q80) / 2 - sd * std_factor
    return torch.tensor([mean], device=dev), torch.tensor([sd], device=dev), std_factor


def _mlp_geom(feat):
    trav_col = (feat + 31) // 32 * 32
    N = {384: 448, 90: 128}[feat]
    ldx = (feat + 63) // 64 * 64
    return trav_col, N, ldx


def _mlp_head_data(M, feat, seed, dev):
    """Layer-3 operands as pack_mlp_kernel lays them out: A = h2 [M, 64] (32 live columns), W [N, 64] with row r < feat
    reconstructing x[r] and row trav_col the logit, zero rows / columns elsewhere; x [M, ldx] bf16."""
    trav_col, N, ldx = _mlp_geom(feat)
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.zeros(M, 64, device=dev)
    a[:, :32] = torch.randn(M, 32, generator=g, device=dev).clamp_min(0)
    w = torch.zeros(N, 64, device=dev)
    w[:feat, :32] = torch.randn(feat, 32, generator=g, device=dev) / math.sqrt(32)
    w[trav_col, :32] = torch.randn(32, generator=g, device=dev) / 2
    b = torch.zeros(N, device=dev)
    b[:feat] = 0.1 * torch.randn(feat, generator=g, device=dev)
    b[trav_col] = 0.3
    x = torch.zeros(M, ldx, device=dev)
    scale = 0.3 + 1.7 * torch.rand(M, 1, generator=g, device=dev)   # spreads the per-row loss
    x[:, :feat] = scale * torch.randn(M, feat, generator=g, device=dev)
    return a.bfloat16(), w.bfloat16(), b, x.bfloat16()


def _check_head(trav, conf, loss, M, ref, tag, regimes=True):
    assert_within(trav[:M], ref["trav"], ref["trav_bound"], f"{tag}_trav")
    if loss is not None:
        assert_within(loss[:M], ref["loss"], ref["loss_bound"], f"{tag}_loss")
    assert_within(conf[:M], ref["conf"], ref["conf_bound"], f"{tag}_conf")
    if regimes:
        lo_n = int((ref["loss"] < ref["lo"]).sum())
        hi_n = int((ref["loss"] > ref["hi"]).sum())
        assert lo_n > 0 and hi_n > 0 and M - lo_n - hi_n > 0, (lo_n, hi_n, M)


@pytest.mark.gpu
@pytest.mark.parametrize("m_case", ["1", "63", "64", "65", "sms*64+1", "2sms*64+130"])
@pytest.mark.parametrize("feat", [384, 90])
def test_mlp_head_epilogue(feat, m_case):
    """The traversability head (EPI_MLP_HEAD) driven directly.  feat 384: N = 448 at BN = 224, two n-chunks per row
    block, so the per-row loss is reduced across chunks; feat 90: one chunk of 128.  A CTA owns whole 64-row blocks:
    M = 64 * SMs + 1 and 2 * 64 * SMs + 130 give CTAs 2 and 3 blocks.  Bounds: see mlp_head_ref."""
    dev = "cuda"
    sms = _sms()
    M = {"1": 1, "63": 63, "64": 64, "65": 65, "sms*64+1": sms * 64 + 1, "2sms*64+130": 2 * sms * 64 + 130}[m_case]
    trav_col, N, ldx = _mlp_geom(feat)
    a, w, b, x = _mlp_head_data(M, feat, 11, dev)
    cg_mean, cg_std, f = _mlp_cg(feat, 11, dev)
    bn = {384: 224, 90: 128}[feat]
    runs = []
    for rm in (0, 1):
        outs = [sentinel((M + 64,), torch.float32, dev) for _ in range(3)]
        trav, conf, loss = outs
        gemm_ex(a, w, epi=EPI_MLP_HEAD, bias=b, block_n=bn, reverse_m=rm, feat=feat, trav_col=trav_col, x=x, ldx=ldx,
                trav=trav, conf=conf, loss_reco=loss, cg_mean=cg_mean, cg_std=cg_std, cg_std_factor=f)
        runs.append(outs)
    torch.cuda.synchronize()
    y, S = gemm_ref(a, w, b)
    eps_y = C_ACC * 64 * U24 * S + 2.0 ** -23 * y.abs()
    ref = mlp_head_ref(y, eps_y, x, feat, trav_col, cg_mean.item(), cg_std.item(), f)
    owned = torch.zeros(M + 64, dtype=torch.bool, device=dev)
    owned[:M] = True
    for name, t in zip(("trav", "conf", "loss"), runs[0]):
        assert_owned_and_untouched(t, sentinel((M + 64,), torch.float32, dev), owned, f"mlp_head_{name}")
    trav, conf, loss = runs[0]
    _check_head(trav, conf, loss, M, ref, "mlp_head", regimes=M >= 63)
    for t0, t1 in zip(runs[0], runs[1]):
        assert torch.equal(_bits(t0), _bits(t1)), "MLP head: reverse_m=1 differs from reverse_m=0"


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [384, 90])
def test_mlp_inference_rows_end_to_end(dim):
    """MlpInference.rows with 128-row chunks over 3 * 128 + 45 rows (several chunks and a tail).  The float64 reference
    mirrors the kernels' rounding points (x to bf16; ReLU then bf16 after layers 1 and 2), and the bound carries each
    layer's accumulator bound plus one bf16 ulp (a rounding decision that may flip) through |W| of the next layer."""
    from wild_visual_navigation_b200 import ops

    dev = "cuda"
    h1, h2, R = 256, 32, 3 * 128 + 45
    g = torch.Generator(device=dev).manual_seed(dim)
    W1 = torch.randn(h1, dim, generator=g, device=dev) / math.sqrt(dim)
    b1 = 0.1 * torch.randn(h1, generator=g, device=dev)
    W2 = torch.randn(h2, h1, generator=g, device=dev) / math.sqrt(h1) * 2
    b2 = 0.1 * torch.randn(h2, generator=g, device=dev)
    W3 = torch.randn(1 + dim, h2, generator=g, device=dev) / math.sqrt(h2)
    b3 = 0.1 * torch.randn(1 + dim, generator=g, device=dev)
    flat = torch.cat([t.reshape(-1) for t in (W1, b1, W2, b2, W3, b3)])
    x = (0.3 + 1.7 * torch.rand(R, 1, generator=g, device=dev)) * torch.randn(R, dim, generator=g, device=dev)
    mlp = ops.MlpInference(dim, h1, h2, chunk_rows=128)
    mlp.set_params(flat)

    bf = lambda t: t.bfloat16().double()  # noqa: E731
    K1, K2, K3 = (dim + 63) // 64 * 64, h1, 64
    xb = bf(x)
    z1 = xb @ bf(W1).T + b1.double()
    e1 = C_ACC * K1 * U24 * (xb.abs() @ bf(W1).abs().T + b1.double().abs()) + 2.0 ** -23 * z1.abs()
    a1 = bf(z1.clamp_min(0))
    d1 = 1.01 * e1 + 2.0 ** -7 * a1.abs()
    z2 = a1 @ bf(W2).T + b2.double()
    e2 = d1 @ bf(W2).abs().T + C_ACC * K2 * U24 * ((a1.abs() + d1) @ bf(W2).abs().T + b2.double().abs()) + \
        2.0 ** -23 * z2.abs()
    a2 = bf(z2.clamp_min(0))
    d2 = 1.01 * e2 + 2.0 ** -7 * a2.abs()
    y = a2 @ bf(W3).T + b3.double()
    S3 = (a2.abs() + d2) @ bf(W3).abs().T + b3.double().abs()
    eps = d2 @ bf(W3).abs().T + C_ACC * K3 * U24 * S3 + 2.0 ** -23 * y.abs()
    # reorder to the head's layout: columns [0, dim) reconstruct x, column dim (any index past feat) the logit
    y, eps = torch.cat([y[:, 1:], y[:, :1]], 1), torch.cat([eps[:, 1:], eps[:, :1]], 1)
    loss_all = ((y[:, :dim] - xb) ** 2).mean(1)
    q20, q80 = torch.quantile(loss_all, 0.2).item(), torch.quantile(loss_all, 0.8).item()
    sd, f = (q80 - q20) / 2, 0.5
    cg_mean = torch.tensor([(q20 + q80) / 2 - sd * f], device=dev)
    cg_std = torch.tensor([sd], device=dev)
    trav, conf = mlp.rows(x, cg_mean, cg_std, f)
    torch.cuda.synchronize()
    ref = mlp_head_ref(y, eps, xb, dim, dim, cg_mean.item(), cg_std.item(), f)
    _check_head(trav, conf, None, R, ref, "mlp_rows")


# ------------------------------------------------------------------------------------------------ attention tail tile
ATTN_GEOM = [(1, 128), (128, 128), (129, 256), (1025, 1152), (3137, 3200), (4097, 4224)]


@pytest.mark.gpu
@pytest.mark.parametrize("H", [6, 12])
@pytest.mark.parametrize("n_valid,npad", ATTN_GEOM)
def test_attention_rows_and_tail_tile(n_valid, npad, H):
    """Every query row (padding rows included) against float64 under attn_bound.  4097 / 4224 is the ViT-B 512/8
    geometry: its last KV tile holds one valid key, which carries ~96 % of the mass of every 5th query row here; for
    those rows, the same computation without the last tile must fail the bound (else the test could not see a
    dropped or mis-masked tile)."""
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
    assert_within(got, ref, bound, "attention")
    if t0 > 0:
        dropped, _, _ = attn_ref(q, k, v, n_valid, 0.125, keys_end=t0)
        rows_fail = ((dropped[:, sel] - ref[:, sel]).abs() > bound[:, sel]).any(dim=-1)
        assert bool(rows_fail.all()), f"dropping the last KV tile stays inside the bound on {int((~rows_fail).sum())} rows"


# ------------------------------------------------------------------------------------------------ ViT schedule knobs
_VIT_CHILD = r"""
import sys
import torch
sys.path.insert(0, sys.argv[1])
from oracle.dino_vit import ViTConfig, synthetic_state_dict
from wild_visual_navigation_b200 import ops
torch.cuda.set_device(0)
cfg = ViTConfig.from_name("vit_small", 8, 224)
vit = ops.ViTBackbone(224, 8, cfg.dim, cfg.depth, cfg.heads, cfg.mlp_dim, synthetic_state_dict(cfg, seed=1),
                      max_batch=6, chunk=2)
img = torch.rand(3, 3, 224, 224, generator=torch.Generator().manual_seed(0)).cuda()
tokens = vit.forward(img)
tta = vit.forward(img, flip_tta=True)
torch.cuda.synchronize()
torch.save({"tokens": tokens.cpu(), "tta": tta.cpu()}, sys.argv[2])
"""


@pytest.mark.gpu
def test_vit_schedule_knobs_bit_identical(tmp_path):
    """ViT-S/8 @224, batch 3 in chunks of 2 (a partial last chunk), plain and flip-TTA.  The knobs are read once per
    process, so each setting runs in its own subprocess: WVN_VIT_SNAKE=0 flips reverse_m of every GEMM and reverse of
    attention and LayerNorm, WVN_VIT_SUBCHUNK=1 splits the MLP half per frame, WVN_VIT_SUB_ATTN=1 writes Q / K / V^T
    at frame offsets.  Every row is computed independently and the residual adds once per element, so all settings
    must give bit-identical tokens."""
    settings = {"default": {}, "snake0": {"WVN_VIT_SNAKE": "0"}, "subchunk1": {"WVN_VIT_SUBCHUNK": "1"},
                "sub_attn1": {"WVN_VIT_SUB_ATTN": "1"}}
    flags = ["-s"] if sys.flags.no_user_site else []
    results = {}
    for name, extra in settings.items():
        env = {k: v for k, v in os.environ.items() if k not in ("WVN_VIT_SNAKE", "WVN_VIT_SUBCHUNK", "WVN_VIT_SUB_ATTN")}
        env.update(extra)
        path = str(tmp_path / f"{name}.pt")
        r = subprocess.run([sys.executable, *flags, "-c", _VIT_CHILD, ROOT, path], env=env, cwd=str(tmp_path),
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, f"{name}: exit {r.returncode}\n{r.stderr[-3000:]}"
        results[name] = torch.load(path)
    base = results["default"]
    assert torch.isfinite(base["tokens"]).all() and torch.isfinite(base["tta"]).all()
    for name, res in results.items():
        for key in ("tokens", "tta"):
            assert torch.equal(res[key].view(torch.int32), base[key].view(torch.int32)), f"{name}: {key} differ"
