"""Element-wise tests of the ViT's memory-bound kernels (csrc/vit_kernels.cu) and of the kernels between the token grid
and image resolution (csrc/dense_kernels.cu), against float64 / exactly emulated references.

The end-to-end bars (tokens within rel-L2 2e-2 after twelve blocks, >= 98 % label agreement) cannot see a NEAREST
source column off by one, a crop offset off by one, a wrong register row or a flip about the wrong axis: each moves a
few patches of a frame.  Here every output element is held to its own bound, every output buffer sits between NaN
sentinels that must stay untouched, and the cases are chosen to hit the edges.  u = 2^-24 (fp32 unit roundoff).

Patch loader (wvn_image_to_patches): integer index work plus two fp32 operations, so it is checked BIT-EXACTLY against
torch: F.interpolate(mode="nearest") on fp32 (source index min(floor(dst * fp32(in / out)), in - 1), the kernel's
formula), the crop int(round((resized - S) / 2)) (half to even), the flip of the whole S-wide crop, im2col in
(c, ky, kx) order and bf16(fp32(fp32(px - mean_f32) * inv_std_f32)), px = fp32(u8) / 255 for uint8 input.  Against the
float64 (px - mean) / std every element also lies within
    2^-8 |ref| + 4 u |ref| + 2 u |mean| / std
(bf16 rounding <= 2^-9 |got|; mean_f32 and inv_std_f32 = fp32(1 / fp32(std)) carry u and 2u relative error, the
subtraction and the product u each; the absolute term is mean_f32's error, which does not scale with |ref| when px
is close to the mean).

Token rows (wvn_init_token_rows): bit-exact, CLS = fp32(cls + pos[0]), registers = reg, padding = +0, patch rows untouched.

LayerNorm (wvn_layernorm_ex), two-pass in fp32, one warp per row (each lane sums D / 32 values as
((a + b) + (c + d)) groups, then a 5-level butterfly): every summation path has at most k = D / 128 + 7 additions.
First-order error terms, with m*, d* = x - m*, rstd* = 1 / sqrt(var* + eps) and y* the float64 values:
    mean       E_m = (k + 2) u mean|x|                 (k additions, the fp32 1/D, the product)
    d          |d - d*| <= E_m + u |d*|
    rstd       rel <= ((k + 1) + 3) u / 2 + 4 u + E_m^2 / (2 (var* + eps))
               (squares and sum, * 1/D, + eps: halved by the square root; rsqrtf's 2 ulp = 4 u; E_m^2 is the variance
                a mean error adds)
    y          |y - y*| <= |g| rstd* (E_m + |d*| (rel_rstd + 3 u)) + u |y*|   (d rstd, * g, + b: three roundings)
The fp32 bound is twice this first-order sum (the doubling covers the neglected second-order terms); the bf16 output
adds half a bf16 ulp of the value returned.  Rows of mean 1e3 / std 1 reject one-pass variance, rows whose variance is
about eps reject eps outside the square root, ordinary rows reject the unbiased variance (CPU controls below).  Rows of
one constant c are held to the same bound, and rows of zeros (what padding rows hold) come out as beta exactly.  A
nonzero constant does not: nvcc contracts the mean's product into the subtraction, d = fma(-sum, fp32(1/D), c), so
d = -c * D * (fp32(1/D) - 1/D) = -c 2^-25 instead of 0 (measured on the H100: |y - beta| = 3.0e-5 c |gamma|, what
1 / sqrt(eps) makes of that d), which is inside E_m.

upsample_tokens_dense (align_corners=True) at the kernel's fp32 source coordinates s = fp32(dst * fp32((in-1)/(out-1))),
i0 = min(int(s), in - 1), w = s - i0 (exact): the float64 blend of the four corners with those weights, bound
    8 u * sum |corner weight * corner value|
(1 - w for x and for y, the x-blend's product and sum, the y-blend's product and sum: six roundings to first order,
with two more for the second-order terms).

logits_argmax (align_corners=False): the kernel's source coordinate (dst + 0.5) * scale - 0.5 may be evaluated with one
rounding (fused) or two, so the float64 reference uses the exact coordinate s64 of the fp32 scale and allows
|s - s64| <= 2^-22 (|s64| + 1), which moves the blend by at most that times twice the largest corner value.  Blend
bound = 8 u sum |w v| (as above) + that coordinate term.  The label must be the float64 argmax wherever the float64
top-2 gap exceeds twice the bound; elsewhere the chosen class lies within twice the bound of the maximum.  Exact ties
resolve to the lower index.

flip_average: bit-exact against fp32 0.5 * (a + b).

attention_f32_debug: float64 softmax(q k^T scale) v on the same fp32 qkv.  Per query row, E_s = 64 u sum|q k| scale +
u max|s| bounds a score's error (64 sequential FMAs, the subtraction of the running max); with n = n_valid keys and
R = ceil(n / 16) possible rescales, the weights' relative error is rel = 2 E_s + (n + 10 R + 8) u (exp 4 u, the running
sums of l and of o over n keys, each rescale's alpha and its two products), and
    |got - ref| <= 2^-8 |ref| + 2 rel * (P |V|)
(the bf16 output, then the error of o and of l, each bounded by rel P|V|).

No constant here is measured.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

U = 2.0 ** -24
BF16_NAN_BITS = 0x7FC1
GUARD = 64  # sentinel elements before and after every output buffer
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)


@pytest.fixture(scope="module")
def ops():
    import __graft_entry__ as g

    g.build()
    from wild_visual_navigation_b200 import _C, ops as o

    _C.require_device()
    return o


# ------------------------------------------------------------------------------------------------ sentinels
def guarded(n, dtype, device="cuda"):
    """A flat buffer of n + 2 GUARD NaN elements -> (buffer, its middle n elements as a contiguous view)."""
    if dtype == torch.bfloat16:
        buf = torch.full((n + 2 * GUARD,), BF16_NAN_BITS, dtype=torch.int16, device=device).view(torch.bfloat16)
    else:
        buf = torch.full((n + 2 * GUARD,), float("nan"), dtype=dtype, device=device)
    return buf, buf[GUARD : GUARD + n]


def bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def assert_guards(buf, tag):
    """The GUARD elements on both sides of the output are still the NaN sentinel, bit for bit."""
    want = BF16_NAN_BITS if buf.dtype == torch.bfloat16 else None
    for part in (buf[:GUARD], buf[-GUARD:]):
        if want is None:
            assert bool(torch.isnan(part).all()), f"{tag}: a sentinel outside the output was overwritten"
        else:
            assert bool((bits(part) == want).all()), f"{tag}: a sentinel outside the output was overwritten"


def assert_within(got, ref, bound, tag):
    got = got.double()
    err = (got - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{tag}: {int(bad.sum())} of {bad.numel()} elements outside the bound; first at {idx}: "
                             f"got {got[idx].item():.9g} ref {ref[idx].item():.9g} bound {bound[idx].item():.3g}")


def assert_bits_equal(got, want, tag):
    ne = bits(got.contiguous()) != bits(want.contiguous())
    if bool(ne.any()):
        idx = tuple(int(i) for i in ne.nonzero()[0])
        raise AssertionError(f"{tag}: {int(ne.sum())} of {ne.numel()} elements differ; first at {idx}: "
                             f"got {got[idx].item()!r} want {want[idx].item()!r}")


def bf16_half_ulp(x):
    """Half the spacing of bf16 values at |x| (0 at x == 0)."""
    _, e = torch.frexp(x.double())
    h = torch.ldexp(torch.ones_like(x, dtype=torch.float64), (e - 9).to(torch.int32))
    return torch.where(x == 0, torch.zeros_like(h), h)


# ------------------------------------------------------------------------------------------------ patch loader
def resized_size(h, w, size):
    """torchvision Resize(size:int): the smaller edge becomes size, the other int(size * long / short)."""
    return (size, int(size * w / h)) if h <= w else (int(size * h / w), size)


# (image_size, patch, in_h, in_w, uint8, batch, frame0, src_frames, flip_from, resized_hw or None)
PATCH_CASES = [
    (224, 8, 224, 224, False, 2, 0, 2, 1 << 30, None),          # no resize
    (224, 8, 224, 375, True, 2, 0, 2, 1 << 30, (224, 375)),     # unresized 375-wide frame: crop round(75.5) = 76
    (224, 14, 270, 360, False, 2, 0, 2, 1 << 30, None),
    (224, 16, 404, 300, True, 2, 0, 2, 1 << 30, None),          # portrait
    (224, 14, 480, 640, False, 4, 1, 2, 2, None),                # TTA: frame0 > 0, src_frames < batch, flip inside
    (448, 8, 480, 640, True, 2, 0, 2, 1 << 30, None),           # 448 x 597: row 238 floors differently in fp64
    (448, 8, 540, 720, False, 2, 0, 2, 1, None),                 # crop round(74.5) = 74; flip from frame 1
    (448, 14, 720, 1280, True, 1, 0, 1, 1 << 30, None),         # 448 x 796: row 308 floors differently in fp64
    (448, 16, 120, 160, False, 2, 0, 2, 1 << 30, None),          # upsampling
    (448, 16, 300, 404, True, 2, 0, 2, 1 << 30, None),
    (518, 8, 480, 640, False, 4, 0, 2, 2, None),                 # 518 % 8 = 6: flipped pass (second half of the batch)
    (518, 8, 270, 360, True, 2, 0, 2, 1 << 30, None),
    (518, 14, 540, 720, False, 2, 0, 2, 1, None),                # 518 = 37 * 14
    (518, 16, 120, 160, True, 2, 0, 2, 1 << 30, None),          # 518 % 16 = 6, upsampling
    (518, 14, 224, 224, False, 3, 2, 3, 3, None),                # upsampled square input, flip from frame 3 - 2 = 1
    (230, 8, 270, 360, False, 4, 0, 2, 2, None),                 # 230 % 8 = 6: STEGO's second pass
    (230, 14, 300, 404, True, 2, 0, 2, 1 << 30, None),          # 230 % 14 = 6
    (230, 16, 404, 300, False, 3, 1, 2, 1, None),                # 230 % 16 = 6, every frame flipped
    (230, 8, 720, 1280, True, 2, 0, 2, 1 << 30, None),
    (224, 16, 720, 1280, False, 2, 0, 2, 1, None),
]


def _case_id(c):
    S, p, h, w, u8, B, f0, src, flip, rhw = c
    return f"S{S}-p{p}-{h}x{w}-{'u8' if u8 else 'f32'}-B{B}" + (f"-tta{f0}.{src}.{flip}" if flip < (1 << 30) else "")


def _geometry(c):
    S, p, h, w, u8, B, f0, src, flip, rhw = c
    rh, rw = resized_size(h, w, S) if rhw is None else rhw
    return rh, rw, int(round((rh - S) / 2.0)), int(round((rw - S) / 2.0))


def patch_reference(img, S, p, rh, rw, batch, frame0, src_frames, flip_from):
    """-> (bf16 patch rows, float64 patch rows) [batch * g * g, 3 p p], both on the CPU."""
    img = img.cpu()
    x = img.permute(0, 3, 1, 2).float() / 255.0 if img.dtype == torch.uint8 else img.float()
    if (rh, rw) != tuple(x.shape[-2:]):
        x = F.interpolate(x, size=(rh, rw), mode="nearest")
    top, left = int(round((rh - S) / 2.0)), int(round((rw - S) / 2.0))
    x = x[:, :, top : top + S, left : left + S]
    frames = [(frame0 + f) % src_frames for f in range(batch)]
    flips = torch.tensor([frame0 + f >= flip_from for f in range(batch)])
    x = x[frames]
    x = torch.where(flips[:, None, None, None], x.flip(3), x)
    g = S // p
    x = x[:, :, : g * p, : g * p]
    mean32 = torch.tensor(np.array(MEAN, dtype=np.float32)).view(1, 3, 1, 1)
    inv32 = torch.tensor(np.float32(1.0) / np.array(STD, dtype=np.float32)).view(1, 3, 1, 1)
    y32 = (x - mean32) * inv32
    y64 = (x.double() - torch.tensor(MEAN, dtype=torch.float64).view(1, 3, 1, 1)) / torch.tensor(
        STD, dtype=torch.float64).view(1, 3, 1, 1)

    def rows(t):
        return t.reshape(batch, 3, g, p, g, p).permute(0, 2, 4, 1, 3, 5).reshape(batch * g * g, 3 * p * p)

    return rows(y32).bfloat16(), rows(y64)


def test_patch_case_list_discriminates():
    """CPU: the case list holds a crop where half-to-even and half-up rounding differ, a covered source row or column
    whose NEAREST index differs between an fp32 and an fp64 scale (and the torch reference follows the fp32 one),
    and a non-divisible size with flipped frames; the reference flips the whole crop."""
    half_even = fp64_row = nondiv_flip = False
    for c in PATCH_CASES:
        S, p, h, w, u8, B, f0, src, flip, rhw = c
        rh, rw, top, left = _geometry(c)
        for r, crop in ((rh, top), (rw, left)):
            if (r - S) % 2 == 1 and crop != math.floor((r - S) / 2.0 + 0.5):
                half_even = True
        for n_in, n_out, off in ((h, rh, top), (w, rw, left)):
            if n_in == n_out:
                continue
            idx = np.arange(off, off + S // p * p)
            f32 = np.minimum(np.floor(idx.astype(np.float32) * (np.float32(n_in) / np.float32(n_out))), n_in - 1)
            f64 = np.minimum(np.floor(idx * (n_in / n_out)), n_in - 1)
            # what torch's nearest resize picks: resize an image of source indices
            src_idx = torch.arange(n_in, dtype=torch.float32)[None, None, :, None].expand(1, 1, n_in, 2)
            picked = F.interpolate(src_idx, size=(n_out, 2), mode="nearest")[0, 0, off : off + S // p * p, 0].numpy()
            assert np.array_equal(picked, f32), (c, "torch nearest does not use the fp32 scale")
            fp64_row |= bool((f32 != f64).any())
        if S % p and flip < f0 + B:
            nondiv_flip = True
    assert half_even and fp64_row and nondiv_flip
    # the flip mirrors the whole S-wide crop: patch column 0 of a flipped 230 / 8 frame starts at crop column 229
    img = torch.arange(230, dtype=torch.float32).view(1, 1, 1, 230).expand(1, 3, 230, 230).contiguous() / 1000
    b16, y64 = patch_reference(img, 230, 8, 230, 230, 1, 0, 1, 0)
    assert y64[0, 0].item() == pytest.approx((0.229 - MEAN[0]) / STD[0])


@pytest.mark.gpu
@pytest.mark.parametrize("case", PATCH_CASES, ids=_case_id)
def test_image_to_patches_bit_exact(ops, case):
    S, p, h, w, u8, B, f0, src, flip, rhw = case
    rh, rw, _, _ = _geometry(case)
    gen = torch.Generator().manual_seed(S * 31 + p * 7 + h + w)
    if u8:
        img = torch.randint(0, 256, (src, h, w, 3), generator=gen, dtype=torch.uint8)
    else:
        img = torch.rand(src, 3, h, w, generator=gen)
    g = S // p
    K, pitch = 3 * p * p, (3 * p * p + 7) // 8 * 8
    rows = B * g * g
    buf, out = guarded(rows * pitch, torch.bfloat16)
    out = out.view(rows, pitch)
    ops.image_to_patches(img.cuda(), S, p, resized_hw=(rh, rw), batch=B, frame0=f0, src_frames=src, flip_from=flip,
                         out=out)
    torch.cuda.synchronize()
    tag = _case_id(case)
    assert_guards(buf, tag)
    got = out.cpu()
    assert bool((bits(got[:, K:]) == BF16_NAN_BITS).all()), f"{tag}: pad columns [3p^2, pitch) were written"
    want, y64 = patch_reference(img, S, p, rh, rw, B, f0, src, flip)
    assert_bits_equal(got[:, :K], want, tag)
    mean_over_std = max(m / s for m, s in zip(MEAN, STD))
    bound = (2.0 ** -8 + 4 * U) * y64.abs() + 2 * U * mean_over_std
    assert_within(got[:, :K], y64, bound, tag + " vs float64")


# ------------------------------------------------------------------------------------------------ token rows
@pytest.mark.gpu
@pytest.mark.parametrize("registers,batch,npad,n_valid,dim", [
    (0, 1, 896, 785, 384),      # DINO ViT-S/8 @ 224
    (0, 3, 896, 785, 768),
    (4, 1, 384, 261, 384),      # DINOv2-reg ViT-S/14 @ 224
    (4, 3, 1408, 1374, 768),    # DINOv2-reg ViT-B/14 @ 518
])
def test_init_token_rows_bit_exact(ops, registers, batch, npad, n_valid, dim):
    gen = torch.Generator(device="cuda").manual_seed(registers + batch + dim)
    cls = torch.randn(dim, generator=gen, device="cuda")
    pos = torch.randn(n_valid - registers, dim, generator=gen, device="cuda")  # [1 + P, dim]
    reg = torch.randn(registers, dim, generator=gen, device="cuda") if registers else None
    buf, x = guarded(batch * npad * dim, torch.float32)
    x = x.view(batch, npad, dim)
    ops.init_token_rows(x, cls, pos, reg, n_valid)
    torch.cuda.synchronize()
    tag = f"init_token_rows R{registers} B{batch}"
    assert_guards(buf, tag)
    want = torch.full_like(x, float("nan"))
    want[:, 0] = cls + pos[0]
    if registers:
        want[:, 1 : 1 + registers] = reg
    want[:, n_valid:] = 0.0
    assert_bits_equal(x, want, tag)   # patch rows [1 + R, n_valid) kept their NaN sentinel


# ------------------------------------------------------------------------------------------------ LayerNorm
LN_EPS = float(np.float32(1e-6))
LN_CONSTANTS = (1.0, -2.5, 3.0, 0.75, 7.0, 0.0)


def ln_rows(rows, dim, seed, device):
    """Rows of several kinds, by row index: mean 1e3 / std 1, variance about eps (std 1e-3, mean 0), one constant
    value each, and ordinary rows N(mu, sigma^2) with mu in [-2, 2], sigma in [0.1, 3]."""
    g = torch.Generator(device=device).manual_seed(seed)
    z = torch.randn(rows, dim, generator=g, device=device, dtype=torch.float64)
    mu = (torch.rand(rows, 1, generator=g, device=device, dtype=torch.float64) - 0.5) * 4
    sig = 0.1 + 2.9 * torch.rand(rows, 1, generator=g, device=device, dtype=torch.float64)
    x = mu + sig * z
    r = torch.arange(rows, device=device)[:, None]
    x = torch.where(r % 7 == 3, 1e3 + z, x)
    x = torch.where(r % 7 == 5, 1e-3 * z, x)
    const = torch.tensor(LN_CONSTANTS, device=device, dtype=torch.float64)[(r // 11) % len(LN_CONSTANTS)]
    x = torch.where(r % 11 == 0, const.expand(rows, dim), x)
    return x.float()


def ln_reference(x, gamma, beta, eps):
    """float64 LayerNorm (biased variance, eps inside the square root) and the fp32 bound of the module docstring."""
    dim = x.shape[1]
    x64, g64, b64 = x.double(), gamma.double(), beta.double()
    m = x64.mean(1, keepdim=True)
    d = x64 - m
    var = (d * d).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    y = d * rstd * g64 + b64
    k = dim // 128 + 7
    e_m = (k + 2) * U * x64.abs().mean(1, keepdim=True)
    rel_rstd = ((k + 4) / 2 + 4) * U + e_m**2 / (2 * (var + eps))
    bound = 2 * (g64.abs() * rstd * (e_m + d.abs() * (rel_rstd + 3 * U)) + U * y.abs())
    return y, bound


def test_layernorm_checker_rejects_wrong_variants():
    """CPU: unbiased variance, eps outside the square root and one-pass variance, each computed in fp32 on the test's
    rows, fall outside the bound; a correct fp32 two-pass LayerNorm falls inside."""
    for dim in (384, 768):
        x = ln_rows(7 * 11 * 4, dim, seed=dim, device="cpu")
        g = torch.Generator().manual_seed(1)
        gamma = 1 + 0.5 * torch.randn(dim, generator=g)
        beta = 0.5 * torch.randn(dim, generator=g)
        ref, bound = ln_reference(x, gamma, beta, LN_EPS)
        m = x.mean(1, keepdim=True)
        d = x - m
        var = (d * d).mean(1, keepdim=True)
        good = d * torch.rsqrt(var + LN_EPS) * gamma + beta
        assert_within(good, ref, bound, f"fp32 two-pass D={dim}")
        variants = {
            "unbiased": d * torch.rsqrt((d * d).sum(1, keepdim=True) / (dim - 1) + LN_EPS) * gamma + beta,
            "eps outside": d / (torch.sqrt(var) + LN_EPS) * gamma + beta,
            "one-pass": d * torch.rsqrt((x * x).mean(1, keepdim=True) - m * m + LN_EPS) * gamma + beta,
        }
        for name, y in variants.items():
            with pytest.raises(AssertionError):
                assert_within(y, ref, bound, name)
    # the constant rows' sums are exact, and sum * fp32(1/D) unrounded is c (1 + 2^-25): the d the kernel sees
    for c in LN_CONSTANTS:
        for dim in (384, 768):
            r = np.float32(1) / np.float32(dim)
            assert float(np.float32(c) * np.float32(dim)) * float(r) == c * (1 + 2.0 ** -25)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [384, 768])
def test_layernorm_per_element(ops, dim):
    """8960 rows (10 frames of 896): more than the 132 * 64 warps of one grid-stride pass."""
    B, npad, n_valid = 10, 896, 785
    rows = B * npad
    x = ln_rows(rows, dim, seed=dim, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(2)
    gamma = 1 + 0.5 * torch.randn(dim, generator=g, device="cuda")
    beta = 0.5 * torch.randn(dim, generator=g, device="cuda")
    outs = {}
    for rev in (0, 1):
        buf, out = guarded(rows * dim, torch.bfloat16)
        ops.layernorm(x, gamma, beta, LN_EPS, out=out.view(rows, dim), reverse=bool(rev))
        torch.cuda.synchronize()
        assert_guards(buf, f"layernorm D={dim} reverse={rev}")
        outs[rev] = out.view(rows, dim).clone()
    assert_bits_equal(outs[1], outs[0], f"layernorm D={dim}: reverse=1 vs reverse=0")
    got = outs[0]
    ref, bound = ln_reference(x, gamma, beta, LN_EPS)
    assert_within(got, ref, bound + bf16_half_ulp(got), f"layernorm bf16 D={dim}")
    zero_rows = torch.arange(0, rows, 11, device="cuda")
    zero_rows = zero_rows[(zero_rows // 11) % len(LN_CONSTANTS) == LN_CONSTANTS.index(0.0)]
    assert_bits_equal(got[zero_rows], beta.bfloat16().expand(len(zero_rows), dim), f"zero rows D={dim}")


@pytest.mark.gpu
@pytest.mark.parametrize("dim,B,npad,n_valid,row0", [
    (384, 10, 896, 785, 1),     # DINO: CLS dropped
    (768, 23, 384, 261, 5),     # 4 registers: CLS and registers dropped; 8832 rows
])
def test_layernorm_fp32_token_output(ops, dim, B, npad, n_valid, row0):
    rows = B * npad
    x = ln_rows(rows, dim, seed=dim + row0, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(4)
    gamma = 1 + 0.5 * torch.randn(dim, generator=g, device="cuda")
    beta = 0.5 * torch.randn(dim, generator=g, device="cuda")
    keep = n_valid - row0
    bbuf, ob = guarded(rows * dim, torch.bfloat16)
    fbuf, of = guarded(B * keep * dim, torch.float32)
    ops.layernorm(x, gamma, beta, LN_EPS, out=ob.view(rows, dim), out_f32=of.view(B * keep, dim), npad=npad,
                  n_valid=n_valid, row0=row0, reverse=True)
    torch.cuda.synchronize()
    tag = f"layernorm fp32 tokens row0={row0}"
    assert_guards(bbuf, tag)
    assert_guards(fbuf, tag)
    got_b = ob.view(B, npad, dim)
    got_f = of.view(B, keep, dim)
    ref, bound = ln_reference(x, gamma, beta, LN_EPS)
    ref, bound = ref.view(B, npad, dim)[:, row0:n_valid], bound.view(B, npad, dim)[:, row0:n_valid]
    assert_within(got_f, ref, bound, tag)
    assert_bits_equal(got_f.bfloat16(), got_b[:, row0:n_valid], tag + ": bf16(fp32 output) vs bf16 output")


# ------------------------------------------------------------------------------------------------ upsample_tokens_dense
def _ac_true_coords(n_in, n_out, device):
    scale = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0)
    s = np.arange(n_out, dtype=np.float32) * scale
    i0 = np.minimum(s.astype(np.int64), n_in - 1)
    i1 = np.minimum(i0 + 1, n_in - 1)
    w = s.astype(np.float64) - i0
    t = lambda a: torch.tensor(a, device=device)
    return t(i0), t(i1), t(w)


def bilinear_reference(tok, gh, gw, out_h, out_w, y_coords, x_coords):
    """tok [B, gh, gw, K] -> float64 blend [B, out_h, out_w, K] and sum |w v| over the four corners."""
    (y0, y1, wy), (x0, x1, wx) = y_coords, x_coords
    t = tok.double()
    wy, wx = wy[None, :, None, None], wx[None, None, :, None]
    v00, v01 = t[:, y0][:, :, x0], t[:, y0][:, :, x1]
    v10, v11 = t[:, y1][:, :, x0], t[:, y1][:, :, x1]
    ref = (1 - wy) * ((1 - wx) * v00 + wx * v01) + wy * ((1 - wx) * v10 + wx * v11)
    s = (1 - wy) * ((1 - wx) * v00.abs() + wx * v01.abs()) + wy * ((1 - wx) * v10.abs() + wx * v11.abs())
    return ref, s


UPSAMPLE_CASES = [  # (B, gh, gw, out_h, out_w, dim)
    (2, 14, 14, 224, 224, 384), (2, 14, 14, 1, 1, 90), (1, 28, 28, 57, 91, 90), (1, 28, 28, 100, 100, 33),
    (1, 37, 37, 518, 518, 33), (1, 64, 64, 448, 448, 33), (1, 64, 64, 127, 200, 384), (2, 7, 12, 1, 13, 90),
    (2, 7, 12, 50, 97, 90), (1, 7, 12, 5, 1, 384),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", UPSAMPLE_CASES, ids=lambda c: "B{}-{}x{}-to-{}x{}-D{}".format(*c))
def test_upsample_tokens_dense_per_element(ops, case):
    B, gh, gw, oh, ow, D = case
    g = torch.Generator(device="cuda").manual_seed(gh * 100 + gw + D)
    tok = torch.randn(B, gh * gw, D, generator=g, device="cuda") * (1 + torch.rand(D, generator=g, device="cuda") * 4)
    buf, out = guarded(B * D * oh * ow, torch.float32)
    from wild_visual_navigation_b200 import _C

    _C.check(_C.lib().wvn_upsample_dense(_C.ptr(tok), _C.ptr(out), B, D, gh, gw, oh, ow, _C.stream()))
    torch.cuda.synchronize()
    tag = "upsample B{} {}x{} -> {}x{} D{}".format(*case)
    assert_guards(buf, tag)
    got = out.view(B, D, oh, ow).permute(0, 2, 3, 1)
    ref, s = bilinear_reference(tok.view(B, gh, gw, D), gh, gw, oh, ow, _ac_true_coords(gh, oh, "cuda"),
                                _ac_true_coords(gw, ow, "cuda"))
    assert_within(got, ref, 8 * U * s, tag)


# ------------------------------------------------------------------------------------------------ logits_argmax
def _ac_false_coords(n_in, n_out, device):
    """Exact (float64) coordinate of the fp32 scale, its corner indices and weights, and the coordinate tolerance."""
    scale = np.float32(n_in) / np.float32(n_out)
    s = np.maximum((np.arange(n_out, dtype=np.float64) + 0.5) * np.float64(scale) - 0.5, 0.0)
    i0 = np.minimum(s.astype(np.int64), n_in - 1)
    i1 = np.minimum(i0 + 1, n_in - 1)
    t = lambda a: torch.tensor(a, device=device)
    return (t(i0), t(i1), t(s - i0)), t(2.0 ** -22 * (s + 1))


LOGIT_CASES = [  # (grid, out_h, out_w, col0, classes, col0_b, classes_b, ld)
    (28, 224, 224, 4, 5, 16, 27, 48),
    (28, 270, 360, 0, 32, 36, 64, 104),
    (64, 518, 518, 4, 5, 16, 27, 48),
    (64, 224, 224, 0, 32, 36, 64, 104),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", LOGIT_CASES, ids=lambda c: "g{}-{}x{}-K{}-{}".format(c[0], c[1], c[2], c[4], c[6]))
def test_logits_argmax_labels(ops, case):
    grid, oh, ow, col0, ka, col0_b, kb, ld = case
    B = 3
    P = grid * grid
    npad = (1 + P + 127) // 128 * 128
    g = torch.Generator(device="cuda").manual_seed(grid + ka)
    logits = torch.full((B, npad, ld), 1e30, device="cuda")   # CLS, padding and other columns: a wrong read wins
    fields, tie = {}, {}
    for name, c0, K in (("a", col0, ka), ("b", col0_b, kb)):
        f = torch.randn(B, grid, grid, K, generator=g, device="cuda")
        # an exact tie between classes 1 and K - 2 at the top of a 6 x 6 block of patches
        f[:, 4:10, 4:10, K - 2] = f[:, 4:10, 4:10, 1] = f[:, 4:10, 4:10].amax(-1) + 3.0
        fields[name], tie[name] = f, 1
        logits[:, 1 : 1 + P, c0 : c0 + K] = f.reshape(B, P, K)
    sa, sb = ops.logits_argmax(logits.view(B * npad, ld), col0, ka, B, npad, grid, grid, oh, ow, col0_b=col0_b,
                               classes_b=kb)
    (yc, ey), (xc, ex) = _ac_false_coords(grid, oh, "cuda"), _ac_false_coords(grid, ow, "cuda")
    for name, got, K in (("a", sa, ka), ("b", sb, kb)):
        tag = "logits_argmax g{} {}x{} K{}".format(grid, oh, ow, K)
        f = fields[name]
        ref, s = bilinear_reference(f, grid, grid, oh, ow, yc, xc)
        vmax = f.abs().amax(-1)  # per patch: the coordinate term's largest corner value
        cmax = torch.maximum(torch.maximum(vmax[:, yc[0]][:, :, xc[0]], vmax[:, yc[0]][:, :, xc[1]]),
                             torch.maximum(vmax[:, yc[1]][:, :, xc[0]], vmax[:, yc[1]][:, :, xc[1]])).double()
        bound = (8 * U * s).amax(-1) + (ey[None, :, None] + ex[None, None, :]) * 2 * cmax
        assert got.shape == (B, oh, ow) and bool(((got >= 0) & (got < K)).all()), tag
        top2 = ref.topk(2, dim=-1).values
        clear = (top2[..., 0] - top2[..., 1]) > 2 * bound
        assert clear.float().mean().item() > 0.9, f"{tag}: too few pixels have a clear winner"
        want = ref.argmax(-1)
        bad = clear & (got != want)
        assert not bool(bad.any()), f"{tag}: {int(bad.sum())} clear labels wrong; first at {bad.nonzero()[0].tolist()}"
        chosen = ref.gather(-1, got[..., None])[..., 0]
        assert bool((chosen >= top2[..., 0] - 2 * bound).all()), f"{tag}: a chosen class is not within the bound"
        # pixels whose four corner patches all lie in the tie block: the lower class index wins
        iny = (yc[0] >= 4) & (yc[1] <= 9)
        inx = (xc[0] >= 4) & (xc[1] <= 9)
        sel = iny[:, None] & inx[None, :]
        assert int(sel.sum()) > 0
        assert bool((got[:, sel] == tie[name]).all()), f"{tag}: exact ties must resolve to the lower index"


@pytest.mark.gpu
def test_logits_argmax_refuses_ranges_past_the_row(ops):
    from wild_visual_navigation_b200._C import WvnError

    B, g, npad = 1, 7, 128
    logits = torch.zeros(B * npad, 16, device="cuda")
    ops.logits_argmax(logits, 8, 8, B, npad, g, g, 14, 14)                       # columns [8, 16): fits
    with pytest.raises(WvnError):
        ops.logits_argmax(logits, 12, 5, B, npad, g, g, 14, 14)                  # reads [12, 20)
    with pytest.raises(WvnError):
        ops.logits_argmax(logits, 0, 4, B, npad, g, g, 14, 14, col0_b=8, classes_b=9)  # second range reads [8, 20)


# ------------------------------------------------------------------------------------------------ flip_average
@pytest.mark.gpu
@pytest.mark.parametrize("grid,ld,B", [(28, 90, 2), (37, 37, 1), (64, 257, 2)])
def test_flip_average_bit_exact(ops, grid, ld, B):
    P = grid * grid
    npad = (1 + P + 127) // 128 * 128
    g = torch.Generator(device="cuda").manual_seed(grid)
    buf, head = guarded(2 * B * npad * ld, torch.float32)
    head.copy_(torch.randn(2 * B * npad * ld, generator=g, device="cuda") * 3)
    before = head.clone().view(2 * B, npad, ld)
    ops.flip_average(head.view(2 * B * npad, ld), B, npad, grid)
    torch.cuda.synchronize()
    tag = f"flip_average g{grid} ld{ld}"
    assert_guards(buf, tag)
    after = head.view(2 * B, npad, ld)
    a = before[:B, 1 : 1 + P].view(B, grid, grid, ld)
    m = before[B:, 1 : 1 + P].view(B, grid, grid, ld).flip(2)
    want = torch.zeros(B, npad, ld, device="cuda")
    want[:, 1 : 1 + P] = (0.5 * (a + m)).view(B, P, ld)
    assert_bits_equal(after[:B], want, tag)
    assert_bits_equal(after[B:], before[B:], tag + ": flipped half")


# ------------------------------------------------------------------------------------------------ attention_f32_debug
@pytest.mark.gpu
@pytest.mark.parametrize("heads,n_valid", [(6, 785), (12, 1370), (6, 257)])
def test_attention_f32_debug_per_element(ops, heads, n_valid):
    B, scale, dim = 2, 0.125, heads * 64
    npad = (n_valid + 127) // 128 * 128
    g = torch.Generator(device="cuda").manual_seed(n_valid + heads)
    q = torch.randn(B, npad, heads, 64, generator=g, device="cuda")
    k = torch.randn(B, npad, heads, 64, generator=g, device="cuda")
    v = torch.randn(B, npad, heads, 64, generator=g, device="cuda")
    # every 7th query row points along a per-head direction that the last valid key shares: most of its mass is there
    u = torch.randn(1, 1, heads, 64, generator=g, device="cuda")
    u = u / u.norm(dim=-1, keepdim=True)
    q[:, ::7] = 12 * u
    k[:, n_valid - 1] = 12 * u[:, 0]
    v[:, n_valid - 1] += 4
    sign = torch.where(torch.rand(B, npad - n_valid, heads, 64, generator=g, device="cuda") < 0.5, -1.0, 1.0)
    k[:, n_valid:] = 1e4 * sign
    v[:, n_valid:] = -1e4 * sign
    qkv = torch.cat([q.reshape(B, npad, dim), k.reshape(B, npad, dim), v.reshape(B, npad, dim)], -1)
    qkv = qkv.reshape(B * npad, 3 * dim).contiguous()
    buf, out = guarded(B * npad * dim, torch.bfloat16)
    ops.attention_f32_debug(qkv, B, heads, npad, n_valid, scale, out=out.view(B * npad, dim))
    torch.cuda.synchronize()
    tag = f"attention_f32_debug H{heads} n{n_valid}"
    assert_guards(buf, tag)
    got = out.view(B, npad, heads, 64).permute(0, 2, 1, 3)
    q64, k64, v64 = (t.double().permute(0, 2, 1, 3)[:, :, :n] for t, n in ((q, npad), (k, n_valid), (v, n_valid)))
    s = q64 @ k64.transpose(-1, -2) * scale
    p = torch.softmax(s, dim=-1)
    ref, pv = p @ v64, p @ v64.abs()
    R = (n_valid + 15) // 16
    e_s = 64 * U * (q64.abs() @ k64.abs().transpose(-1, -2) * scale).amax(-1, keepdim=True) + U * s.abs().amax(-1, keepdim=True)
    rel = 2 * e_s + (n_valid + 10 * R + 8) * U
    assert_within(got, ref, 2.0 ** -8 * ref.abs() + 2 * rel * pv, tag)
    assert (p[:, :, ::7, -1].min().item()) > 0.9   # the peaked rows really sit on the last valid key


# ------------------------------------------------------------------------------------------------ STEGO end to end
@pytest.mark.gpu
def test_stego_flip_tta_at_non_divisible_size():
    """StegoInterface at 230 px (230 % 8 = 6) with the flip TTA: its code against oracle.stego_head.stego_inference on
    wvn_transform frames, whose second pass flips the whole 230-wide transformed image before the stride-8 conv."""
    from oracle.dino_vit import ViTConfig, synthetic_state_dict, vit_feature_map
    from oracle.stego_head import stego_inference, synthetic_head
    from oracle.wvn_path import wvn_transform
    from wild_visual_navigation_b200.feature_extractor import StegoInterface

    S = 230
    cfg = ViTConfig.from_name("vit_small", 8, S)
    sd = synthetic_state_dict(cfg, seed=6)
    hd = synthetic_head(384, 90, 32, 27, seed=3)
    si = StegoInterface("cuda", input_size=S, backbone_type="vit_small", patch_size=8, head_state_dict=hd,
                        backbone_state_dict=sd, flip_tta=True, max_batch=2)
    H, W = 270, 360
    img = torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(7)).cuda()
    si.inference(img)
    sdc = {k: v.cuda() for k, v in sd.items()}
    hdc = {k: v.cuda() for k, v in hd.items()}
    timg = wvn_transform(img, S)
    feats = vit_feature_map(timg, sdc, cfg)
    feats_f = vit_feature_map(timg.flip(dims=[3]), sdc, cfg)
    code_ref, _, _ = stego_inference(feats, feats_f, hdc, (S, S), out_h=H)
    code = si.features
    rel = ((code - code_ref).norm() / code_ref.norm()).item()
    print("stego 230 flip-TTA code rel_l2", rel)
    assert rel <= 3e-2
