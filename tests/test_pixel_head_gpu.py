"""The fused per-pixel traversability head (pixel_head.cu) pixel by pixel against a float64 reference on its own
operands, at every token-window width, across frame chunks, and where tokens share a large common component.

The head interpolates G = tokens W1^T + b1 instead of x and evaluates the reconstruction loss as
    D loss = h2^T (R^T R) h2 + 2 (R^T c).h2 + c.c - 2 (h2.U + cT_hi + cT_lo) + |x|^2,     U = tokens R, cT = tokens c
so an error that moves trav / conf by less than the end-to-end bars (2e-2 / 3e-2) is invisible there.  Here every
pixel is held to its own bound.

Reference (float64, per frame on the device): tokens, W1, W2, w0 = W3[0] and R = W3[1:] rounded to bf16; b1, b2, b3
in fp32; h1 = bf16(ReLU(bilinear(G))); h2 = ReLU(W2 h1 + b2) without rounding; x = bilinear(bf16 tokens);
trav = sigmoid(w0.h2 + b0); D loss = |R h2 + c - x|^2.  The source rows / columns and blend weights are the kernel's
(ac_true in float32), so the bound carries no interpolation-weight error; test_interpolation_weights_match_torch
checks those weights against F.interpolate(align_corners=True).

Bound, layer by layer (u = 2^-24, C_ACC the GEMM accumulator constant of test_kernel_edges_gpu, K1 = dim_p):
  G      per token: C_ACC K1 u (|t| |W1|^T + |b1|) + 2^-23 |G|; the vertical and horizontal fp32 blends
         (fma(w, b - a, a)) add at most 7 u max|G| over the pixel's four source tokens, and carry the token errors
         through weights that sum to 1: eG = max4(e_token + 7 u |G_token|).
  h1     bf16(ReLU(.)) is monotone, so the kernel's h1 lies between the roundings of G - eG and G + eG: d1 is the
         larger distance from the reference h1 to either (a rounding decision that may flip).
  h2     e2 = d1 |W2|^T + C_ACC 256 u ((|h1| + d1) |W2|^T + |b2|) + 2^-23 |z2|; ReLU is 1-Lipschitz.
  trav   logit error e2.|w0| + 33 u (h2+.|w0| + |b0|) (32 fma), then mlp_head_ref's rule (trav_ref).
  loss   D dloss <=
         2 |R^T (r - x)|.e2 + | |R| e2 |^2               h2's error, exactly: |d + R e|^2 - |d|^2
         + (D/4 + 71) u Q,   Q = | |R| h2+ + |c| |^2       R^T R, 2 R^T c, c.c (4 chains of D/4 fma, two adds) and the
                                                          epilogue's quadratic form (2 x 33 fma)
         + 2 [h2+.eU + e_cT + 34 u (h2+.|U| + |cT_hi| + |cT_lo|)]     cross term: U and cT GEMM bounds (as for G,
                                                          blended), the residual |x|.|c - c_hi - c_lo| (~2^-17 |c|),
                                                          and the 33-term fp32 dot product
         + (K1/32 + 25) u X,  X = | bilinear(|t|) |^2    token Gram (K1/32 fma per lane, 5 shuffles) and its two
                                                          blends (phase A and the epilogue)
         + 2 u (Q + 2 XR + X),  XR = bilinear(|t|).(|R| h2+ + |c|)    q - 2 cross + gram in fp32: bounded by the
                                                          terms' magnitudes, not by the (cancelled) result
         then the clamp at 0 (1-Lipschitz, the reference is >= 0) and the division by D (+ 2 u loss).
         h2+ = h2 + e2 bounds the kernel's h2.
  conf   mlp_head_ref's Lipschitz rule (conf_ref) on that loss bound.
Only the GEMM terms carry C_ACC; every CUDA-core sum is bounded by its worst case (n u per n-term chain).

Reading the loss: with cg_mean = 0, std_factor = 0.5 and cg_std = s, lo = 0 and hi = 1.5 s.  Setting hi just above
the largest reference loss makes conf = 1 - loss / hi at every pixel, so conf carries the loss (the "loss window").
Each case runs again with lo / hi at the 20 % / 80 % quantiles of the loss (the "quantile window"), where pixels must
clamp at both ends and fall between.

Worst error / bound ratios are printed at the end of the module (pytest -s) and recorded in DESIGN.md §4.
"""
import os
import sys
from ctypes import c_void_p

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_kernel_edges_gpu as edges  # noqa: E402
from test_kernel_edges_gpu import (C_ACC, U24, assert_owned_and_untouched, assert_within, conf_ref,  # noqa: E402
                                   mlp_head_ref, sentinel, trav_ref)

U = U24
H1, H2 = 256, 32
TILE_W, WIN_MAX = 64, 10   # pixel_head.cu kTileW / kWinMax

_CANCEL = {}   # |m| / |x'| -> [worst |loss err|, worst loss err / bound, worst |conf err|, median cancellation factor]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    tags = {k: v for k, v in edges._WORST.items() if k.startswith("ph_")}
    if tags:
        print("\nfused pixel head, worst error / bound:")
        for tag in sorted(tags):
            print(f"  {tag:34s} {tags[tag][0]:.4f}")
    if _CANCEL:
        print("common component |m| / |x'|: worst |loss err|, worst loss err/bound, worst |conf err| (quantile window), "
              "median (|q| + 2|cross| + |gram|) / (D loss)")
        for r in sorted(_CANCEL):
            a, b, c, d = _CANCEL[r]
            print(f"  {r:4g}   {a:.3e}   {b:.4f}   {c:.3e}   {d:.1f}")


def _cancel_record(ratio, loss_err, loss_ratio, conf_err, factor):
    old = _CANCEL.get(ratio, [0.0, 0.0, 0.0, factor])
    _CANCEL[ratio] = [max(old[0], loss_err), max(old[1], loss_ratio), max(old[2], conf_err), factor]


# ------------------------------------------------------------------------------------------------ geometry emulation
F32 = np.float32


def ac_true(n_out, n_in):
    """The kernels' align_corners=True source index and weight of every destination, in float32 (pixel_head.cu /
    dense_kernels.cu): s = dst * fp32((n_in - 1) / (n_out - 1)), i0 = min(int(s), n_in - 1), w = s - i0."""
    scale = F32(F32(n_in - 1) / F32(n_out - 1))
    s = np.arange(n_out, dtype=F32) * scale
    i0 = np.minimum(s.astype(np.int64), n_in - 1)
    return i0, (s - i0.astype(F32)).astype(F32)


def window_width(gh, gw, H, W):
    """pixel_head_supported: the token-window width ww of a 2 x 64 tile, 0 when the fused head does not take it."""
    if H % 2 or W % TILE_W or H < 2 or W < 2:
        return 0
    sx = F32(F32(gw - 1) / F32(W - 1))
    ww = int(F32(TILE_W - 1) * sx) + 3
    return ww if 2 <= ww <= WIN_MAX else 0


def _tables(n_out, n_in, dev):
    i0, w = ac_true(n_out, n_in)
    i1 = np.minimum(i0 + 1, n_in - 1)
    return (torch.from_numpy(i0).to(dev), torch.from_numpy(i1).to(dev), torch.from_numpy(w.astype(np.float64)).to(dev))


def _corners(Q, ty, tx, rows):
    """The four source values of every pixel in output rows `rows` of a per-token map Q [gh, gw, C]."""
    y0, y1, wy = (t[rows] for t in ty)
    x0, x1, wx = tx
    top, bot = Q[y0], Q[y1]
    return top[:, x0], top[:, x1], bot[:, x0], bot[:, x1], wy[:, None, None], wx[None, :, None]


def bilerp(Q, ty, tx, rows):
    q00, q01, q10, q11, wy, wx = _corners(Q, ty, tx, rows)
    out = (1 - wy) * ((1 - wx) * q00 + wx * q01) + wy * ((1 - wx) * q10 + wx * q11)
    return out.reshape(-1, Q.shape[-1])


def max4(Q, ty, tx, rows):
    q00, q01, q10, q11, _, _ = _corners(Q, ty, tx, rows)
    return torch.maximum(torch.maximum(q00, q01), torch.maximum(q10, q11)).reshape(-1, Q.shape[-1])


def _bf(t):
    """Round to bf16 the way the kernels do (fp32, then round-to-nearest bf16), back in float64."""
    return t.float().bfloat16().double()


def _relu_bf16_flip(v, e, relu=True):
    """bf16(ReLU(v)) and the largest distance to bf16(ReLU(v')) over |v' - v| <= e: both steps are monotone, so the
    kernel's value lies between the roundings of v - e and v + e (a rounding decision that may flip)."""
    act = (lambda z: z.clamp_min(0)) if relu else (lambda z: z)
    a = _bf(act(v))
    lo, hi = _bf(act(v - 1.01 * e)), _bf(act(v + 1.01 * e))
    return a, torch.maximum(a - lo, hi - a)


# ------------------------------------------------------------------------------------------------ operands and data
def head_operands(sd, rounded=True):
    """The fused head's operands in float64.  rounded=False: the unrounded model (the product definition)."""
    r = _bf if rounded else (lambda t: t.double())
    W3, b3 = sd["layers.4.weight"], sd["layers.4.bias"]
    c32 = b3[1:].float()
    if rounded:
        c_hi = c32.bfloat16().float()
        c_lo = (c32 - c_hi).bfloat16().float()   # c - c_hi is exact in fp32
    else:
        c_hi, c_lo = c32, torch.zeros_like(c32)
    c = c32.double()
    D = W3.shape[0] - 1
    return {"D": D, "K1": (D + 63) // 64 * 64, "rounded": rounded,
            "W1": r(sd["layers.0.weight"]), "b1": sd["layers.0.bias"].double(),
            "W2": r(sd["layers.2.weight"]), "b2": sd["layers.2.bias"].double(),
            "w0": r(W3[0]), "b0": b3[0].double(), "R": r(W3[1:]), "c": c,
            "c_hi": c_hi.double(), "c_lo": c_lo.double(), "c_res": c - c_hi.double() - c_lo.double()}


def make_weights(D, dev, ratio=0.0, variant="", seed=42):
    """oracle.wvn_path.mlp_init (seeded) scaled by 3, as test_pixel_inference_vs_oracle does.  With a common token
    component m (ratio > 0): b3[1:] = m, the reconstruction's offset a trained head learns, and b1 -= W1 m, so the
    hidden layers see only the deviation from m and D loss stays O(D) while |x|^2, q and 2 cross grow as |m|^2 (the
    cancellation regime).  variant "wide": the logit row scaled so that trav saturates at both ends; "fixed_h2": W2 = 0,
    so h2 = ReLU(b2) exactly and the loss's bound is free of h1's rounding (which otherwise dominates it): the cross,
    Gram and quadratic-form terms are then resolved at their own size."""
    from oracle.wvn_path import mlp_init

    sd = {k: 3.0 * v.to(dev) for k, v in mlp_init(D, seed=seed).items()}
    m = None
    if ratio:
        g = torch.Generator(device=dev).manual_seed(seed + 1)
        m = ratio * torch.randn(D, generator=g, device=dev)
        sd["layers.4.bias"][1:] = m
        sd["layers.0.bias"] -= sd["layers.0.weight"] @ m
    if variant == "wide":
        sd["layers.4.weight"][0] *= 40.0
    if variant == "fixed_h2":
        sd["layers.2.weight"].zero_()
    flat = torch.cat([sd[k].reshape(-1) for k in ("layers.0.weight", "layers.0.bias", "layers.2.weight",
                                                  "layers.2.bias", "layers.4.weight", "layers.4.bias")])
    return sd, flat, m


def make_tokens(B, P, D, dev, m=None, seed=7):
    """B + 1 frames of unit-variance tokens (+ m); the last frame is never read (the head runs on B frames)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    t = torch.randn(B + 1, P, D, generator=g, device=dev)
    return t if m is None else t + m


# ------------------------------------------------------------------------------------------------ references
def fused_head_ref(tok, op, gh, gw, H, W, tx_override=None, chunk_px=1 << 16):
    """One frame: tok [P, D] fp32 -> float64 [H*W] maps: logit, logit_bound, loss, loss_bound, x_dot_clo, cancel."""
    dev = tok.device
    D, K1 = op["D"], op["K1"]
    W1, b1, W2, b2, w0, b0, R, c = (op[k] for k in ("W1", "b1", "W2", "b2", "w0", "b0", "R", "c"))
    t = _bf(tok) if op["rounded"] else tok.double()
    ta = t.abs()
    ty = _tables(H, gh, dev)
    tx = _tables(W, gw, dev) if tx_override is None else tx_override

    def gemm(w, bias=None):   # per-token GEMM value and its bound (test_kernel_edges_gpu.gemm_bound, fp32 output)
        v = t @ w.T if w.dim() == 2 else t @ w
        s = ta @ w.abs().T if w.dim() == 2 else ta @ w.abs()
        if bias is not None:
            v, s = v + bias, s + bias.abs()
        return v, C_ACC * K1 * U * s + 2.0 ** -23 * v.abs()

    Gt, eGt = gemm(W1, b1)
    Ut, eUt = gemm(R.T)
    ch, ech = gemm(op["c_hi"])
    cl, ecl = gemm(op["c_lo"])
    vals = torch.cat([Gt, Ut, ch[:, None], cl[:, None]], 1).view(gh, gw, -1)
    errs = torch.cat([eGt + 7 * U * Gt.abs(), eUt + 7 * U * Ut.abs(),
                      (ech + ecl + 7 * U * (ch.abs() + cl.abs()) + ta @ op["c_res"].abs())[:, None],
                      Ut.abs(), (ch.abs() + cl.abs())[:, None]], 1).view(gh, gw, -1)
    t3, ta3 = t.view(gh, gw, D), ta.view(gh, gw, D)
    xclo_t = (t @ op["c_lo"]).view(gh, gw, 1)
    out = {k: torch.empty(H * W, dtype=torch.float64, device=dev)
           for k in ("logit", "logit_bound", "loss", "loss_bound", "x_dot_clo", "cancel")}
    Ra, w0a = R.abs(), w0.abs()
    rows_per = max(1, chunk_px // W)
    for y in range(0, H, rows_per):
        rows = torch.arange(y, min(H, y + rows_per), device=dev)
        sl = slice(y * W, (y + len(rows)) * W)
        v = bilerp(vals, ty, tx, rows)
        e = max4(errs, ty, tx, rows)
        G, Upx = v[:, :H1], v[:, H1:H1 + H2]
        eG, eU, ecT = e[:, :H1], e[:, H1:H1 + H2], e[:, H1 + H2]
        aU, acT = e[:, H1 + H2 + 1:H1 + 2 * H2 + 1], e[:, -1]
        if op["rounded"]:
            a1, d1 = _relu_bf16_flip(G, eG)
        else:
            a1, d1 = G.clamp_min(0), torch.zeros_like(G)
        z2 = a1 @ W2.T + b2
        e2 = d1 @ W2.abs().T + C_ACC * H1 * U * ((a1.abs() + d1) @ W2.abs().T + b2.abs()) + 2.0 ** -23 * z2.abs()
        h2 = z2.clamp_min(0)
        hp = h2 + e2
        out["logit"][sl] = h2 @ w0 + b0
        out["logit_bound"][sl] = e2 @ w0a + 33 * U * (hp @ w0a + b0.abs())
        x = bilerp(t3, ty, tx, rows)
        xa = bilerp(ta3, ty, tx, rows)
        d = h2 @ R.T + c - x
        Dl = (d * d).sum(1)
        rabs = hp @ Ra.T + c.abs()
        Q, X, XR = (rabs * rabs).sum(1), (xa * xa).sum(1), (xa * rabs).sum(1)
        Db = (2 * ((d @ R).abs() * e2).sum(1) + ((e2 @ Ra.T) ** 2).sum(1)
              + (D / 4 + 71) * U * Q
              + 2 * ((hp * eU).sum(1) + ecT + 34 * U * ((hp * aU).sum(1) + acT))
              + (K1 / 32 + 25) * U * X
              + 2 * U * (Q + 2 * XR + X))
        out["loss"][sl] = Dl / D
        out["loss_bound"][sl] = Db / D + 2 * U * Dl / D
        out["x_dot_clo"][sl] = bilerp(xclo_t, ty, tx, rows)[:, 0]
        out["cancel"][sl] = (Q + 2 * XR + X) / Dl.clamp_min(1e-30)
    return out


def unfused_head_ref(tok, sd, gh, gw, H, W, chunk_px=1 << 16):
    """One frame of the unfused path (interp_pixel_rows + three GEMMs): x = bf16(bilinear(fp32 tokens)), then the
    bounds of test_mlp_inference_rows_end_to_end with every bf16 rounding bounded by _relu_bf16_flip.  The fp32
    interpolation is off by at most 10 u max|t| over the four source tokens before x is rounded.
    -> float64 y [H*W, D + 1] (reconstruction columns, then the logit), eps_y, x."""
    dev = tok.device
    D = tok.shape[1]
    K1 = (D + 63) // 64 * 64
    W1, b1 = _bf(sd["layers.0.weight"]), sd["layers.0.bias"].double()
    W2, b2 = _bf(sd["layers.2.weight"]), sd["layers.2.bias"].double()
    W3, b3 = _bf(sd["layers.4.weight"]), sd["layers.4.bias"].double()
    W3 = torch.cat([W3[1:], W3[:1]])      # the head's layout: reconstruction rows, then the logit
    b3 = torch.cat([b3[1:], b3[:1]])
    t3 = tok.double().view(gh, gw, D)
    ta3 = t3.abs()
    ty, tx = _tables(H, gh, dev), _tables(W, gw, dev)
    ys, es, xs = [], [], []
    rows_per = max(1, chunk_px // W)
    for y in range(0, H, rows_per):
        rows = torch.arange(y, min(H, y + rows_per), device=dev)
        x64 = bilerp(t3, ty, tx, rows)
        xb, dx = _relu_bf16_flip(x64, 10 * U * max4(ta3, ty, tx, rows), relu=False)
        z1 = xb @ W1.T + b1
        e1 = dx @ W1.abs().T + C_ACC * K1 * U * ((xb.abs() + dx) @ W1.abs().T + b1.abs()) + 2.0 ** -23 * z1.abs()
        a1, d1 = _relu_bf16_flip(z1, e1)
        z2 = a1 @ W2.T + b2
        e2 = d1 @ W2.abs().T + C_ACC * H1 * U * ((a1.abs() + d1) @ W2.abs().T + b2.abs()) + 2.0 ** -23 * z2.abs()
        a2, d2 = _relu_bf16_flip(z2, e2)
        yv = a2 @ W3.T + b3
        eps = d2 @ W3.abs().T + C_ACC * 64 * U * ((a2.abs() + d2) @ W3.abs().T + b3.abs()) + 2.0 ** -23 * yv.abs()
        eps[:, :D] += dx                      # the loss compares against the kernel's own x
        ys.append(yv), es.append(eps), xs.append(xb)
    return torch.cat(ys), torch.cat(es), torch.cat(xs)


# ------------------------------------------------------------------------------------------------ windows and checks
def loss_window(max_loss):
    """cg_mean = 0, std_factor = 0.5, cg_std = s: lo = 0, hi = 1.5 s just above the largest loss."""
    return 0.0, 1.02 * max_loss / 1.5, 0.5


def quantile_window(loss):
    flat = loss.reshape(-1)
    if flat.numel() > 1 << 22:
        flat = flat[:: (flat.numel() >> 22) + 1]
    q20, q80 = torch.quantile(flat, 0.2).item(), torch.quantile(flat, 0.8).item()
    sd, f = (q80 - q20) / 2, 0.5
    return (q20 + q80) / 2 - sd * f, sd, f


def check_maps(trav, conf, ref, cg, tag, regimes):
    """trav / conf [B, H, W] against the stacked reference maps under the window cg = (mean, std, std_factor)."""
    tr = trav_ref(ref["logit"], ref["logit_bound"])
    assert_within(trav.reshape(-1), tr["trav"], tr["trav_bound"], f"{tag}_trav")
    cr = conf_ref(ref["loss"], ref["loss_bound"], *cg)
    assert_within(conf.reshape(-1), cr["conf"], cr["conf_bound"], f"{tag}_conf")
    if regimes:
        n = ref["loss"].numel()
        lo_n, hi_n = int((ref["loss"] < cr["lo"]).sum()), int((ref["loss"] > cr["hi"]).sum())
        assert lo_n > 0 and hi_n > 0 and n - lo_n - hi_n > 0, (lo_n, hi_n, n)
    return cr


def stack_refs(refs):
    return {k: torch.cat([r[k] for r in refs]) for k in refs[0]}


# ------------------------------------------------------------------------------------------------ CPU tests
# name: (gh, gw, H, W, batch, D, |m| / |x'|, weight variant): the fused cases run on the GPU
CASES = {
    "bench_56_448": (56, 56, 448, 448, 9, 384, 0, ""),
    "bench_56_448_b17_m4": (56, 56, 448, 448, 17, 384, 4, ""),
    "vitb8_64_512": (64, 64, 512, 512, 9, 768, 0, "wide"),
    "dinov2_32_448": (32, 32, 448, 448, 17, 384, 0, ""),
    "dinov2_37_512": (37, 37, 512, 512, 1, 768, 1, ""),
    "reg224_16_256": (16, 16, 256, 256, 9, 384, 16, ""),
    "one_token_1_2x64": (1, 1, 2, 64, 9, 384, 0, ""),
    "smallest_2_64": (2, 2, 64, 64, 17, 90, 0, ""),
    "nonsquare_24x40": (24, 40, 194, 320, 9, 202, 0, ""),
    "nonsquare_40x24": (40, 24, 322, 192, 9, 384, 4, "wide"),
    "ww3_2_128": (2, 2, 128, 128, 1, 90, 0, ""),
    "ww4_5_192": (5, 5, 192, 192, 9, 202, 0, ""),
    "ww5_8_192": (8, 8, 192, 192, 1, 768, 16, ""),
    "ww8_12_128": (12, 12, 128, 128, 17, 384, 1, ""),
    "ww9_14_128": (14, 14, 128, 128, 9, 90, 4, ""),
    "ratio1_56_448": (56, 56, 448, 448, 1, 384, 1, ""),
    "ratio16_56_448": (56, 56, 448, 448, 1, 384, 16, ""),
    "ratio16_64_512_d768": (64, 64, 512, 512, 1, 768, 16, ""),
    "fixed_h2_56_448_m4": (56, 56, 448, 448, 9, 384, 4, "fixed_h2"),
    "fixed_h2_40x24_m16": (40, 24, 322, 192, 9, 768, 16, "fixed_h2"),
    "fixed_h2_16_256": (16, 16, 256, 256, 1, 202, 0, "fixed_h2"),
}


def test_window_invariant_all_geometries():
    """For every grid g <= 128 and every W <= 4096 the fused head accepts (W a multiple of 64): every pixel's left
    window column c0 satisfies c0 <= ww - 2, so its right column is inside the window.  Otherwise the pixel's h1 row
    is never written (phase B walks cells 0 .. ww - 2) and it inherits the previous tile's."""
    accepted = 0
    for g in range(1, 129):
        for W in range(64, 4097, 64):
            ww = window_width(g, g, 2, W)
            if not ww:
                continue
            accepted += 1
            x0, _ = ac_true(W, g)
            c0 = x0 - np.repeat(x0[::TILE_W], TILE_W)
            assert c0.min() == 0 and c0.max() <= ww - 2, (g, W, ww, int(c0.max()))
    assert accepted > 5000, accepted


def test_cases_cover_every_window_width():
    """The GPU cases take the fused path with every ww the head accepts, fewer tiles than CTAs and more than two
    tiles per CTA, batches across the 8-frame chunk boundary, and D = 384 / 768 / 90 / 202 (202 % 4 != 0: the
    constants kernel's tail loop)."""
    wws = {name: window_width(*c[:4]) for name, c in CASES.items()}
    assert all(wws.values()), wws
    assert set(wws.values()) == set(range(3, WIN_MAX + 1)), sorted(set(wws.values()))
    assert wws["bench_56_448"] == WIN_MAX and wws["vitb8_64_512"] == WIN_MAX and wws["dinov2_32_448"] == 7
    tiles = {name: c[4] * (c[2] // 2) * (c[3] // TILE_W) for name, c in CASES.items()}
    assert min(tiles.values()) < 132 and max(tiles.values()) > 2 * 132
    assert {c[4] for c in CASES.values()} == {1, 9, 17} and {c[5] for c in CASES.values()} == {384, 768, 90, 202}
    assert any(c[0] != c[1] for c in CASES.values()) and all(c[2] % 4 for n, c in CASES.items() if "nonsquare" in n)


@pytest.mark.parametrize("n_in,n_out", [(56, 448), (64, 512), (32, 448), (37, 512), (16, 256), (24, 194), (40, 320),
                                        (2, 64), (9, 64), (28, 224), (128, 4096), (14, 128)])
def test_interpolation_weights_match_torch(n_in, n_out):
    """The kernels' fp32 source coordinates i0 + w equal F.interpolate(align_corners=True)'s (float64) to within
    4 fp32 ulps of the largest coordinate, with 0 <= w < 1 (the reference uses the kernel's, so weight rounding is
    not part of the bound)."""
    i0, w = ac_true(n_out, n_in)
    ramp = torch.arange(n_in, dtype=torch.float64).view(1, 1, n_in)
    src = F.interpolate(ramp, size=n_out, mode="linear", align_corners=True).view(-1).numpy()
    assert np.all(w >= 0) and np.all(w < 1)
    assert np.abs(i0 + w.astype(np.float64) - src).max() <= 4 * 2.0 ** -24 * n_in


@pytest.mark.parametrize("D,ratio", [(384, 0), (90, 0), (384, 4)])
def test_reference_matches_product_definition(D, ratio):
    """Fed unrounded operands, fused_head_ref is the product's definition: oracle.wvn_path.pixel_inference on
    F.interpolate(align_corners=True) features, trav and conf within 1e-6."""
    from oracle.wvn_path import pixel_inference

    gh, gw, H, W = 5, 9, 33, 65   # scales 1/8: the fp32 weights are exact, so both sides blend with the same ones
    sd, _, m = make_weights(D, "cpu", ratio=ratio)
    tok = make_tokens(1, gh * gw, D, "cpu", m)[0]
    ref = fused_head_ref(tok, head_operands(sd, rounded=False), gh, gw, H, W)
    mean, std, f = quantile_window(ref["loss"])
    dense = F.interpolate(tok.double().view(1, gh, gw, D).permute(0, 3, 1, 2), (H, W), mode="bilinear",
                          align_corners=True)
    sd64 = {k: v.double() for k, v in sd.items()}
    t_ref, c_ref = pixel_inference(dense, sd64, torch.tensor([mean], dtype=torch.float64),
                                   torch.tensor([std], dtype=torch.float64), f)
    conf = conf_ref(ref["loss"], ref["loss_bound"], mean, std, f)["conf"]
    assert (torch.sigmoid(ref["logit"]) - t_ref.reshape(-1)).abs().max() <= 1e-6
    assert (conf - c_ref.double().reshape(-1)).abs().max() <= 1e-6
    assert 0.1 < float(c_ref.mean()) < 0.9


def _cpu_case(gh=16, gw=16, H=128, W=128, B=1, D=384, ratio=0, variant=""):
    sd, _, m = make_weights(D, "cpu", ratio=ratio, variant=variant)
    tok = make_tokens(B, gh * gw, D, "cpu", m)
    op = head_operands(sd)
    refs = [fused_head_ref(tok[b], op, gh, gw, H, W) for b in range(B)]
    return sd, tok, op, refs


def _as_kernel(ref, cg):
    """What a correct kernel returns: the reference maps rounded to fp32."""
    return (torch.sigmoid(ref["logit"]).float(), conf_ref(ref["loss"], ref["loss_bound"], *cg)["conf"].float())


def test_checker_accepts_correct_maps():
    for ratio, variant in ((0, ""), (16, ""), (4, "fixed_h2")):
        _, _, _, refs = _cpu_case(ratio=ratio, variant=variant)
        ref = refs[0]
        for cg, regimes in ((loss_window(ref["loss"].max().item()), False), (quantile_window(ref["loss"]), True)):
            trav, conf = _as_kernel(ref, cg)
            check_maps(trav, conf, ref, cg, "cpu_positive", regimes)


def test_checker_rejects_neighbouring_blend_weight():
    """Pixel column 62 of every 64-pixel tile blended with column 63's weight (pt->wx[px + 1])."""
    gh, gw, H, W = 16, 16, 128, 128
    sd, tok, op, refs = _cpu_case(gh, gw, H, W)
    x0, x1, wx = _tables(W, gw, "cpu")
    wx_bad = wx.clone()
    wx_bad[TILE_W - 2::TILE_W] = wx[TILE_W - 1::TILE_W]
    bad = fused_head_ref(tok[0], op, gh, gw, H, W, tx_override=(x0, x1, wx_bad))
    cg = quantile_window(refs[0]["loss"])
    trav, conf = _as_kernel(bad, cg)
    with pytest.raises(AssertionError, match="outside the bound"):
        check_maps(trav, conf, refs[0], cg, "neg", False)


def _gram_lower_as_bottom(tok, gh, gw, H, W, row):
    """D loss change when the token Gram of token row `row` (not the bottom row) is built as if it had no lower
    neighbour (has_d false): v = |t00|^2 and d = an = t00.t01 for the pixels whose upper source row is `row`."""
    t = _bf(tok).view(gh, gw, -1)
    (y0, y1, wy), (x0, x1, wx) = _tables(H, gh, "cpu"), _tables(W, gw, "cpu")
    sel = (y0 == row).nonzero().view(-1)
    t00, t01, t10, t11 = t[y0[sel]][:, x0], t[y0[sel]][:, x1], t[y1[sel]][:, x0], t[y1[sel]][:, x1]
    s00_0, s00_1 = (t00 * t00).sum(-1), (t01 * t01).sum(-1)
    v_0, v_1 = (t00 * t10).sum(-1), (t01 * t11).sum(-1)
    h0, dd, an = (t00 * t01).sum(-1), (t00 * t11).sum(-1), (t01 * t10).sum(-1)
    u, w = 1 - wy[sel][:, None], wy[sel][:, None]
    ux, wxx = 1 - wx[None, :], wx[None, :]
    dnn0, dnn1 = 2 * u * w * (s00_0 - v_0), 2 * u * w * (s00_1 - v_1)
    dxx = u * w * (2 * h0 - dd - an)
    delta = torch.zeros(H, W, dtype=torch.float64)
    delta[sel] = ux * ux * dnn0 + 2 * ux * wxx * dxx + wxx * wxx * dnn1
    return delta.reshape(-1)


def test_checker_rejects_gram_without_lower_neighbour():
    """token_gram's has_d tested against gw on a grid with gh > gw: interior rows y >= gw - 1 lose their lower
    neighbour terms.  (The right and bottom border special cases themselves carry zero weight: the last token column
    and row are only ever blended with weight 0, so no checker can see them; see DESIGN.md §4.)"""
    gh, gw, H, W = 20, 12, 130, 128
    sd, tok, op, refs = _cpu_case(gh, gw, H, W)
    ref = refs[0]
    bad = dict(ref)
    bad["loss"] = ref["loss"] + _gram_lower_as_bottom(tok[0], gh, gw, H, W, gw - 1) / op["D"]
    cg = loss_window(ref["loss"].max().item())
    trav, conf = _as_kernel(bad, cg)
    with pytest.raises(AssertionError, match="outside the bound"):
        check_maps(trav, conf, ref, cg, "neg", False)


@pytest.mark.parametrize("ratio", [4, 16])
def test_checker_rejects_dropped_c_lo(ratio):
    """The c_lo row of Wcat zeroed: cross loses x.c_lo, so D loss grows by 2 x.c_lo.  With tokens m + x' and
    b3[1:] = m that shift is systematic (x ~ m at every pixel).  It is about 1e-3 of the loss at |m| / |x'| = 4, below
    the bound's h1-rounding term, so it is resolved with the fixed_h2 weights (a GPU case of its own)."""
    _, _, op, refs = _cpu_case(ratio=ratio, variant="fixed_h2")
    ref = refs[0]
    bad = dict(ref)
    bad["loss"] = ref["loss"] + 2 * ref["x_dot_clo"] / op["D"]
    cg = loss_window(ref["loss"].max().item())
    trav, conf = _as_kernel(bad, cg)
    with pytest.raises(AssertionError, match="outside the bound"):
        check_maps(trav, conf, ref, cg, "neg", False)


def test_checker_rejects_frame_written_over_another():
    """Frame 8's maps written over frame 0's (a chunk written without its b0 offset)."""
    _, _, _, refs = _cpu_case(2, 2, 64, 64, B=9, D=90)
    ref = stack_refs(refs)
    cg = quantile_window(ref["loss"])
    trav, conf = _as_kernel(ref, cg)
    trav, conf = trav.view(9, -1).clone(), conf.view(9, -1).clone()
    trav[0], conf[0] = trav[8], conf[8]
    with pytest.raises(AssertionError, match="outside the bound"):
        check_maps(trav, conf, ref, cg, "neg", False)


# ------------------------------------------------------------------------------------------------ GPU driver
def _p(t):
    return c_void_p(t.data_ptr())


def run_pixels(mlp, tokens, B, gh, gw, H, W, cg):
    """wvn_mlp_infer_pixels into NaN-prefilled [B + 1, H, W] maps; frame B must stay untouched."""
    from wild_visual_navigation_b200 import _C

    mean, std, f = cg
    dev = tokens.device
    cm, cs = torch.tensor([mean], device=dev), torch.tensor([std], device=dev)
    trav, conf = sentinel((B + 1, H, W), torch.float32, dev), sentinel((B + 1, H, W), torch.float32, dev)
    _C.check(_C.lib().wvn_mlp_infer_pixels(mlp._h, _p(tokens), B, gh, gw, H, W, _p(cm), _p(cs), float(f), _p(trav),
                                           _p(conf), _C.stream()))
    torch.cuda.synchronize()
    owned = torch.zeros(B + 1, H, W, dtype=torch.bool, device=dev)
    owned[:B] = True
    init = sentinel((B + 1, H, W), torch.float32, dev)
    assert_owned_and_untouched(trav, init, owned, "pixels_trav")
    assert_owned_and_untouched(conf, init, owned, "pixels_conf")
    return trav[:B], conf[:B]


def _mlp(D, flat):
    from wild_visual_navigation_b200 import ops

    mlp = ops.MlpInference(D, H1, H2)
    mlp.set_params(flat)
    return mlp


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_fused_head_pixel_by_pixel(case):
    gh, gw, H, W, B, D, ratio, variant = CASES[case]
    dev = "cuda"
    sd, flat, m = make_weights(D, dev, ratio=ratio, variant=variant)
    tok = make_tokens(B, gh * gw, D, dev, m)
    op = head_operands(sd)
    ref = stack_refs([fused_head_ref(tok[b], op, gh, gw, H, W) for b in range(B)])
    if variant == "wide":
        tr = torch.sigmoid(ref["logit"])
        assert bool((tr < 1e-9).any()) and bool((tr > 1 - 1e-9).any()), "trav does not saturate at both ends"
    mlp = _mlp(D, flat)
    tag = "ph_fused" + (f"_m{ratio:g}" if ratio else "") + (f"_{variant}" if variant else "")
    # 1. the loss window: conf = 1 - loss / hi everywhere
    cg = loss_window(ref["loss"].max().item())
    trav, conf = run_pixels(mlp, tok, B, gh, gw, H, W, cg)
    cr = check_maps(trav, conf, ref, cg, f"{tag}_losswin", regimes=False)
    hi = cr["hi"]
    loss_got = (1 - conf.reshape(-1).double()) * hi
    loss_err = (loss_got - ref["loss"]).abs()
    # 2. the quantile window: clamps at both ends and between
    cg2 = quantile_window(ref["loss"])
    trav2, conf2 = run_pixels(mlp, tok, B, gh, gw, H, W, cg2)
    cr2 = check_maps(trav2, conf2, ref, cg2, f"{tag}_quantwin", regimes=True)
    assert torch.equal(trav, trav2), "trav depends on the confidence window"
    conf_err = (conf2.reshape(-1).double() - cr2["conf"]).abs().max().item()
    if variant != "fixed_h2":
        _cancel_record(ratio, loss_err.max().item(), (loss_err / (ref["loss_bound"] * 1.0)).max().item(), conf_err,
                       ref["cancel"].median().item())


@pytest.mark.gpu
def test_handle_regrowth_bit_identical():
    """One handle run over growing token grids (16^2, 56^2, 64^2; its workspaces regrow twice) gives the same bits as
    a fresh handle per grid."""
    dev = "cuda"
    sd, flat, _ = make_weights(384, dev)
    grown = _mlp(384, flat)
    for g, S in ((16, 256), (56, 448), (64, 512)):
        tok = make_tokens(9, g * g, 384, dev, seed=g)
        cg = (0.3, 0.2, 0.5)
        a = run_pixels(grown, tok, 9, g, g, S, S, cg)
        b = run_pixels(_mlp(384, flat), tok, 9, g, g, S, S, cg)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), f"grid {g}: regrown handle differs"


@pytest.mark.gpu
def test_pixels_from_vit_matches_pixels_at_batch_9():
    """pixels_from_vit on a DINO ViT-S/8 handle at B = 9 (npad rows per frame, patch tokens from row 1, a second
    chunk starting 8 frames into the backbone's token buffer) equals pixels on the same tokens bit for bit."""
    from oracle.dino_vit import ViTConfig, synthetic_state_dict
    from wild_visual_navigation_b200 import ops

    dev = "cuda"
    cfg = ViTConfig.from_name("vit_small", 8, 448)
    vit = ops.ViTBackbone(448, 8, cfg.dim, cfg.depth, cfg.heads, cfg.mlp_dim, synthetic_state_dict(cfg, seed=3),
                          max_batch=9)
    img = torch.rand(9, 3, 448, 448, generator=torch.Generator().manual_seed(1)).to(dev)
    tokens = vit.forward(img)
    sd, flat, _ = make_weights(384, dev)
    mlp = _mlp(384, flat)
    cm, cs = torch.tensor([0.3], device=dev), torch.tensor([0.2], device=dev)
    tv, cv = mlp.pixels_from_vit(vit, 9, (448, 448), cm, cs, 0.5)
    tp, cp = mlp.pixels(tokens, (56, 56), (448, 448), cm, cs, 0.5)
    torch.cuda.synchronize()
    assert torch.isfinite(tv).all() and torch.isfinite(cv).all()
    assert torch.equal(tv, tp) and torch.equal(cv, cp)


UNFUSED = {
    "w224_28": (28, 28, 224, 224, 2, 384),       # the production output at 224 input: W % 64 != 0
    "ww11_9_64": (9, 9, 64, 64, 9, 384),          # one column past kWinMax
    "forced_56_448": (56, 56, 448, 448, 1, 90),   # a fused geometry with WVN_PIXEL_HEAD=unfused
}


def test_unfused_cases_take_the_unfused_path():
    assert window_width(*UNFUSED["w224_28"][:4]) == 0 and window_width(*UNFUSED["ww11_9_64"][:4]) == 0
    assert int(F32(TILE_W - 1) * F32(F32(8) / F32(63))) + 3 == WIN_MAX + 1
    assert window_width(*UNFUSED["forced_56_448"][:4]) == WIN_MAX


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(UNFUSED))
def test_unfused_head_pixel_by_pixel(case, monkeypatch):
    """The unfused fallback (interp_pixel_rows + three GEMMs) against unfused_head_ref, under the same windows."""
    gh, gw, H, W, B, D = UNFUSED[case]
    if case.startswith("forced"):
        monkeypatch.setenv("WVN_PIXEL_HEAD", "unfused")   # read when the handle is created
    dev = "cuda"
    sd, flat, _ = make_weights(D, dev)
    tok = make_tokens(B, gh * gw, D, dev)
    ys, es, xs = [], [], []
    for b in range(B):
        y, e, x = unfused_head_ref(tok[b], sd, gh, gw, H, W)
        ys.append(y), es.append(e), xs.append(x)
    y, eps, x = torch.cat(ys), torch.cat(es), torch.cat(xs)
    loss = ((y[:, :D] - x) ** 2).mean(1)
    mlp = _mlp(D, flat)
    for cg, regimes, win in ((loss_window(loss.max().item()), False, "losswin"), (quantile_window(loss), True, "quantwin")):
        ref = mlp_head_ref(y, eps, x, D, D, *cg)
        trav, conf = run_pixels(mlp, tok, B, gh, gw, H, W, cg)
        assert_within(trav.reshape(-1), ref["trav"], ref["trav_bound"], f"ph_unfused_{win}_trav")
        assert_within(conf.reshape(-1), ref["conf"], ref["conf_bound"], f"ph_unfused_{win}_conf")
        if regimes:
            n = loss.numel()
            lo_n, hi_n = int((loss < ref["lo"]).sum()), int((loss > ref["hi"]).sum())
            assert lo_n > 0 and hi_n > 0 and n - lo_n - hi_n > 0
