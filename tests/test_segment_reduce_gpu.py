"""The per-segment reductions (segment_kernels.cu: ops.segment_reduce, ops.relabel, ops.pool_supervision) element by
element against float64 references, on every accumulate and pooling path, at the token grids, feature widths, segment
counts, batch sizes and map shapes the pipeline produces.

The end-to-end checks elsewhere hold feat to 2e-3 max|ref|, which cannot see one pixel counted against the wrong token.
Here every output element is held to its own bound, and what a kernel must not write is checked bit for bit.

feat reference.  The kernel never forms the dense (B, D, h, h) map: feat[s] = (sum_p W[s, p] t[p]) / count[s], with
W[s, p] the sum over the segment's pixels of the bilinear (align_corners=True) weight of token p.  The reference builds
W the way the kernel does up to the blend weights: the fp32 source coordinate float32(x) * float32((g - 1) / (h - 1))
(the dense map is (h, h), so both axes use h), i0 = min(int(s), g - 1), i1 = min(i0 + 1, g - 1) and the fp32 fraction
w = s - i0, exactly as ac_true_coord forms them.  Everything after that is float64: 1 - w, the four products, the
scatter-add over pixels, W @ tokens and the division by the count.  test_reference_matches_product_definition checks
this reference against oracle/wvn_path.sparsify_features on F.interpolate(align_corners=True) in float64.

feat bound, first order on magnitudes (u = 2^-24).  Let S = sum_p W[s, p] |t[p]| / count and, per segment row,
n = (the most terms summed into one W cell: four per pixel, of which i0 == i1 duplicates) + (the number of non-zero
W[s, p]).
  W      every term (1 - wy)(1 - wx) etc. is formed with at most three roundings (1 - wy, 1 - wx, the product; the tiled
         kernel's run sums of (1 - wx) are part of the summation tree) and is non-negative, so the fp32 sum of a cell's
         terms, in any order and through any mix of register, shared and global atomics, is within
         (n_cell - 1 + 3) u of the exact one.  Carried through the tokens: (n_cell + 2) u S.
  GEMM   the fp32 FMA chain over a split's tokens and the ksplit partial sums (vector atomics) form a summation tree
         of depth <= nnz over the non-zero W, each term a product with one rounding: nnz u S.
  div    one rounding: u |ref|.  The count is an integer < 2^24, exact in fp32.
  =>     |got - ref| <= (C n + 3) u S + u |ref|
With C = 1 this is the worst case.  C is measured: assert_within records max (|err| - 3 u S - u |ref|) / (n u S), and
C is set at about 4x the largest value seen on an H100 (DESIGN.md §4).  The tokens share a common offset four times
their spread, so that the bound, which scales with |t|, has to resolve a difference 1 / count of the spread: a relative
tolerance on |ref| of the kind the end-to-end tests use would accept a pixel counted against the wrong token.

Exact outputs.  centers: the coordinate sums and counts are integers in uint64 and the quotient is formed in double,
so centers must be bit-identical to the float64 quotient rounded to fp32.  edges: the set of directed (left / top id,
right / bottom id) pairs of 4-neighbour pixels with different ids, both in [0, smax), in the order torch.unique gives
left + right * (max + 1); rows past n_edges untouched, n_edges = -(true count) when max_edges overflows, with the first
max_edges rows written.  relabel: exact, counts exact.  Ids outside [0, smax) (or [0, num_labels)) contribute nothing,
make no edge and are left as they are by relabel: that is the contract the tests pin.

pool_supervision: the pixel signal is the nanmean over the mask's channels (at most C - 1 adds and one division,
(C + 1) u), all-NaN pixels are skipped, and the per-segment mean is a sum of cnt such values through shared and global
atomics and one division.  Worst case, no measured constant: |got - ref| <= (cnt + C + 2) u sum|signal| / cnt.  The
labels are chosen so that every segment mean is either exactly 0 or farther than that bound from 0, so valid is exact.

The path rules of segment_accumulate / segment_pool are restated in Python (`paths`) and test_cases_cover_every_path
asserts that the case list reaches each of them.  The checkers are tested on the CPU (no gpu mark): each negative
control corrupts a correct result in one place and must be rejected.
"""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_kernel_edges_gpu as edges  # noqa: E402
from test_kernel_edges_gpu import assert_within  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

U = 2.0 ** -24
F32 = np.float32
# accumulator constant of the feat bound: the worst (|err| - 3 u S - u |ref|) / (n u S) measured on one H100 80GB HBM3
# (700 W) over this module's cases was 0.050 (tiled accumulate, scalar pool), and C is set at 4x that (DESIGN.md §4);
# 1 is the worst case
C_SEG = 0.2
K_FIX = 3
TILE_H, TILE_W, PRIV_MAX_SEG, PRIV_SMEM = 32, 64, 128, 160 * 1024   # segment_kernels.cu
EDGE_SENTINEL = -7777
GUARD = 64


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    tags = {k: v for k, v in edges._WORST.items() if k.startswith("seg_")}
    if tags:
        print("\nsegment reductions, worst error / bound (and the C each check needs):")
        for tag in sorted(tags):
            r, a = tags[tag]
            print(f"  {tag:40s} {r:.4f}" + (f"   C needed {a:.4f}" if a is not None else ""))


# ------------------------------------------------------------------------------------------------ path rules
def f32_scale(g, h):
    """api.cu: (g - 1) / (h - 1) in fp32; 0 when h == 1."""
    return F32(F32(g - 1) / F32(h - 1)) if h > 1 else F32(0)


def paths(B, h, w, smax, grid, D):
    """segment_accumulate / segment_pool's choice for a call: accumulate kernel, pool kernel, ksplit, column blocks."""
    gh, gw = grid if grid is not None else (1, 1)
    sy, sx = f32_scale(gh, h), f32_scale(gw, h)
    win_h = int(F32(TILE_H - 1) * sy) + 3
    win_w = int(F32(TILE_W - 1) * sx) + 3
    words = (smax + 31) // 32
    smem = 4 * smax * win_h * win_w + 4 * smax * 3 + 4 * smax * words
    if smax <= PRIV_MAX_SEG and smem <= PRIV_SMEM:
        acc = "tiled"
    else:
        acc = "untiled_smax" if smax > PRIV_MAX_SEG else "untiled_smem"
    if grid is None:
        return {"acc": acc, "pool": None, "ksplit": 0, "col_blocks": 0, "partial": False}
    P = gh * gw
    if D % 4 == 0:
        v4 = D // 4
        cb = (v4 + 95) // 96
        return {"acc": acc, "pool": "vector", "ksplit": (P + 127) // 128, "col_blocks": cb, "partial": v4 % 96 != 0}
    return {"acc": acc, "pool": "scalar", "ksplit": (P + 447) // 448, "col_blocks": (D + 63) // 64,
            "partial": D % 64 != 0}


# ------------------------------------------------------------------------------------------------ maps
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def map_grid(h, w, cell, seed=0):
    y = torch.arange(h)[:, None] // cell
    x = torch.arange(w)[None, :] // cell
    return y * ((w + cell - 1) // cell) + x


def map_scattered(h, w, smax, seed, frac=0.3):
    g = _gen(seed)
    m = torch.full((h, w), -1, dtype=torch.int64)
    on = torch.rand(h, w, generator=g) < frac
    m[on] = torch.randint(0, smax, (int(on.sum()),), generator=g)
    return m


def map_stego(h, w, k, seed):
    """Non-connected clusters: coarse random labels, nearest-upsampled, with 25 % of the pixels re-drawn (runs break)."""
    g = _gen(seed)
    lo = torch.randint(0, k, ((h + 3) // 4, (w + 3) // 4), generator=g)
    m = lo.repeat_interleave(4, 0).repeat_interleave(4, 1)[:h, :w].clone()
    noise = torch.rand(h, w, generator=g) < 0.25
    m[noise] = torch.randint(0, k, (int(noise.sum()),), generator=g)
    return m


def map_slic(h, w, k, seed):
    """Blobs: nearest of k random seeds (a Voronoi map)."""
    g = _gen(seed)
    pts = torch.rand(k, 2, generator=g) * torch.tensor([h, w])
    yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    d = (yy[..., None] - pts[:, 0]) ** 2 + (xx[..., None] - pts[:, 1]) ** 2
    return d.argmin(-1)


def map_checker(h, w, smax, seed):
    """Pixel checkerboard: black pixels take ids in [0, smax/2), white ones in [smax/2, smax) -> the densest edge set."""
    g = _gen(seed)
    half = max(smax // 2, 1)
    m = torch.randint(0, half, (h, w), generator=g)
    par = (torch.arange(h)[:, None] + torch.arange(w)[None, :]) % 2
    return m + par * half


def make_map(kind, h, w, smax, seed):
    if kind == "grid":
        cell = {196: 32, 784: 16, 1024: 14}[smax]
        return map_grid(h, w, cell)
    if kind == "scattered":
        return map_scattered(h, w, smax, seed)
    if kind == "stego":
        return map_stego(h, w, smax, seed)
    if kind == "slic":
        return map_slic(h, w, smax, seed)
    if kind == "vstripes":
        return (torch.arange(w)[None, :] % smax).expand(h, w).clone()
    if kind == "hstripes":
        return (torch.arange(h)[:, None] % smax).expand(h, w).clone()
    if kind == "one":
        return torch.zeros(h, w, dtype=torch.int64)
    if kind == "checker":
        return map_checker(h, w, smax, seed)
    raise ValueError(kind)


def add_out_of_range(m, smax, seed, frac=0.03):
    """Sprinkle ids the kernels must ignore: negative ones and ones >= smax."""
    g = _gen(seed + 1000)
    bad = torch.tensor([-1, -5, smax, smax + 3, 1 << 40])
    on = torch.rand(m.shape, generator=g) < frac
    m = m.clone()
    m[on] = bad[torch.randint(0, len(bad), (int(on.sum()),), generator=g)]
    return m


def batch_map(kind, B, h, w, smax, seed, oob=False):
    frames = []
    for b in range(B):
        m = make_map(kind, h, w, smax, seed + 17 * b)
        frames.append(add_out_of_range(m, smax, seed + 17 * b) if oob else m)
    return torch.stack(frames).contiguous()


def make_tokens(B, P, D, seed, device):
    """Tokens with a common offset four times their spread."""
    g = torch.Generator(device=device).manual_seed(seed)
    off = 4.0 * torch.randn(D, device=device, generator=g).sign()
    return (off + torch.randn(B, P, D, device=device, generator=g)).contiguous()


# ------------------------------------------------------------------------------------------------ references
def coord_tables(n, g, h, device):
    """ac_true_coord for destinations 0..n-1 with the scale (g - 1) / (h - 1), in fp32 -> i0, i1, w (float64)."""
    s = np.arange(n, dtype=F32) * f32_scale(g, h)
    i0 = np.minimum(s.astype(np.int64), g - 1)
    i1 = np.minimum(i0 + 1, g - 1)
    w = (s - i0.astype(F32)).astype(F32)
    return [torch.from_numpy(a).to(device) for a in (i0, i1, w.astype(np.float64))]


def pixel_tables(h, w, gh, gw, device):
    """Per-pixel (y0, y1, wy, x0, x1, wx), each [h, w] (cloned: the negative controls edit single pixels)."""
    y0, y1, wy = coord_tables(h, gh, h, device)
    x0, x1, wx = coord_tables(w, gw, h, device)
    col = lambda t: t[:, None].expand(h, w).clone()  # noqa: E731
    row = lambda t: t[None, :].expand(h, w).clone()  # noqa: E731
    return {"y0": col(y0), "y1": col(y1), "wy": col(wy), "x0": row(x0), "x1": row(x1), "wx": row(wx)}


def weights_ref(seg, smax, gh, gw, tables=None):
    """seg [B, h, w] -> W [B, smax, P] float64, terms per cell [B, smax, P], count [B, smax] float64."""
    B, h, w = seg.shape
    dev = seg.device
    P = gh * gw
    t = tables if tables is not None else pixel_tables(h, w, gh, gw, dev)
    ok = (seg >= 0) & (seg < smax)
    row = (torch.arange(B, device=dev)[:, None, None] * smax + seg.clamp(0, smax - 1))[ok]
    W = torch.zeros(B * smax * P, dtype=torch.float64, device=dev)
    n = torch.zeros(B * smax * P, dtype=torch.float64, device=dev)
    for yk, xk, wgt in (("y0", "x0", (1 - t["wy"]) * (1 - t["wx"])), ("y0", "x1", (1 - t["wy"]) * t["wx"]),
                        ("y1", "x0", t["wy"] * (1 - t["wx"])), ("y1", "x1", t["wy"] * t["wx"])):
        cell = (t[yk] * gw + t[xk]).expand(B, h, w)[ok]
        W.index_add_(0, row * P + cell, wgt.expand(B, h, w)[ok])
        n.index_add_(0, row * P + cell, torch.ones_like(cell, dtype=torch.float64))
    cnt = torch.zeros(B * smax, dtype=torch.float64, device=dev).index_add_(
        0, row, torch.ones_like(row, dtype=torch.float64))
    return W.view(B, smax, P), n.view(B, smax, P), cnt.view(B, smax)


def feat_ref(seg, smax, tokens, grid, tables=None):
    """-> ref [B, smax, D] (NaN rows for empty segments), S = W|t| / count, n per row, count."""
    gh, gw = grid
    W, npix, cnt = weights_ref(seg, smax, gh, gw, tables)
    t64 = tokens.double()
    ref = (W @ t64) / cnt[..., None]
    S = (W @ t64.abs()) / cnt[..., None]
    n = npix.amax(-1) + (W != 0).sum(-1).double()
    return ref, S, n, cnt


def centers_ref(seg, smax):
    """-> centers [B, smax, 2] fp32: the float64 quotient of the exact integer sums, rounded once; NaN when empty."""
    B, h, w = seg.shape
    dev = seg.device
    ok = (seg >= 0) & (seg < smax)
    row = (torch.arange(B, device=dev)[:, None, None] * smax + seg.clamp(0, smax - 1))[ok]
    xs = torch.arange(w, device=dev, dtype=torch.float64)[None, None, :].expand(B, h, w)[ok]
    ys = torch.arange(h, device=dev, dtype=torch.float64)[None, :, None].expand(B, h, w)[ok]
    z = lambda: torch.zeros(B * smax, dtype=torch.float64, device=dev)  # noqa: E731
    cnt = z().index_add_(0, row, torch.ones_like(xs))        # integer sums < 2^53: exact in float64
    sx, sy = z().index_add_(0, row, xs), z().index_add_(0, row, ys)
    return torch.stack([sx / cnt, sy / cnt], -1).float().view(B, smax, 2)


def edges_ref(frame, smax):
    """One frame [h, w] -> [n, 2] int64 (left / top id, right / bottom id), ordered by left + right * smax."""
    hl, hr = frame[:, :-1].reshape(-1), frame[:, 1:].reshape(-1)
    vt, vb = frame[:-1, :].reshape(-1), frame[1:, :].reshape(-1)
    left, right = torch.cat([hl, vt]), torch.cat([hr, vb])
    keep = (left != right) & (left >= 0) & (left < smax) & (right >= 0) & (right < smax)
    key = torch.unique(left[keep] + right[keep] * smax)
    return torch.stack([key % smax, key // smax], 1)


def relabel_ref(seg, num_labels):
    """Per frame: the labels in [0, num_labels) present, in sorted order, become 0..S-1; other values stay."""
    out = seg.clone()
    counts = []
    for b in range(seg.shape[0]):
        f = seg[b]
        ok = (f >= 0) & (f < num_labels)
        uniq = torch.unique(f[ok])
        out[b][ok] = torch.searchsorted(uniq, f[ok])
        counts.append(len(uniq))
    return out, torch.tensor(counts, dtype=torch.int32)


def supervision_ref(seg, mask, smax, nan_channels_count=False):
    """float64 update_supervision_signal restricted to ids in [0, smax) -> mean [B, smax], valid, bound.
    nan_channels_count: the negative control's wrong signal, which divides by every channel."""
    B, C, h, w = mask.shape
    dev = seg.device
    m64 = mask.double()
    if nan_channels_count:
        has = (~torch.isnan(m64)).any(1)
        sig = torch.where(has, m64.nan_to_num(0).sum(1) / C, torch.full_like(m64[:, 0], float("nan")))
    else:
        sig = m64.nanmean(1)
    ok = ~torch.isnan(sig) & (seg >= 0) & (seg < smax)
    row = (torch.arange(B, device=dev)[:, None, None] * smax + seg.clamp(0, smax - 1))[ok]
    z = lambda: torch.zeros(B * smax, dtype=torch.float64, device=dev)  # noqa: E731
    cnt = z().index_add_(0, row, torch.ones_like(sig[ok]))
    tot = z().index_add_(0, row, sig[ok])
    mag = z().index_add_(0, row, sig[ok].abs())
    mean = (tot / cnt).nan_to_num(0)
    bound = ((cnt + C + 2) * U * mag / cnt.clamp_min(1))
    return mean.view(B, smax), (mean > 0).view(B, smax), bound.view(B, smax), cnt.view(B, smax)


# ------------------------------------------------------------------------------------------------ checkers
def check_feat(got, ref, S, n, cnt, tag, c=C_SEG):
    empty = cnt == 0
    if bool(empty.any()):
        bad = ~torch.isnan(got[empty])
        assert not bool(bad.any()), f"{tag}: {int(bad.sum())} elements of empty segments are not NaN"
    live = ~empty
    if not bool(live.any()):
        return
    g, r, s = got[live], ref[live], S[live]
    nn = n[live][:, None].expand_as(s)
    acc = nn * U * s
    rest = K_FIX * U * s + U * r.abs()
    assert_within(g, r, c * acc + rest, tag, acc, rest)


def _f32_bits(t):
    return t.contiguous().view(torch.int32)


def check_centers(got, ref, tag):
    nan_ref, nan_got = torch.isnan(ref), torch.isnan(got)
    assert torch.equal(nan_ref, nan_got), f"{tag}: NaN pattern differs ({int((nan_ref != nan_got).sum())} elements)"
    diff = (_f32_bits(got) != _f32_bits(ref)) & ~nan_ref
    if bool(diff.any()):
        idx = tuple(int(i) for i in diff.nonzero()[0])
        raise AssertionError(f"{tag}: {int(diff.sum())} centers not bit-identical; first at {idx}: got "
                             f"{got[idx].item():.9g} ref {ref[idx].item():.9g}")


def check_edges(buf, n_edges, seg, smax, max_edges, tag):
    """buf: the flat int64 edge buffer (B * max_edges * 2 + GUARD) the kernel wrote into, pre-filled with the sentinel."""
    B = seg.shape[0]
    body = buf[: B * max_edges * 2].view(B, max_edges, 2)
    for b in range(B):
        ref = edges_ref(seg[b], smax)
        ne = ref.shape[0]
        if ne <= max_edges:
            assert int(n_edges[b]) == ne, f"{tag}: frame {b}: n_edges {int(n_edges[b])}, reference {ne}"
            assert torch.equal(body[b, :ne], ref), f"{tag}: frame {b}: edge rows differ from the reference"
            assert bool((body[b, ne:] == EDGE_SENTINEL).all()), f"{tag}: frame {b}: rows past n_edges were written"
        else:
            assert int(n_edges[b]) == -ne, f"{tag}: frame {b}: overflow flag {int(n_edges[b])}, expected {-ne}"
            assert torch.equal(body[b], ref[:max_edges]), f"{tag}: frame {b}: first max_edges rows differ"
    assert bool((buf[B * max_edges * 2:] == EDGE_SENTINEL).all()), f"{tag}: the guard past the last frame was written"


def check_supervision(y, valid, ref, ref_valid, bound, cnt, tag):
    assert torch.equal((y[cnt == 0]).double(), ref[cnt == 0]), f"{tag}: segments without labelled pixels must be 0"
    assert_within(y, ref, bound + U * ref.abs(), tag)
    # valid is decided by the sign: every mean is exactly 0 or farther than its bound from 0, so it must be exact
    assert bool(((ref == 0) | (ref.abs() > bound + U * ref.abs())).all()), f"{tag}: a segment mean lies within its bound of 0"
    assert torch.equal(valid, ref_valid), f"{tag}: valid differs at {int((valid != ref_valid).sum())} segments"


# ------------------------------------------------------------------------------------------------ raw kernel call
def segment_reduce_raw(seg, smax, tokens=None, grid=None, centers=True, max_edges=None, seed=0):
    """wvn_segment_reduce with sentinel-filled outputs that end in a guard, and a workspace full of garbage."""
    from wild_visual_navigation_b200._C import check, lib, ptr, stream

    B, h, w = seg.shape
    dev = seg.device
    gh, gw = grid if grid is not None else (1, 1)
    D = tokens.shape[-1] if tokens is not None else 0
    ws = torch.randint(0, 256, (lib().wvn_segment_workspace_bytes(B, smax, gh, gw),), dtype=torch.uint8, device=dev,
                       generator=torch.Generator(device=dev).manual_seed(seed))
    feat_buf = torch.full((B * smax * D + GUARD,), 1234.5, device=dev) if tokens is not None else None
    cen_buf = torch.full((B * smax * 2 + GUARD,), 1234.5, device=dev) if centers else None
    edge_buf = torch.full((B * max_edges * 2 + GUARD,), EDGE_SENTINEL, dtype=torch.int64, device=dev) \
        if max_edges is not None else None
    n_edges = torch.full((B,), 99999, dtype=torch.int32, device=dev) if max_edges is not None else None
    check(lib().wvn_segment_reduce(ptr(seg), B, h, w, smax, ptr(tokens), gh, gw, D, ptr(feat_buf), ptr(cen_buf),
                                   ptr(edge_buf), ptr(n_edges), max_edges or 0, ptr(ws), stream()))
    torch.cuda.synchronize()
    out = {"edge_buf": edge_buf, "n_edges": n_edges}
    if feat_buf is not None:
        assert bool((feat_buf[B * smax * D:] == 1234.5).all()), "feat guard written"
        out["feat"] = feat_buf[: B * smax * D].view(B, smax, D)
    if cen_buf is not None:
        assert bool((cen_buf[B * smax * 2:] == 1234.5).all()), "centers guard written"
        out["centers"] = cen_buf[: B * smax * 2].view(B, smax, 2)
    return out


# ------------------------------------------------------------------------------------------------ cases
# name -> (B, h, w, grid or None, D, smax, map kind, out-of-range ids sprinkled)
CASES = {
    "dino8_448_slic100": (3, 448, 448, (56, 56), 384, 100, "slic", True),
    "dino8_448_grid196_d768": (1, 448, 448, (56, 56), 768, 196, "grid", False),
    "vits14_448_grid784_d1024": (1, 448, 448, (32, 32), 1024, 784, "grid", True),
    "dino8_448_grid1024": (1, 448, 448, (56, 56), 384, 1024, "grid", False),
    "dinov2_518_stego20": (3, 518, 518, (37, 37), 384, 20, "stego", True),
    "p14_224_stego128_d90": (3, 224, 224, (16, 16), 90, 128, "stego", False),
    "p8_224_slic129_d33": (3, 224, 224, (28, 28), 33, 129, "slic", True),
    "one_token_224_d4": (3, 224, 224, (1, 1), 4, 1, "one", False),
    "full_res_64_scattered128_d16": (3, 64, 64, (64, 64), 16, 128, "scattered", False),
    "full_res_45x37_stego20_d33": (1, 45, 37, (45, 45), 33, 20, "stego", True),
    "nonsquare_450x333_scattered1024": (2, 450, 333, (56, 56), 384, 1024, "scattered", False),
    "nonsquare_450x333_stego20_d90": (3, 450, 333, (56, 56), 90, 20, "stego", True),
    "vstripes_224_128": (1, 224, 224, (28, 28), 384, 128, "vstripes", False),
    "hstripes_224x200_129_d4": (1, 224, 200, (28, 28), 4, 129, "hstripes", False),
    "checker_130x97_100": (1, 130, 97, (16, 16), 384, 100, "checker", False),
    "one_segment_448_smax1": (1, 448, 448, (56, 56), 384, 1, "one", False),
    "bench_b32_448_stego20": (32, 448, 448, (56, 56), 384, 20, "stego", False),
    # centers and edges only (no tokens): the ResNet path, including maps wider than tall
    "edges_only_333x450_slic100": (2, 333, 450, None, 0, 100, "slic", True),
    "edges_only_320x448_grid784": (1, 320, 448, None, 0, 784, "grid", False),
    "edges_only_97x130_checker128": (3, 97, 130, None, 0, 128, "checker", True),
}


def test_cases_cover_every_path():
    """The case list reaches every accumulate and pooling path of the restated host rules, at the shapes the
    pipeline uses."""
    got = {name: paths(B, h, w, smax, grid, D) for name, (B, h, w, grid, D, smax, _, _) in CASES.items()}
    accs = {p["acc"] for p in got.values()}
    assert accs == {"tiled", "untiled_smax", "untiled_smem"}, accs
    pools = {(p["pool"], p["col_blocks"], p["partial"]) for p in got.values() if p["pool"]}
    assert ("vector", 1, False) in pools and ("vector", 2, False) in pools       # D = 384, 768
    assert ("vector", 3, True) in pools and ("vector", 1, True) in pools         # D = 1024, 4 / 16
    assert any(p == "scalar" for p, _, _ in pools)
    for kind in ("vector", "scalar"):   # ksplit > 1 on frames other than 0
        assert any(p["pool"] == kind and p["ksplit"] > 1 and CASES[n][0] > 1 for n, p in got.items()), kind
    assert any(p["pool"] is None and p["acc"] == "tiled" for p in got.values())
    assert any(p["pool"] is None and p["acc"] != "tiled" for p in got.values())
    Ds = {c[4] for c in CASES.values()}
    assert {384, 768, 1024, 4, 90, 33} <= Ds
    assert {1, 20, 100, 128, 129, 196, 784, 1024} <= {c[5] for c in CASES.values()}
    assert {1, 3, 32} <= {c[0] for c in CASES.values()}
    grids = {(c[3][0], c[1]) for c in CASES.values() if c[3]}
    assert {(56, 448), (32, 448), (37, 518), (16, 224), (28, 224), (1, 224), (64, 64), (45, 45)} <= grids
    assert any(c[2] < c[1] and c[1] % 8 and c[2] % 8 and c[3] for c in CASES.values())   # w < h, neither % 8
    assert any(c[2] > c[1] and c[3] is None for c in CASES.values())                     # w > h, no tokens
    assert {"grid", "scattered", "stego", "slic", "vstripes", "hstripes", "one", "checker"} <= {c[6] for c in CASES.values()}
    bench = CASES["bench_b32_448_stego20"]
    assert bench[:6] == (32, 448, 448, (56, 56), 384, 20)
    # grid = image forces the untiled fallback through shared memory at smax = 128
    assert got["full_res_64_scattered128_d16"]["acc"] == "untiled_smem"


# ------------------------------------------------------------------------------------------------ CPU: the reference
@pytest.mark.parametrize("h,w,grid", [(37, 37, (5, 5)), (41, 23, (6, 6)), (12, 12, (12, 12)), (20, 13, (1, 1)),
                                      (33, 30, (4, 7))])
def test_reference_matches_product_definition(h, w, grid):
    """feat_ref (fp32 source coordinates, then float64) against oracle/wvn_path.sparsify_features on the float64
    F.interpolate(align_corners=True) map; centers, edges, relabel and supervision against their oracle definitions."""
    from oracle import wvn_path

    gh, gw = grid
    D, S = 6, 9
    seg = map_slic(h, w, S, seed=h * w)
    seg = torch.unique(seg, return_inverse=True)[1]            # ids 0..S'-1, all present
    S = int(seg.max()) + 1
    tok = make_tokens(1, gh * gw, D, seed=5, device="cpu").double()
    dense = F.interpolate(tok.reshape(1, gh, gw, D).permute(0, 3, 1, 2), (h, h), mode="bilinear", align_corners=True)
    want = wvn_path.sparsify_features(dense, seg)
    ref, _, _, cnt = feat_ref(seg[None], S, tok, grid)
    assert bool((cnt > 0).all())
    # the only difference is the fp32 source coordinate: ~u g per weight
    assert (ref[0] - want).abs().max().item() <= 1e-6 * max(gh, gw) * tok.abs().max().item()
    c = centers_ref(seg[None], S)[0]
    assert (c - wvn_path.centers(seg[None, None])).abs().max().item() <= 1e-5 * max(h, w)
    assert torch.equal(edges_ref(seg, S), wvn_path.adjacency_list(seg[None, None]))
    raw = seg * 3 + 2
    out, counts = relabel_ref(raw[None], 3 * S + 2)
    assert torch.equal(out[0], wvn_path.relabel(raw)) and int(counts[0]) == S
    mask = torch.rand(3, h, w, generator=_gen(1))
    mask[torch.rand(3, h, w, generator=_gen(2)) < 0.4] = float("nan")
    mean, valid, _, _ = supervision_ref(seg[None], mask[None], S)
    want_m, want_v = wvn_path.update_supervision_signal(mask.double(), seg)
    assert (mean[0] - want_m).abs().max().item() <= 1e-12 and torch.equal(valid[0], want_v)


# ------------------------------------------------------------------------------------------------ CPU: negative controls
def _small_case():
    h, w, grid, D, smax = 40, 30, (6, 6), 8, 12
    seg = add_out_of_range(map_slic(h, w, smax, seed=3), smax, seed=3)[None]
    tok = make_tokens(1, grid[0] * grid[1], D, seed=7, device="cpu")
    ref, S, n, cnt = feat_ref(seg, smax, tok, grid)
    return seg, smax, tok, grid, ref, S, n, cnt


def test_checker_accepts_correct_feat_and_centers():
    seg, smax, tok, grid, ref, S, n, cnt = _small_case()
    check_feat(ref.float(), ref, S, n, cnt, "neg_ok")
    c = centers_ref(seg, smax)
    check_centers(c.clone(), c, "neg_ok")


def test_checker_rejects_pixel_weighted_by_neighbouring_token_column():
    seg, smax, tok, grid, ref, S, n, cnt = _small_case()
    t = pixel_tables(seg.shape[1], seg.shape[2], grid[0], grid[1], "cpu")
    y, x = 17, 11      # an interior pixel: its right neighbour column of tokens exists
    assert int(seg[0, y, x]) in range(smax) and int(t["x1"][y, x]) + 1 < grid[1]
    t["x0"][y, x] += 1
    t["x1"][y, x] += 1
    bad, _, _, _ = feat_ref(seg, smax, tok, grid, tables=t)
    with pytest.raises(AssertionError):
        check_feat(bad.float(), ref, S, n, cnt, "neg_column")


def test_checker_rejects_row_missing_one_pixel():
    seg, smax, tok, grid, ref, S, n, cnt = _small_case()
    s2 = seg.clone()
    y, x = 5, 7
    assert int(s2[0, y, x]) in range(smax)
    s2[0, y, x] = -1
    bad, _, _, _ = feat_ref(s2, smax, tok, grid)
    with pytest.raises(AssertionError):
        check_feat(bad.float(), ref, S, n, cnt, "neg_missing")


def test_checker_rejects_center_one_ulp_off():
    seg, smax, *_ = _small_case()
    c = centers_ref(seg, smax)
    bad = c.clone()
    k = int(seg[0, 20, 15])
    bad[0, k, 1] = torch.nextafter(bad[0, k, 1], torch.tensor(float("inf")))
    with pytest.raises(AssertionError):
        check_centers(bad, c, "neg_ulp")


def _edge_buffer(seg, smax, max_edges, edit=None):
    B = seg.shape[0]
    buf = torch.full((B * max_edges * 2 + GUARD,), EDGE_SENTINEL, dtype=torch.int64)
    n = torch.zeros(B, dtype=torch.int32)
    for b in range(B):
        ref = edges_ref(seg[b], smax)
        rows = ref if edit is None else edit(ref)
        k = min(rows.shape[0], max_edges)
        buf[b * max_edges * 2: b * max_edges * 2 + 2 * k] = rows[:k].reshape(-1)
        n[b] = rows.shape[0] if rows.shape[0] <= max_edges else -rows.shape[0]
    return buf, n


def test_edge_checker_accepts_correct_and_overflow():
    seg, smax, *_ = _small_case()
    ne = edges_ref(seg[0], smax).shape[0]
    for me in (ne + 5, ne, ne - 1, 3):
        buf, n = _edge_buffer(seg, smax, me)
        check_edges(buf, n, seg, smax, me, "neg_edges_ok")


def test_edge_checker_rejects_swapped_and_extra_edges():
    seg, smax, *_ = _small_case()
    me = smax * smax
    swap = lambda r: torch.cat([r[:3], r[4:5], r[3:4], r[5:]])  # noqa: E731
    extra = lambda r: torch.cat([r, torch.tensor([[0, smax - 1]])])  # noqa: E731
    for edit in (swap, extra):
        buf, n = _edge_buffer(seg, smax, me, edit)
        with pytest.raises(AssertionError):
            check_edges(buf, n, seg, smax, me, "neg_edges")
    # one extra row written past n_edges, with the count left right
    buf, n = _edge_buffer(seg, smax, me)
    ne = int(n[0])
    buf[2 * ne: 2 * ne + 2] = torch.tensor([0, 1])
    with pytest.raises(AssertionError):
        check_edges(buf, n, seg, smax, me, "neg_edges_past")


def _supervision_case(C, smax, seed, device="cpu"):
    """Labels in [0.05, 1] with NaN channels and all-NaN pixels; one segment labelled 0 everywhere, one unlabelled."""
    seg = torch.stack([add_out_of_range(map_slic(48, 40, smax, seed + b), smax, seed + b) for b in range(2)])
    g = _gen(seed)
    mask = 0.05 + 0.95 * torch.rand(2, C, 48, 40, generator=g)
    mask[torch.rand(mask.shape, generator=g) < 0.3] = float("nan")
    mask[:, :, torch.rand(48, 40, generator=g) < 0.1] = float("nan")
    mask[0][:, seg[0] == 1] = 0.0
    mask[1][:, seg[1] == 2] = float("nan")
    return seg.to(device), mask.to(device)


def test_supervision_checker_rejects_mean_counting_a_nan_channel():
    seg, mask = _supervision_case(3, 12, seed=4)
    ref, rv, bound, cnt = supervision_ref(seg, mask, 12)
    check_supervision(ref.float(), rv, ref, rv, bound, cnt, "neg_sup_ok")
    bad, _, _, _ = supervision_ref(seg, mask, 12, nan_channels_count=True)
    with pytest.raises(AssertionError):
        check_supervision(bad.float(), rv, ref, rv, bound, cnt, "neg_sup")


# ------------------------------------------------------------------------------------------------ GPU
def _run_case(name, seg, smax, grid, D, seed):
    B, h, w = seg.shape
    tok = make_tokens(B, grid[0] * grid[1], D, seed, "cuda") if grid is not None else None
    me = smax * smax if smax <= 256 else min(smax * smax, 64 * smax)
    r = segment_reduce_raw(seg, smax, tok, grid, centers=True, max_edges=me, seed=seed)
    if tok is not None:
        ref, S, n, cnt = feat_ref(seg, smax, tok, grid)
        check_feat(r["feat"], ref, S, n, cnt, f"seg_feat_{paths(B, h, w, smax, grid, D)['acc']}_"
                                              f"{paths(B, h, w, smax, grid, D)['pool']}")
    check_centers(r["centers"], centers_ref(seg, smax), f"{name} centers")
    check_edges(r["edge_buf"], r["n_edges"], seg, smax, me, f"{name} edges")
    return r, tok


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_segment_reduce_vs_float64(name):
    B, h, w, grid, D, smax, kind, oob = CASES[name]
    seg = batch_map(kind, B, h, w, smax, seed=len(name), oob=oob).cuda()
    _run_case(name, seg, smax, grid, D, seed=len(name))


@pytest.mark.gpu
def test_public_wrapper_matches_raw_call():
    """ops.segment_reduce (its own workspace and default max_edges): feat within the bound, centers and edges
    bit-identical to the raw call (feat's float atomics make it run-to-run different in the last bits)."""
    from wild_visual_navigation_b200 import ops

    seg = batch_map("stego", 2, 224, 224, 20, seed=9, oob=True).cuda()
    tok = make_tokens(2, 784, 384, 9, "cuda")
    a = ops.segment_reduce(seg, 20, tokens=tok, grid=(28, 28))
    b = segment_reduce_raw(seg, 20, tok, (28, 28), max_edges=a["max_edges"])
    ref, S, n, cnt = feat_ref(seg, 20, tok, (28, 28))
    check_feat(a["feat"], ref, S, n, cnt, "seg_feat_tiled_vector")
    assert torch.equal(_f32_bits(a["centers"]), _f32_bits(b["centers"]))
    assert torch.equal(a["n_edges"], b["n_edges"])
    for f in range(2):
        ne = int(a["n_edges"][f])
        assert torch.equal(a["edges"][f, :ne], b["edge_buf"][: 2 * 20 * 20 * 2].view(2, -1, 2)[f, :ne])


@pytest.mark.gpu
def test_tiled_and_untiled_accumulate_agree():
    """The same map at smax = 128 (tiled kernel) and 129 (untiled, one extra empty segment): centers and edges
    bit-identical, feat within the bound in both, row 128 NaN."""
    B, h, w, grid, D = 2, 448, 448, (56, 56), 384
    seg = torch.stack([map_slic(h, w, 128, seed=b) for b in range(B)])
    g = _gen(77)
    on = torch.rand(seg.shape, generator=g) < 0.02
    seg[on] = torch.tensor([-1, 129, 4000])[torch.randint(0, 3, (int(on.sum()),), generator=g)]
    seg = seg.cuda()
    assert paths(B, h, w, 128, grid, D)["acc"] == "tiled" and paths(B, h, w, 129, grid, D)["acc"] == "untiled_smax"
    r128, tok = _run_case("tiled128", seg, 128, grid, D, seed=1)
    r129 = segment_reduce_raw(seg, 129, tok, grid, max_edges=128 * 128)
    ref, S, n, cnt = feat_ref(seg, 129, tok, grid)
    check_feat(r129["feat"], ref, S, n, cnt, "seg_feat_untiled_smax_vector")
    assert bool(torch.isnan(r129["feat"][:, 128]).all()) and bool(torch.isnan(r129["centers"][:, 128]).all())
    assert torch.equal(_f32_bits(r128["centers"]), _f32_bits(r129["centers"][:, :128]))
    assert torch.equal(r128["n_edges"], r129["n_edges"])
    for b in range(B):
        ne = int(r128["n_edges"][b])
        e128 = r128["edge_buf"][: B * 128 * 128 * 2].view(B, -1, 2)[b, :ne]
        e129 = r129["edge_buf"][: B * 128 * 128 * 2].view(B, -1, 2)[b, :ne]
        assert torch.equal(e128, e129)


@pytest.mark.gpu
@pytest.mark.parametrize("smax", [40, 300])
def test_out_of_range_ids_are_ignored(smax):
    """Ids < 0 and >= smax contribute nothing and make no edge, in the tiled (40) and untiled (300) kernels: the
    outputs equal those of the same map with every such id replaced by -1 (centers and edges bit for bit, feat within
    its bound: an ignored pixel ends a run of the tiled kernel, which changes the fp32 summation order)."""
    B, h, w, grid, D = 2, 200, 180, (25, 25), 64
    base = torch.stack([map_stego(h, w, smax, seed=b) for b in range(B)])
    noisy = add_out_of_range(base, smax, seed=5, frac=0.2)
    clean = torch.where((noisy >= 0) & (noisy < smax), noisy, torch.full_like(noisy, -1))
    tok = make_tokens(B, 625, D, 3, "cuda")
    a = segment_reduce_raw(noisy.cuda(), smax, tok, grid, max_edges=smax * smax)
    b = segment_reduce_raw(clean.cuda(), smax, tok, grid, max_edges=smax * smax)
    assert torch.equal(_f32_bits(a["centers"]), _f32_bits(b["centers"]))
    assert torch.equal(a["n_edges"], b["n_edges"]) and torch.equal(a["edge_buf"], b["edge_buf"])
    ref, S, n, cnt = feat_ref(clean.cuda(), smax, tok, grid)
    check_feat(a["feat"], ref, S, n, cnt, f"seg_feat_{paths(B, h, w, smax, grid, D)['acc']}_vector")
    check_edges(a["edge_buf"], a["n_edges"], noisy.cuda(), smax, smax * smax, "oob edges")


@pytest.mark.gpu
def test_adjacency_overflow_flag():
    """max_edges below, at and one under the true count: n_edges = -(true count) on overflow, the first max_edges rows
    equal the reference's first rows, nothing past them is written."""
    smax = 64
    seg = batch_map("checker", 3, 96, 130, smax, seed=2).cuda()
    true = [edges_ref(seg[b], smax).shape[0] for b in range(3)]
    assert min(true) > 1000
    for me in (100, min(true) - 1, max(true), max(true) + 1):
        r = segment_reduce_raw(seg, smax, None, None, centers=False, max_edges=me)
        check_edges(r["edge_buf"], r["n_edges"], seg, smax, me, f"overflow max_edges={me}")
        if me < min(true):
            assert bool((r["n_edges"] < 0).all())


# ------------------------------------------------------------------------------------------------ relabel
def _slice_geometry(pix):
    """relabel_compact: slices per frame and pixels per slice of label_presence_kernel."""
    slices = min((pix + 4095) // 4096, 32)
    per = (pix + slices - 1) // slices
    return slices, per


def _outside(f, num_labels, g):
    f = f.clone()
    on = torch.rand(f.shape, generator=g) < 0.01
    f[on] = torch.tensor([-1, -3, num_labels, num_labels + 9])[torch.randint(0, 4, (int(on.sum()),), generator=g)]
    return f


def _relabel_map(B, h, w, num_labels, seed):
    """Per frame a different set of base labels; labels whose only occurrence is the first or the last pixel of a
    label_presence slice; and values outside [0, num_labels) that must stay."""
    pix = h * w
    slices, per = _slice_geometry(pix)
    frames = []
    for b in range(B):
        g = _gen(seed + b)
        if num_labels == 1:
            f = torch.where(torch.rand(pix, generator=g) < 0.5, 0, -1)
            if b == 1:
                f = torch.full((pix,), -1, dtype=torch.int64)     # no label present at all
        else:
            half = num_labels // 2
            base = torch.randperm(half, generator=g)[: max(half // 3, 1)]
            f = base[torch.randint(0, len(base), (pix,), generator=g)]
            f = _outside(f, num_labels, g)
            special = half + torch.randperm(num_labels - half, generator=g)
            k = 0
            for j in range(slices):
                p0, p1 = j * per, min(pix, (j + 1) * per)
                for p in (p0, p1 - 1):
                    if k < len(special):
                        f[p] = special[k]
                        k += 1
        if num_labels == 1:
            f = _outside(f, num_labels, g)
        frames.append(f.view(h, w))
    return torch.stack(frames).contiguous()


RELABEL_CASES = [(3, 448, 448, 1024), (2, 333, 450, 128), (3, 50, 50, 27), (2, 1, 4097, 300), (3, 64, 64, 1),
                 (32, 224, 224, 20)]


def test_relabel_cases_cover_slices():
    sl = {_slice_geometry(h * w)[0] for _, h, w, _ in RELABEL_CASES}
    assert 1 in sl and 2 in sl and 32 in sl and any(1 < s < 32 for s in sl)
    assert {1, 1024} <= {c[3] for c in RELABEL_CASES} and any(c[0] > 1 for c in RELABEL_CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("B,h,w,num_labels", RELABEL_CASES)
def test_relabel_vs_reference(B, h, w, num_labels):
    from wild_visual_navigation_b200 import ops

    raw = _relabel_map(B, h, w, num_labels, seed=h + w)
    want, want_counts = relabel_ref(raw, num_labels)
    seg = raw.cuda()
    counts = ops.relabel(seg, num_labels)
    assert torch.equal(counts.cpu(), want_counts), (counts.cpu(), want_counts)
    assert torch.equal(seg.cpu(), want)


# ------------------------------------------------------------------------------------------------ supervision
SUP_CASES = [(2, 1, 448, 448, 20, "stego"), (3, 3, 333, 450, 100, "slic"), (1, 3, 224, 224, 1, "one"),
             (2, 3, 448, 448, 4096, "scattered"), (3, 2, 97, 130, 20, "checker"), (2, 1, 45, 37, 1, "scattered")]


@pytest.mark.gpu
@pytest.mark.parametrize("B,C,h,w,smax,kind", SUP_CASES)
def test_pool_supervision_vs_float64(B, C, h, w, smax, kind):
    from wild_visual_navigation_b200 import ops

    ids = 4000 if smax == 4096 else smax            # ids stop short of smax: entries past the map's max id stay 0
    seg = torch.stack([add_out_of_range(m, smax, seed=b) for b, m in enumerate(batch_map(kind, B, h, w, ids, smax + C))])
    g = _gen(smax * 7 + C)
    mask = 0.05 + 0.95 * torch.rand(B, C, h, w, generator=g)
    mask[torch.rand(mask.shape, generator=g) < 0.3] = float("nan")
    mask[:, :, torch.rand(h, w, generator=g) < 0.1] = float("nan")            # all-NaN pixels
    if ids > 2:
        mask[0][:, seg[0] == 1] = 0.0                                         # a segment labelled 0 throughout
        mask[B - 1][:, seg[B - 1] == 2] = float("nan")                        # a segment with no labelled pixel
    seg, mask = seg.cuda(), mask.cuda()
    y, valid = ops.pool_supervision(seg, mask if C > 1 else mask[:, 0], smax)
    ref, rv, bound, cnt = supervision_ref(seg, mask, smax)
    check_supervision(y, valid, ref, rv, bound, cnt, f"seg_sup_C{C}")
    if ids < smax:
        assert bool((y[:, ids:] == 0).all()) and not bool(valid[:, ids:].any())
