"""The per-image k-means (stego_kmeans.cu, ops.stego_kmeans) element by element against a float64 Lloyd run, at every
template and shared-memory plan the host can pick for what the public API accepts (n_image_clusters <= 64).

Input: K Gaussian blobs whose centres are far apart relative to their spread, written at HEAD_CODE_COL of a head-layout
buffer [B * npad, 256] whose CLS row, padding rows and other columns hold sentinel NaNs.  The row at each initial
position (2k + 1) P / (2K) belongs to blob k.  The float64 run (the oracle/stego_head.image_kmeans definition, restated
in `lloyd64` with its bounds) then has one unambiguous assignment per iteration, and the test asserts it: at every
iteration every row's gap between its best and second-best float64 score exceeds twice the largest bound on a kernel
score of that row (the score bound below plus the effect of the centroids' own bound).  So the kernel takes the same
assignment, and comparing centroids element by element is justified rather than assumed.

Centroid bound (u = 2^-24).  A centroid channel is the fp32 sum of its cluster's rows: a warp-private chain, then the
n_priv warp copies, then the team's T ranks in rank order, then one division by the (exact) count:
    |c - c64| <= (cnt + n_priv + T) u sum|x| / cnt + u |c64|          worst case, no measured constant
An empty cluster keeps its centroid bit for bit.
Score bound: the kernel's scores x.c - |c|^2 / 2 are held to float64 on its OWN returned centroids: four fp32 FMA
chains of CREG / 4 terms, two adds, |c|^2 as per-lane chains of <= 4 FMA and 5 shuffle adds, the subtraction:
    |s - s64| <= (CREG / 4 + 10) u (sum|x||c| + |c|^2 / 2)
Ties: duplicate rows at two initial positions j, j + 1 (j even, so both are scored in the same pass) give two identical
initial centroids; their scores are equal bit for bit, the lower index wins every tie of the first assignment, and
cluster j + 1 stays empty and keeps its initial row bit for bit.

The team size and shared-memory plan are restated in Python (`plan`, 132 SMs on the CPU and the device's count on the
GPU) and test_cases_cover_every_plan asserts that the case list reaches each template and plan.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_kernel_edges_gpu as edges  # noqa: E402
from test_kernel_edges_gpu import assert_owned_and_untouched, assert_within  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

U = 2.0 ** -24
LD, CODE_COL, LOGIT_COL = 256, 0, 128   # HEAD_OUT, HEAD_CODE_COL, HEAD_CLUSTER_COL of feature_extractor/weights.py
K_TEAM, K_MAX_TEAM, K_WARPS, K_MAX_K, BUDGET = 8, 32, 16, 64, 220 * 1024   # stego_kmeans.cu


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    tags = {k: v for k, v in edges._WORST.items() if k.startswith("km_")}
    if tags:
        print("\nk-means, worst error / bound:")
        for tag in sorted(tags):
            print(f"  {tag:40s} {tags[tag][0]:.4f}")


def team_size(B, sms):
    fit = sms // B
    return K_TEAM if fit < K_TEAM else min(fit, K_MAX_TEAM)


def plan(B, P, K, C, sms=132):
    """stego_kmeans's host choice: team size, CREG template, rows in shared memory, warp-private copies."""
    T = team_size(B, sms)
    CP = 96 if C <= 96 else 128
    per = (P + T - 1) // T
    fixed = 4 * (K * CP + K_MAX_K + K_WARPS * K_MAX_K)
    per_copy = 4 * K * CP
    rows = 4 * per * (C + 1)
    rows_smem = fixed + rows + 4 * per_copy <= BUDGET
    n_priv = min((BUDGET - fixed - (rows if rows_smem else 0)) // per_copy, K_WARPS)
    return {"team": T, "creg": CP, "rows_smem": rows_smem, "n_priv": n_priv, "ctas": B * T}


# name -> (B, P, K, C)
CASES = {
    "b1_p3136_k20_c90": (1, 3136, 20, 90),
    "b3_p1369_k7_c90": (3, 1369, 7, 90),
    "b5_p1024_k2_c33": (5, 1024, 2, 33),
    "b17_p784_k1_c90": (17, 784, 1, 90),
    "b17_p784_k20_c90": (17, 784, 20, 90),
    "b32_p3136_k20_c90": (32, 3136, 20, 90),
    "b32_p3136_k40_c90": (32, 3136, 40, 90),
    "b32_p3136_k64_c90": (32, 3136, 64, 90),
    "b3_p784_k64_c128": (3, 784, 64, 128),
    "b5_p1369_k7_c128": (5, 1369, 7, 128),
    "b1_p1024_k64_c33": (1, 1024, 64, 33),
}
TIE_CASES = {"tie_b3_p784_k20_c90": (3, 784, 20, 90, 2), "tie_b32_p3136_k7_c128": (32, 3136, 7, 128, 4)}
ITERS = [0, 1, 2, 10]


def test_cases_cover_every_plan():
    plans = {n: plan(*c) for n, c in CASES.items()}
    assert {p["team"] for p in plans.values()} >= {32, 26, 8}
    assert [team_size(b, 132) for b in (1, 3, 5, 17, 32)] == [32, 32, 26, 8, 8]
    assert plans["b17_p784_k1_c90"]["ctas"] > 132 and plans["b32_p3136_k20_c90"]["ctas"] == 256   # two rounds
    assert {p["creg"] for p in plans.values()} == {96, 128}
    assert {(p["creg"], p["rows_smem"]) for p in plans.values()} >= {(96, True), (96, False), (128, True)}
    assert not plans["b32_p3136_k64_c90"]["rows_smem"]
    assert plans["b32_p3136_k40_c90"]["n_priv"] == 4 and min(p["n_priv"] for p in plans.values()) <= 5
    assert max(p["n_priv"] for p in plans.values()) == K_WARPS
    assert {1, 2, 7, 20, 40, 64} <= {c[2] for c in CASES.values()}
    assert {3136, 1369, 1024, 784} <= {c[1] for c in CASES.values()}
    assert {90, 33, 128} <= {c[3] for c in CASES.values()}
    assert any(k % 2 for _, _, k, _ in CASES.values())                        # the one-centroid tail of a pass
    assert all(j % 2 == 0 for *_, j in TIE_CASES.values())                    # ties inside one pass


# ------------------------------------------------------------------------------------------------ data and reference
def init_index(P, K):
    return ((2 * torch.arange(K) + 1) * P) // (2 * K)


def blobs(B, P, K, C, seed, device, tie=None):
    """(B, P, C) fp32 rows of K well-separated blobs; the row at initial position k is in blob k.  tie = j: blob j + 1
    is empty and its initial row is a copy of blob j's."""
    g = torch.Generator(device=device).manual_seed(seed)
    centres = 3.0 * torch.randn(B, K, C, device=device, generator=g)
    label = torch.randint(0, K, (B, P), device=device, generator=g)
    idx = init_index(P, K).to(device)
    label[:, idx] = torch.arange(K, device=device)
    if tie is not None:
        label[label == tie + 1] = tie
    x = torch.gather(centres, 1, label[..., None].expand(B, P, C)) + 0.3 * torch.randn(B, P, C, device=device,
                                                                                       generator=g)
    if tie is not None:
        x[:, idx[tie + 1]] = x[:, idx[tie]]
    return x.contiguous()


def head_buffer(x, npad):
    """Head layout [B * npad, LD] full of sentinel NaNs, with the rows' code at CODE_COL of rows 1..P of each frame."""
    B, P, C = x.shape
    rows = torch.full((B * npad, LD), float("nan"), device=x.device)
    rows.view(B, npad, LD)[:, 1: 1 + P, CODE_COL: CODE_COL + C] = x
    return rows


def score_bound(x64, c64, creg):
    """(CREG / 4 + 10) u (|x| |c| + |c|^2 / 2) -> (B, P, K)."""
    return (creg / 4 + 10) * U * (x64.abs() @ c64.abs().transpose(1, 2) + 0.5 * (c64 ** 2).sum(-1)[:, None, :])


def lloyd64(x, K, iters, n_priv, team, creg, tie=None):
    """float64 Lloyd iterations with image_kmeans's rules -> centroids (B, K, C), centroid bound, and asserts that
    every iteration's assignment is unambiguous under the kernel's bounds."""
    x64 = x.double()
    B, P, C = x64.shape
    c = x64[:, init_index(P, K).to(x.device)].clone()
    e = torch.zeros_like(c)
    distinct = torch.ones(K, dtype=torch.bool, device=x.device)
    if tie is not None:
        distinct[tie + 1] = False
    for _ in range(iters):
        s = x64 @ c.transpose(1, 2) - 0.5 * (c ** 2).sum(-1)[:, None, :]
        assign = s.argmax(-1)
        if K > 1:
            sd = s[..., distinct]
            top = sd.topk(2, dim=-1).values
            gap = top[..., 0] - top[..., 1]
            # a kernel score differs from s by its rounding bound plus the effect of the centroids' error
            sb = score_bound(x64, c + e, creg) + (x64.abs() + c.abs().amax(1, keepdim=True) + e.amax(1, keepdim=True)) \
                .matmul(e.transpose(1, 2))
            margin = 2 * sb.amax(-1)
            assert bool((gap > margin).all()), f"ambiguous assignment: min gap / margin {(gap / margin).min().item()}"
        oh = torch.nn.functional.one_hot(assign, K).double()
        cnt = oh.sum(1)
        sums = oh.transpose(1, 2) @ x64
        mag = oh.transpose(1, 2) @ x64.abs()
        live = cnt[..., None] > 0
        new = sums / cnt[..., None].clamp_min(1)
        e = torch.where(live, (cnt[..., None] + n_priv + team) * U * mag / cnt[..., None].clamp_min(1) + U * new.abs(),
                        e)
        c = torch.where(live, new, c)
    return c, e


def test_lloyd64_matches_image_kmeans():
    from oracle.stego_head import image_kmeans

    B, P, K, C = 2, 196, 7, 33
    x = blobs(B, P, K, C, seed=1, device="cpu")
    for it in (0, 1, 3):
        c, _ = lloyd64(x, K, it, 16, 32, 96)
        want = image_kmeans(x.double().transpose(1, 2).reshape(B, C, 14, 14), K, it)
        assert (c - want).abs().max().item() <= 1e-12


def test_lloyd64_rejects_ambiguous_data():
    """The unambiguity assertion bites: two blobs' worth of rows placed on the midpoint of two centroids."""
    B, P, K, C = 1, 196, 4, 33
    x = blobs(B, P, K, C, seed=2, device="cpu")
    idx = init_index(P, K)
    x[0, 5] = 0.5 * (x[0, idx[0]] + x[0, idx[1]])
    with pytest.raises(AssertionError):
        lloyd64(x, K, 1, 16, 32, 96)


# ------------------------------------------------------------------------------------------------ GPU
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(x, K, iters, npad):
    from wild_visual_navigation_b200 import ops

    B, P, C = x.shape
    rows = head_buffer(x, npad)
    before = rows.clone()
    cent = torch.full((B * K * C + 64,), float("nan"), device=x.device)
    ops.stego_kmeans(rows, B, npad, P, CODE_COL, C, LOGIT_COL, K, iters, centroids_out=cent)
    torch.cuda.synchronize()
    assert bool(torch.isnan(cent[B * K * C:]).all()), "centroids_out written past its end"
    owned = torch.zeros(B, npad, LD, dtype=torch.bool, device=x.device)
    owned[:, 1: 1 + P, LOGIT_COL: LOGIT_COL + K] = True
    assert_owned_and_untouched(rows, before, owned.view(B * npad, LD), "kmeans head buffer")
    score = rows.view(B, npad, LD)[:, 1: 1 + P, LOGIT_COL: LOGIT_COL + K]
    return cent[: B * K * C].view(B, K, C), score, rows


def _check(x, K, iters, cent, score, p, tag, tie=None):
    c64, e = lloyd64(x, K, iters, p["n_priv"], p["team"], p["creg"], tie)
    if iters == 0:
        assert torch.equal(cent.double(), c64), f"{tag}: initial centroids are not the rows at (2k + 1) P / 2K"
    assert_within(cent, c64, e, f"km_centroids_{tag}")
    x64, ck = x.double(), cent.double()
    ref = x64 @ ck.transpose(1, 2) - 0.5 * (ck ** 2).sum(-1)[:, None, :]
    assert_within(score, ref, score_bound(x64, ck, p["creg"]), f"km_scores_{tag}")


@pytest.mark.gpu
@pytest.mark.parametrize("iters", ITERS)
@pytest.mark.parametrize("name", list(CASES))
def test_kmeans_vs_float64(name, iters):
    B, P, K, C = CASES[name]
    p = plan(B, P, K, C, _sms())
    x = blobs(B, P, K, C, seed=len(name) + iters, device="cuda")
    cent, score, _ = _run(x, K, iters, npad=P + 6)
    _check(x, K, iters, cent, score, p, f"team{p['team']}_creg{p['creg']}_{'smem' if p['rows_smem'] else 'gmem'}")


@pytest.mark.gpu
@pytest.mark.parametrize("iters", [0, 1])
@pytest.mark.parametrize("name", list(TIE_CASES))
def test_kmeans_ties_and_empty_cluster(name, iters):
    """Centroids j and j + 1 start identical, so the first assignment ties on every row.  iters = 0: the scores of
    j + 1 equal those of j bit for bit.  iters = 1: the lower index won every tie, so cluster j + 1 is empty and kept
    its initial row bit for bit, and cluster j is its blob's mean.  (Later iterations move centroid j to that mean,
    after which the two no longer tie.)"""
    B, P, K, C, j = TIE_CASES[name]
    p = plan(B, P, K, C, _sms())
    x = blobs(B, P, K, C, seed=11, device="cuda", tie=j)
    cent, score, _ = _run(x, K, iters, npad=P + 3)
    _check(x, K, iters, cent, score, p, "ties", tie=j)
    init = x[:, init_index(P, K).to(x.device)]
    assert torch.equal(cent[:, j + 1].view(torch.int32), init[:, j + 1].view(torch.int32)), "empty cluster moved"
    if iters == 0:
        assert torch.equal(score[..., j].contiguous().view(torch.int32), score[..., j + 1].contiguous().view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["b3_p1369_k7_c90", "b32_p3136_k20_c90", "b32_p3136_k64_c90"])
def test_kmeans_deterministic(name):
    """Two launches give bit-identical centroids and head buffers (the arrival counters are reset per launch)."""
    B, P, K, C = CASES[name]
    x = blobs(B, P, K, C, seed=5, device="cuda")
    c1, _, r1 = _run(x, K, 10, P + 6)
    c2, _, r2 = _run(x, K, 10, P + 6)
    assert torch.equal(c1.view(torch.int32), c2.view(torch.int32))
    assert torch.equal(r1.view(torch.int32), r2.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("P,K,C,logit_col", [(784, 0, 90, 128), (784, 65, 90, 128), (784, 20, 129, 192),
                                             (10, 20, 90, 128), (784, 20, 90, 64)])
def test_kmeans_rejects(P, K, C, logit_col):
    """K = 0 and 65, code_dim = 129, fewer patches than clusters, and a logit range over the code columns raise
    and leave the buffer untouched."""
    from wild_visual_navigation_b200 import ops
    from wild_visual_navigation_b200._C import WvnError

    B, npad = 2, 800
    rows = torch.randn(B * npad, LD, device="cuda")
    before = rows.clone()
    with pytest.raises(WvnError):
        ops.stego_kmeans(rows, B, npad, P, CODE_COL, C, logit_col, K, 10)
    torch.cuda.synchronize()
    assert torch.equal(rows, before)
