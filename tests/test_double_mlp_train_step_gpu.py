"""The DoubleMLP train step (csrc/double_mlp_train.cu) phase by phase against a one-step float64 reference: the
statistics, the ConfidenceGenerator update, the per-row confidence, every element of the 12 gradient tensors, the
confidence-weighted traversability sum, Adam and the loss metrics, at every tile, tail, padding and live-row geometry
of the shared fp32 GEMM (csrc/train_core.cu) and the step's row kernels.

wvn_double_mlp_train_step_padded runs by phase_mask 1, 2 and 4 (as ops.DoubleMlpTrainer does without a library
communicator) and the state is read in between:
  after 1  the statistics block (sum_lr, sum_lr2, sum_raw, n_valid, n_rows, reserved, x_min, x_max);
  after 2  cg_mean / cg_std, var and the running sums (bound to test tensors with set_confidence), conf of every
           compacted row (rows past n_live untouched), the flat gradient and Σ raw·w (statistics block entry 8, fp64);
  after 4  metrics, params, exp_avg, exp_avg_sq and the step counter.
Every step's reference starts from the kernel's own state before that step (params, moments, step counter, generator
state), so every step is held to a one-step bound.  Three steps per case carry running_mean's sums, kalman_filter's
state and moving_average's window; the test keeps its own float64 window (test_train_step_gpu.generator_ref).  Only
published state is read: lo / hi are derived from the published mean / std with 3 u of slack, moving_average's
clipped extrema from the float64 extrema.

Error model of this step's kernels.  First order, on magnitudes, in float64, u = 2^-24; a sum of n fp32 terms with
S = sum |terms| gets acc(n, S) = (C_DOUBLE n + 2) u S (the + 2 covers the last roundings when n is small); errors of
inputs are carried through |W| and |a| (the worst-case rule of test_train_step_gpu.py: the nets are three layers deep).
  tiled GEMM      every output element is one thread's fma chain over K in K order (no split-K, no atomics), then
                  + bias, then fmaxf(v, 0) or the ReLU mask: acc(K + 1, |a||W|^T + |b|) plus the carried e_a |W|^T
  forward         per net: z1 (K = D), z2 (K = h1), z3 (K = h2); ReLU = fmaxf is 1-Lipschitz, e_a = e_z.
                  Layer 3 writes column 0 = 1 / (1 + expf(-v)) of net 0: 1/4 e_z3 + 6 u t; columns 1..D from net 1
  loss rows       loss_reco = (warp tree over D) / D: each lane's fma chain of ceil(D / 32) squares, 5 butterfly adds,
                  the division: the squares carry 2 |df| (e_rec + u |df|), the accumulation (ceil(D / 32) + 5) u
                  sum df^2, + u loss_reco.  raw = (t - y)^2: 2 |dt| (e_t + u |dt|) + u raw
  statistics      fp64 sums of the rows' values: the row bounds summed (+ 2^-50 relative for the fp64 adds); counts
                  exact; the extrema (fminf / fmaxf, NaN skipped) within the largest row bound
  dOut            column 0: g_trav w (t - y) t (1 - t), g_trav = w_trav 2 / n_rows over the global row count, w = 1 -
                  conf for unlabelled rows when anomaly_balanced (else 1); columns 1..D: g_reco (rec - x) on labelled
                  rows, g_reco = w_reco 2 / (n_valid D).  conf = L e_lr + 8 u, L the method's Lipschitz constant
  data gradients  net 0: dA2 = dOut_0 W3_0 (K = 1); net 1: dA2 = dOut_1..D W3_1 (K = D); dA1 = dZ2 W2 (K = h2); each
                  masked by a > 0 of its own net's activations.  A (row, unit) whose float64 pre-activation lies within
                  its own bound of 0 may take either mask: |dz| + e_dz of that row is added to its bound
  weight grads    one six-problem launch over the n_live rows: dW = dZ^T A, e_dZ^T |A| + |dZ|^T e_A + acc(n_live,
                  |dZ|^T |A|); db = the plain fp32 column sum of dZ accumulated alongside in K order: acc(n_live, ...)
  Σ raw·w         wraw = raw w in fp32 (+ u), summed in fp64
  Adam            test_train_step_gpu.adam_ref on the kernel's own gradient
  metrics         from the kernel's own fp64 sums as double_finish_kernel forms them: loss_trav, loss_reco and
                  loss_trav_confidence are one fp64 division rounded to fp32 and must be equal bit for bit, mean / std
                  are the published ones; loss_total (two fp32 products, one sum, possibly contracted) within 3 u.
C_DOUBLE is measured as C_TRAIN and C_FLOW were: the bound is affine in c to first order, so for every element
(|err| - bound at c = 0) / (bound - bound at c = 0) * c is the smallest c that covers it.  Its maximum over a check is
the check's "c needed", printed at the end of the module (pytest -s) with the worst error / bound, and recorded in
DESIGN.md §4 with the chosen margin.

NaN: with n_valid = 0 (mean of an empty set) or 1 (std of one element) the reference produces NaN; the kernel's
metrics, conf and gradients must be NaN in exactly the same places, and every finite element within its bound.

Padding: a padded step must equal the same rows compacted bit for bit (one launch sequence bounded by the device live
count), also for the LinearRnvp step, whose compaction filters by n_rows and y_valid at once.  Stale workspace rows of
an earlier, larger step must not be read.  A step that outgrows max_rows must continue the generator exactly.

The CPU section (no gpu mark) checks the float64 reference against oracle/double_mlp.train_step's autograd gradients
and holds the negative controls: each corrupts a correct record in one place and the checker must reject it.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_kernel_edges_gpu as edges  # noqa: E402
import test_train_step_gpu as ts  # noqa: E402

U = 2.0 ** -24
# accumulator constant of acc(n, S).  Measured over this module on one H100 80GB HBM3 (700 W), the smallest c that
# covers every element of every check is 0 (the + 2 floor and the carried terms suffice); 0.01 keeps the fused step's
# margin above that, and every negative control below is rejected at it (DESIGN.md §4)
C_DOUBLE = 0.01
METHODS = ts.METHODS
CFG = dict(w_trav=0.03, w_reco=0.5, std_factor=0.5, anomaly_balanced=True, lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
STATS = ["sum_lr", "sum_lr2", "sum_raw", "n_valid", "n_rows", "reserved", "x_min", "x_max"]
LAYERS = ("W1", "b1", "W2", "b2", "W3", "b3")
SENTINEL = 12345.0


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    tags = {k: v for k, v in edges._WORST.items() if k.startswith("dm_")}
    if tags:
        print(f"\nDoubleMLP train step, worst error / bound at c = {C_DOUBLE} (c needed: the smallest c covering every "
              "element):")
        for tag in sorted(tags):
            need = ts._NEED.get(tag)
            print(f"  {tag:22s} {tags[tag][0]:.4f}   c needed {need[0] if need else 0.0:.4f}   "
                  f"worst at {need[1] if need else ts._WHERE.get(tag, (0, '-'))[1]}")


def _one(v):
    return torch.tensor(v, dtype=torch.float64)


def check(got, ref, bound, tag, b0=None):
    ts.check(got, ref, bound, tag, b0, c=C_DOUBLE)


def acc(n, S, c):
    return (c * n + 2) * U * S


# ------------------------------------------------------------------------------------------------ float64 reference
def unflat(P, D, h1, h2):
    """The flat parameter vector -> [net 0, net 1], each {layer: view}, in parameters() order."""
    nets, o = [], 0
    for last in (1, D):
        net = {}
        for name, shape in zip(LAYERS, ((h1, D), (h1,), (h2, h1), (h2,), (last, h2), (last,))):
            k = math.prod(shape)
            net[name] = P[o:o + k].view(shape)
            o += k
        nets.append(net)
    return nets


def forward_ref(P, x, y, D, h1, h2, c=C_DOUBLE):
    """Both nets, the output and the per-row loss terms in float64, each value with its bound (module docstring)."""
    nets = unflat(P, D, h1, h2)
    fw = dict(nets=nets, net=[])
    for W in nets:
        z1 = x @ W["W1"].T + W["b1"]
        e_z1 = acc(D + 1, x.abs() @ W["W1"].abs().T + W["b1"].abs(), c)
        a1 = z1.clamp_min(0)
        z2 = a1 @ W["W2"].T + W["b2"]
        e_z2 = e_z1 @ W["W2"].abs().T + acc(h1 + 1, (a1 + e_z1) @ W["W2"].abs().T + W["b2"].abs(), c)
        a2 = z2.clamp_min(0)
        z3 = a2 @ W["W3"].T + W["b3"]
        e_z3 = e_z2 @ W["W3"].abs().T + acc(h2 + 1, (a2 + e_z2) @ W["W3"].abs().T + W["b3"].abs(), c)
        fw["net"].append(dict(z1=z1, e_z1=e_z1, a1=a1, z2=z2, e_z2=e_z2, a2=a2, z3=z3, e_z3=e_z3))
    n0, n1 = fw["net"]
    t = torch.sigmoid(n0["z3"][:, 0])
    e_t = 0.25 * n0["e_z3"][:, 0] + 6 * U * t
    rec, e_rec = n1["z3"], n1["e_z3"]
    df = rec - x
    sq = df * df
    lr = sq.mean(1)
    e_lr = ((2 * df.abs() * (e_rec + U * df.abs())).sum(1) + (-(-D // 32) + 5) * U * sq.sum(1)) / D + U * lr
    dt = t - y
    raw = dt * dt
    e_raw = 2 * dt.abs() * (e_t + U * dt.abs()) + U * raw
    fw.update(t=t, e_t=e_t, rec=rec, e_rec=e_rec, lr=lr, e_lr=e_lr, raw=raw, e_raw=e_raw)
    return fw


def stats_ref(fw, yv, drop=None):
    """test_train_step_gpu.stats_ref; drop: rows left out of the three sums (a negative control)."""
    if drop is None:
        return ts.stats_ref(fw, yv)
    keep = torch.ones_like(yv)
    keep[drop] = False
    part = ts.stats_ref(dict(lr=fw["lr"][keep], e_lr=fw["e_lr"][keep], raw=fw["raw"][keep], e_raw=fw["e_raw"][keep]),
                        yv[keep])
    st = ts.stats_ref(fw, yv)
    st.update({k: part[k] for k in ("sum_lr", "sum_lr2", "sum_raw")})
    return st


def published_view(method, mean, std, st, f):
    """What a row's confidence needs (lo, hi, cmin, cmax), derived from the kernel's published mean / std, and their
    slack: 3 u of the fp32 arithmetic that forms them; moving_average's clipped extrema from the float64 extrema."""
    m, sd = np.float64(mean), np.float64(std)
    with np.errstate(all="ignore"):
        if method == "kalman_filter":
            return dict(lo=float(m), hi=float(1 / (sd * f)), cmin=0.0, cmax=0.0), 0.0
        if method == "moving_average":
            lo, hi = m - 2 * sd, m + 2 * sd
            e = 3 * U * (abs(m) + 2 * abs(sd))
            cmin = float(np.fmin(np.fmax(st["x_min"][0], lo), hi))
            cmax = float(np.fmin(np.fmax(st["x_max"][0], lo), hi))
            return dict(lo=float(lo), hi=float(hi), cmin=cmin, cmax=cmax), max(e, st["x_min"][1])
        lo, hi = float(np.fmax(m + sd * f - sd, 0.0)), float(m + sd * f + sd)
        return dict(lo=lo, hi=hi, cmin=0.0, cmax=0.0), 3 * U * (abs(m) + (f + 1) * abs(sd))


def loss_scales(cfg, n_valid, n_rows, D):
    """g_reco and g_trav as double_conf_kernel forms them, over the (global) counts: one fp32 rounding each."""
    with np.errstate(all="ignore"):
        return (float(np.float64(ts.f32(cfg["w_reco"]) * 2) / (np.float64(n_valid) * D)),
                float(np.float64(ts.f32(cfg["w_trav"]) * 2) / np.float64(n_rows)))


def _relu_back(da, e_da, z, e_z):
    on, amb = z > 0, z.abs() <= e_z
    dz = torch.where(on, da, torch.zeros_like(da))
    e_dz = torch.where(on, e_da, torch.zeros_like(da)) + torch.where(amb, da.abs() + e_da, torch.zeros_like(da))
    return dz, e_dz


def backward_ref(fw, x, y, yv, method, g, cfg, e_lohi=0.0, c=C_DOUBLE, w_unl=None, drop=None, short_db=None,
                 w_on=None, swap_masks=False):
    """conf, dOut, the 12 gradient tensors and Σ raw·w in float64, with bounds.  g: lo, hi, cmin, cmax, g_reco, g_trav
    (derived from published values: e_lohi and one rounding of g are their slack).  w_unl: the unlabelled rows'
    weights in place of 1 - conf (the oracle's own fp32 weights).  Negative controls: drop (rows left out of every
    gradient sum and of Σ raw·w), short_db ((net, layer) whose bias gradient stops a row short), w_on (labelled rows
    given the 1 - conf weight), swap_masks (each net's layer-2 ReLU mask read from the other net's activations)."""
    conf, L = ts.row_conf_ref(method, fw["lr"], g["lo"], g["hi"], g["cmin"], g["cmax"])
    e_conf = L * (fw["e_lr"] + 3 * e_lohi) + 8 * U
    full = yv | (not cfg["anomaly_balanced"])
    if w_on is not None:
        full = full.clone()
        full[w_on] = False
    wgt = torch.where(full, torch.ones_like(conf), 1 - conf if w_unl is None else w_unl.to(conf))
    e_wgt = torch.where(full, torch.zeros_like(conf), e_conf)
    t, e_t = fw["t"], fw["e_t"]
    q = (t - y) * t * (1 - t)
    e_q = (0.25 + (t - y).abs() * (1 - 2 * t).abs()) * e_t
    gt, gr = g["g_trav"], g["g_reco"]
    d0 = gt * wgt * q
    e_d0 = gt * (e_wgt * q.abs() + wgt * e_q) + 8 * U * d0.abs()
    with np.errstate(all="ignore"):
        dr = torch.where(yv[:, None], gr * (fw["rec"] - x), torch.zeros_like(x))
        e_dr = torch.where(yv[:, None], gr * fw["e_rec"] + 4 * U * dr.abs(), torch.zeros_like(x))
    R = x.shape[0]
    keep = torch.ones(R, dtype=x.dtype, device=x.device)
    if drop is not None:
        keep[drop] = 0
    nets, rows = fw["nets"], []
    for k, (dz3, e_dz3) in enumerate(((d0[:, None], e_d0[:, None]), (dr, e_dr))):
        W, N = nets[k], fw["net"][k]
        M = fw["net"][1 - k] if swap_masks else N
        K3 = dz3.shape[1]
        da2 = dz3 @ W["W3"]
        dz2, e_dz2 = _relu_back(da2, e_dz3 @ W["W3"].abs() + acc(K3, dz3.abs() @ W["W3"].abs(), c), M["z2"], M["e_z2"])
        da1 = dz2 @ W["W2"]
        dz1, e_dz1 = _relu_back(da1, e_dz2 @ W["W2"].abs() + acc(W["W2"].shape[0], dz2.abs() @ W["W2"].abs(), c),
                                N["z1"], N["e_z1"])
        rows.append(dict(dz3=dz3, dz2=dz2, dz1=dz1))
        out = {}
        for (lw, lb), dz, e_dz, a, e_a in ((("W3", "b3"), dz3, e_dz3, N["a2"], N["e_z2"]),
                                           (("W2", "b2"), dz2, e_dz2, N["a1"], N["e_z1"]),
                                           (("W1", "b1"), dz1, e_dz1, x, None)):
            dzk, e_dzk = dz * keep[:, None], e_dz * keep[:, None]
            prop = e_dzk.T @ a.abs() + (dzk.abs().T @ e_a if e_a is not None else 0)
            out[lw] = (dzk.T @ a, prop + acc(R, dzk.abs().T @ a.abs(), c))
            sb = dzk.sum(0)
            if short_db == (k, lb):
                sb = sb - dzk[-1]
            out[lb] = (sb, e_dzk.sum(0) + acc(R, dzk.abs().sum(0), c))
        grads_k = out
        rows[-1]["grads"] = grads_k
    rw = fw["raw"] * wgt * keep
    tw = rw.sum()
    e_tw = (fw["e_raw"] * wgt + fw["raw"] * e_wgt).mul(keep).sum() + (U + 2.0 ** -50) * rw.abs().sum()
    return dict(conf=(conf, e_conf), rows=rows, trav_w=(tw, e_tw))


def flat_grads(bw, i):
    """Value (i = 0) or bound (i = 1) of every gradient as one vector in parameters() order."""
    return torch.cat([bw["rows"][k]["grads"][name][i].reshape(-1) for k in (0, 1) for name in LAYERS])


# ------------------------------------------------------------------------------------------------ the checker
def check_step(tag, rec, x, y, yv, D, h1, h2, method="latest_measurement", cfg=CFG, window=None, where="", need=True):
    """Every phase of one recorded step against the float64 reference started from the kernel's state before it.
    x / y / yv: the live rows, compacted.  need: also take the reference at c = 0, for "c needed".  Returns
    moving_average's new window."""
    b, dev = rec["before"], x.device
    P, x64, y64 = b["params"].to(dev), x.double(), y.double()
    R, f = x.shape[0], cfg["std_factor"]
    ts._CTX[0] = f"{tag} {method} D={D} h={h1}/{h2} R={R} {where}".strip()
    fw = forward_ref(P, x64, y64, D, h1, h2)
    fw0 = forward_ref(P, x64, y64, D, h1, h2, c=0.0) if need else None
    st = stats_ref(fw, yv)
    st0 = stats_ref(fw0, yv) if need else None
    # ---- phase 1: the statistics block
    p1 = rec["p1"]
    assert p1["n_valid"] == st["n_valid"][0] and p1["n_rows"] == R and p1["reserved"] == 0, \
        f"{tag}: counts {p1['n_valid']} / {p1['n_rows']} / {p1['reserved']}, want {st['n_valid'][0]} / {R} / 0"
    for k in ("sum_lr", "sum_lr2", "sum_raw", "x_min", "x_max"):
        check(_one([p1[k]]), _one([st[k][0]]), _one([st[k][1]]), f"dm_{k}", _one([st0[k][1]]) if need else None)
    # ---- phase 2: generator, confidence, gradients, Σ raw·w
    p2 = rec["p2"]
    gen, window = ts.generator_ref(method, st, b, window or [], f)
    check(_one([p2["cg_mean"]]), _one([gen["mean"][0]]), _one([gen["mean"][1]]), "dm_gen_mean")
    if not (method == "running_mean" and abs(gen["var"][0]) <= gen["var"][1] and math.isnan(p2["cg_std"])):
        # a running variance of 0 within its bound may round below 0 in fp32 (its sqrtf is NaN), as in the reference
        check(_one([p2["cg_std"]]), _one([gen["std"][0]]), _one([gen["std"][1]]), "dm_gen_std")
    if "var" in gen:
        check(_one([p2["var"]]), _one([gen["var"][0]]), _one([gen["var"][1]]), "dm_gen_var")
    if method == "running_mean":
        assert p2["running"][0] == gen["running_n"][0], f"{tag}: running_n {p2['running'][0]}"
        for i, k in ((1, "running_sum"), (2, "running_sumsq")):
            check(_one([p2["running"][i]]), _one([gen[k][0]]), _one([gen[k][1]]), f"dm_gen_{k}")
    g, e_lohi = published_view(method, p2["cg_mean"], p2["cg_std"], st, f)
    g["g_reco"], g["g_trav"] = loss_scales(cfg, p1["n_valid"], p1["n_rows"], D)
    bw = backward_ref(fw, x64, y64, yv, method, g, cfg, e_lohi)
    if need:
        g0, e0 = published_view(method, p2["cg_mean"], p2["cg_std"], st0, f)
        g0.update(g_reco=g["g_reco"], g_trav=g["g_trav"])
        bw0 = backward_ref(fw0, x64, y64, yv, method, g0, cfg, e0, c=0.0)
    check(p2["conf"][:R], bw["conf"][0], bw["conf"][1], "dm_conf", bw0["conf"][1] if need else None)
    assert bool((p2["conf"][R:] == SENTINEL).all()), f"{tag}: conf written past the {R} live rows"
    grads = p2["grads"].to(dev).double()
    o = 0
    for k in (0, 1):
        for name in LAYERS:
            ref, bound = bw["rows"][k]["grads"][name]
            n = ref.numel()
            check(grads[o:o + n].view(ref.shape), ref, bound, f"dm_d{name}.{k}",
                  bw0["rows"][k]["grads"][name][1] if need else None)
            o += n
    assert o == grads.numel()
    tw, e_tw = bw["trav_w"]
    check(_one([p2["trav_w"]]), tw.reshape(1).cpu(), e_tw.reshape(1).cpu(), "dm_trav_w",
          bw0["trav_w"][1].reshape(1).cpu() if need else None)
    # ---- phase 4: metrics from the kernel's own sums, Adam on the kernel's own gradient
    a = rec["after"]
    assert a["step"] == b["step"] + 1, f"{tag}: step counter {b['step']} -> {a['step']}"
    met = a["metrics"]
    with np.errstate(all="ignore"):
        lreco = ts.f32(np.float64(p1["sum_lr"]) / np.float64(p1["n_valid"]))
        ltrav = ts.f32(np.float64(p1["sum_raw"]) / np.float64(p1["n_rows"]))
        ltc = ts.f32(np.float64(p2["trav_w"]) / np.float64(p1["n_rows"]))
    ts.same(met[1], ltrav, f"{tag}: loss_trav")
    ts.same(met[2], lreco, f"{tag}: loss_reco")
    ts.same(met[3], ltc, f"{tag}: loss_trav_confidence")
    wt, wr = ts.f32(cfg["w_trav"]), ts.f32(cfg["w_reco"])
    check(_one([met[0]]), _one([wt * ltc + wr * lreco]), _one([3 * U * (abs(wt * ltc) + abs(wr * lreco))]),
          "dm_loss_total")
    ts.same(met[4], p2["cg_mean"], f"{tag}: metrics mean")
    ts.same(met[5], p2["cg_std"], f"{tag}: metrics std")
    b1, b2 = (ts.f32(v) for v in cfg["betas"])
    (p, e_p), (mm, e_m), (vv, e_v) = ts.adam_ref(P, grads, b["m"].to(dev), b["v"].to(dev), a["step"],
                                                 ts.f32(cfg["lr"]), b1, b2, ts.f32(cfg["eps"]))
    check(a["m"], mm, e_m, "dm_adam_m")
    check(a["v"], vv, e_v, "dm_adam_v")
    check(a["params"], p, e_p, "dm_adam_p")
    return window


# ------------------------------------------------------------------------------------------------ the GPU driver
def make_model(D, h1, h2, seed=42, device="cuda"):
    from wild_visual_navigation_b200 import DoubleMLP

    torch.manual_seed(seed)
    return DoubleMLP(D, [h1, h2, 1]).to(device)


class Trainer:
    """ops.DoubleMlpTrainer driven phase by phase, with its generator state in tensors the test can read (or private
    to the handle: bound=False)."""

    def __init__(self, model, max_rows=4096, method="latest_measurement", cfg=CFG, bound=True):
        from wild_visual_navigation_b200 import ops

        self.model, self.cfg = model, cfg
        self.tr = ops.DoubleMlpTrainer(model, max_rows=max_rows, w_trav=cfg["w_trav"], w_reco=cfg["w_reco"],
                                       std_factor=cfg["std_factor"], anomaly_balanced=cfg["anomaly_balanced"],
                                       lr=cfg["lr"], betas=cfg["betas"], eps=cfg["eps"])
        self.var = torch.ones(1, 1, device="cuda")
        self.running = torch.zeros(3, dtype=torch.float64, device="cuda")
        if bound:
            self.tr.set_confidence(METHODS[method], self.var, self.running[0:1], self.running[1:2], self.running[2:3])
        else:
            self.tr.set_confidence(METHODS[method])

    def state(self):
        tr = self.tr
        return dict(params=self.model.flat_params.double().clone(), m=tr.exp_avg.double().clone(),
                    v=tr.exp_avg_sq.double().clone(), step=int(tr.step_counter.item()), cg_mean=tr.cg_mean.item(),
                    cg_std=tr.cg_std.item(), var=self.var.item(), running=self.running.tolist())

    def run(self, x, y, yv, groups=1, rpg=None, n_rows=None):
        """One step by phase_mask 1, 2, 4; x is [groups * rpg, D] (padded per group when n_rows is given), y / yv in
        compacted numbering."""
        from wild_visual_navigation_b200._C import check as ccheck, lib, ptr, stream

        tr, rec = self.tr, {}
        rpg = x.shape[0] if rpg is None else rpg
        tr._reserve(groups * rpg)
        rec["before"] = self.state()
        tr.conf.fill_(SENTINEL)   # conf is written at the compacted rows only
        x, y, yv = x.contiguous().float(), y.contiguous().float(), yv.contiguous().to(torch.uint8)

        def phase(mask):
            ccheck(lib().wvn_double_mlp_train_step_padded(
                tr._h, ptr(self.model.flat_params), ptr(tr.exp_avg), ptr(tr.exp_avg_sq), ptr(tr.step_counter), ptr(x),
                groups, rpg, ptr(n_rows), ptr(y), ptr(yv), ptr(tr.cg_mean), ptr(tr.cg_std), ptr(tr.conf),
                ptr(tr.metrics), mask, stream()))

        phase(1)
        rec["p1"] = dict(zip(STATS, tr.stats[:8].tolist()))
        phase(2)
        rec["p2"] = dict(cg_mean=tr.cg_mean.item(), cg_std=tr.cg_std.item(), var=self.var.item(),
                         running=self.running.tolist(), conf=tr.conf.clone(), grads=tr.grads.clone(),
                         trav_w=tr.stats[8].item())
        phase(4)
        rec["after"] = dict(self.state(), metrics=tr.metrics.tolist())
        return rec


def rows(R, D, seed, p_valid=0.3, scale=1.0, device="cuda"):
    """x ~ N(0.1, 0.8^2) (scaled), about p_valid of the rows labelled (the first two always) with y in (0, 1]."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(R, D, generator=g) * 0.8 + 0.1) * scale
    yv = torch.rand(R, generator=g) < p_valid
    yv[:2] = True
    y = torch.where(yv, torch.rand(R, generator=g).clamp(min=0.001), torch.zeros(R))
    return x.to(device), y.to(device), yv.to(device)


def run_steps(tag, D, h1, h2, counts, method="latest_measurement", cfg=CFG, max_rows=4096, seed=0, p_valid=0.3):
    """One step per entry of counts on one trainer (the same model init), each checked."""
    T = Trainer(make_model(D, h1, h2), max_rows, method, cfg)
    window = []
    for s, R in enumerate(counts):
        x, y, yv = rows(R, D, 1000 * seed + 10 * s + R, p_valid)
        window = check_step(tag, T.run(x, y, yv), x, y, yv, D, h1, h2, method, cfg, window, where=f"step {s}")
    return T


# ------------------------------------------------------------------------------------------------ GPU: methods, geometry
@pytest.mark.gpu
@pytest.mark.parametrize("method,balanced", [(m, True) for m in METHODS] + [("latest_measurement", False)])
def test_methods(method, balanced):
    """The shipped shape D = 384, [64, 32, 1]: every generator method, three steps of different sizes."""
    run_steps("methods", 384, 64, 32, [700, 1100, 300], method, dict(CFG, anomaly_balanced=balanced), seed=7)


ROWS = [1, 2, 7, 8, 9, 15, 16, 17, 63, 64, 65, 255, 256, 257, 1023, 1024, 1025, 4096, 4097]


@pytest.mark.gpu
@pytest.mark.parametrize("R", ROWS)
def test_compacted_rows(R):
    """8 rows per block of the row kernels, the weight gradients' 16-row K chunk, the 64-row M tile, the statistics
    kernel's 256-thread stride, and 4097 rows, which regrows the trainer past its default max_rows.  The methods rotate
    over the row list; the last row is labelled, so a live bound one short drops a labelled row."""
    method = list(METHODS)[ROWS.index(R) % 4]
    T = Trainer(make_model(384, 64, 32), 4096, method)
    window = []
    for s in range(3):
        x, y, yv = rows(R, 384, R + 10 * s)
        yv[-1] = True
        y[-1] = 0.5
        window = check_step("rows", T.run(x, y, yv), x, y, yv, 384, 64, 32, method, window=window, where=f"step {s}")
    assert T.tr.max_rows >= R


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 2, 31, 32, 33, 63, 64, 65, 90, 384, 768, 1023, 1024])
def test_widths(D):
    """Layer 3's N tail (D + 1 output columns), layer 1's K tail, the weight gradients' M / N tails and the row
    kernels' lane loop."""
    run_steps("widths", D, 64, 32, [1000, 997, 1001], list(METHODS)[D % 4], seed=D)


HIDDEN = [(384, 4, 1, [700]), (384, 60, 15, [700]), (384, 64, 16, [700]), (384, 68, 17, [700]),
          (384, 252, 31, [700]), (384, 256, 32, [700]), (1024, 256, 32, [4097]), (1, 4, 1, [1, 65])]


@pytest.mark.gpu
@pytest.mark.parametrize("D,h1,h2,counts", HIDDEN, ids=[f"{d}x{a}x{b}" for d, a, b, _ in HIDDEN])
def test_hidden_sizes(D, h1, h2, counts):
    """h1 in {4, 60, 64, 68, 252, 256}, h2 in {1, 15, 16, 17, 31, 32}, and the extremes (1024, 256, 32) at 4097 rows
    and (1, 4, 1) at 1 and 65 rows.  Three steps (the first count repeats)."""
    counts = (counts * 3)[:3]
    run_steps("hidden", D, h1, h2, counts, "moving_average" if h1 % 8 else "running_mean", seed=h1 + h2)


# ------------------------------------------------------------------------------------------------ GPU: labels
LABELS = ["all", "one", "two", "none", "one_of_many", "none_unbalanced"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", LABELS)
def test_labels(case):
    """Every row labelled; one or two rows (all labelled); none (the mean of an empty set is NaN); one among many (the
    std of one element is NaN, so conf and the unlabelled rows' weights are NaN); none with anomaly_balanced off.  The
    values are checked wherever the reference is finite, and NaN must appear exactly where the reference has it."""
    R, D = 300, 384
    cfg = dict(CFG, anomaly_balanced=not case.endswith("unbalanced"))
    x, y, yv = rows(R, D, 7)
    if case == "all":
        yv[:] = True
    elif case in ("one", "two"):
        R = 1 if case == "one" else 2
        x, y, yv = x[:R], y[:R], torch.ones(R, dtype=torch.bool, device="cuda")
    elif case.startswith("none"):
        yv[:] = False
    elif case == "one_of_many":
        yv[:] = False
        yv[17] = True
    y = torch.where(yv, torch.rand(R, generator=torch.Generator().manual_seed(3)).cuda().clamp(min=0.001),
                    torch.zeros_like(y))
    T = Trainer(make_model(D, 64, 32), 512, "latest_measurement", cfg)
    rec = T.run(x, y, yv)
    check_step("labels", rec, x, y, yv, D, 64, 32, cfg=cfg)
    assert bool(torch.isnan(rec["p2"]["grads"]).any()) == (case in ("none", "one_of_many")), case
    assert math.isnan(rec["after"]["metrics"][0]) == (case.startswith("none") or case == "one_of_many"), case


# ------------------------------------------------------------------------------------------------ GPU: padded rows
def _geometry(name, seed):
    g = torch.Generator().manual_seed(seed)
    if name == "64x100":
        n = torch.randint(0, 101, (64,), generator=g)
        n[5], n[40] = 0, 100
        return 100, n.tolist()
    if name == "1000x3":
        return 3, torch.randint(0, 4, (1000,), generator=g).tolist()
    if name == "1x4096":
        return 4096, [4095]
    if name == "7x1":
        return 1, [1, 0, 1, 1, 0, 1, 1]
    return 50, [0] * 11 + [37]   # every group empty but the last


PADDED = ["64x100", "1000x3", "1x4096", "7x1", "last_only"]


def padded_rows(name, D, seed, p_valid=0.3):
    """feat [G, S, D] with NaN in every padding row, n_rows [G] int32, the live rows compacted, y / y_valid
    (compacted numbering)."""
    S, counts = _geometry(name, seed)
    G = len(counts)
    x, y, yv = rows(G * S, D, seed, p_valid, device="cpu")
    feat = x.view(G, S, D).clone()
    live = torch.arange(S)[None, :] < torch.tensor(counts)[:, None]
    feat[~live] = float("nan")
    n = int(live.sum())
    return (feat.cuda(), torch.tensor(counts, dtype=torch.int32).cuda(), feat[live].cuda(), y[:n].cuda(),
            yv[:n].cuda())


@pytest.mark.gpu
@pytest.mark.parametrize("geometry", PADDED)
def test_padded_step(geometry):
    """The padded step through the full checker (three steps, moving_average, NaN in the padding), and bit for bit
    against ops.DoubleMlpTrainer.step on the same rows compacted.  64 x 100, 1000 x 3 and 1 x 4096 put more than 1024
    padded rows in one compact_rows launch, so each thread walks several rows across group boundaries; 64 x 100
    also regrows the trainer; the last geometry has every group empty but the last."""
    D = 384
    T = Trainer(make_model(D, 64, 32), 4096, "moving_average")
    C = Trainer(make_model(D, 64, 32), 4096, "moving_average")
    window = []
    for s in range(3):
        feat, n_rows, live, y, yv = padded_rows(geometry, D, 100 * s + len(geometry))
        G, S = feat.shape[:2]
        rec = T.run(feat.view(G * S, D), y, yv, groups=G, rpg=S, n_rows=n_rows)
        window = check_step("padded", rec, live, y, yv, D, 64, 32, "moving_average", window=window,
                            where=f"{geometry} step {s}")
        conf = C.tr.step(live, y, yv)
        n = live.shape[0]
        for a, b, what in ((T.model.flat_params, C.model.flat_params, "params"), (T.tr.exp_avg, C.tr.exp_avg, "m"),
                           (T.tr.exp_avg_sq, C.tr.exp_avg_sq, "v"), (T.tr.grads, C.tr.grads, "grads"),
                           (T.tr.metrics, C.tr.metrics, "metrics"), (T.tr.stats[:9], C.tr.stats[:9], "stats"),
                           (rec["p2"]["conf"][:n], conf[:n], "conf"), (T.tr.cg_mean, C.tr.cg_mean, "cg_mean"),
                           (T.tr.cg_std, C.tr.cg_std, "cg_std"), (T.var, C.var, "var"),
                           (T.tr.step_counter, C.tr.step_counter, "step")):
            assert torch.equal(a, b), f"{geometry} step {s}: padded and compacted {what} differ"


@pytest.mark.gpu
@pytest.mark.parametrize("geometry", PADDED)
@pytest.mark.parametrize("mask", ["odds", "half"])
def test_flow_padded_step_equals_compacted_step(geometry, mask):
    """The LinearRnvp padded step, whose compaction filters by n_rows and by y_valid (compacted numbering) at once,
    against its compacted step on the same rows, bit for bit, at the same geometries (two steps, running_mean)."""
    from test_linear_rnvp_gpu import _model
    from wild_visual_navigation_b200 import ops

    D = 384
    runs = []
    for variant in ("padded", "compacted"):
        m = _model(D, 200, mask)
        tr = ops.FlowTrainer(m, max_rows=4096)
        st = (torch.ones(1, 1, device="cuda"), torch.zeros(3, dtype=torch.float64, device="cuda"))
        tr.set_confidence(METHODS["running_mean"], st[0], st[1][0:1], st[1][1:2], st[1][2:3])
        for s in range(2):
            feat, n_rows, live, y, yv = padded_rows(geometry, D, 200 + 100 * s + len(geometry), p_valid=0.6)
            if variant == "padded":
                tr.step_padded(feat, n_rows, y, yv)
            else:
                tr.step(live, yv)
        n = int(yv.sum())
        runs.append([m.flat_params, tr.exp_avg, tr.exp_avg_sq, tr.step_counter, tr.grads, tr.metrics, tr.cg_mean,
                     tr.cg_std, tr.conf[:n], st[0], st[1]])
    for i, (a, b) in enumerate(zip(*runs)):
        assert torch.equal(a, b), f"{geometry} {mask}: padded and compacted differ at state entry {i}"
    assert torch.isfinite(runs[0][0]).all()


# ------------------------------------------------------------------------------------------------ GPU: workspace, growth
@pytest.mark.gpu
def test_stale_workspace_rows_are_never_read():
    """A 3000-row step with features x8 leaves large activations and gradients in the workspaces; a following
    500-row padded step must be bit-identical to the same step on a fresh trainer (new, zeroed workspaces) given the
    first trainer's params, moments, step counter and generator state."""
    from wild_visual_navigation_b200._C import check as ccheck, lib, stream

    D, method = 384, "running_mean"
    A = Trainer(make_model(D, 64, 32), 4096, method)
    x, y, yv = rows(3000, D, 31, scale=8.0)
    window = check_step("stale", A.run(x, y, yv), x, y, yv, D, 64, 32, method, where="3000 rows x8")
    B = Trainer(make_model(D, 64, 32), 500, method)
    with torch.no_grad():
        B.model.flat_params.copy_(A.model.flat_params)
    for name in ("exp_avg", "exp_avg_sq", "step_counter", "cg_mean", "cg_std"):
        getattr(B.tr, name).copy_(getattr(A.tr, name))
    B.var.copy_(A.var)
    B.running.copy_(A.running)
    ccheck(lib().wvn_trainer_copy_confidence(B.tr._h, A.tr._h, stream()))   # the handle's private state
    g = torch.Generator().manual_seed(32)
    counts = torch.randint(0, 51, (10,), generator=g)
    counts[3] = 50
    n = int(counts.sum())
    xp = torch.full((10, 50, D), float("nan"))
    xl, y, yv = rows(n, D, 33, device="cpu")
    xp[torch.arange(50)[None, :] < counts[:, None]] = xl
    xp, xl, y, yv, n_rows = xp.cuda(), xl.cuda(), y.cuda(), yv.cuda(), counts.to(torch.int32).cuda()
    recs = [T.run(xp.view(500, D), y, yv, groups=10, rpg=50, n_rows=n_rows) for T in (A, B)]
    check_step("stale", recs[0], xl, y, yv, D, 64, 32, method, window=window, where="500 padded after 3000")
    a, b = recs

    def bits(v):   # bit patterns, so that NaN compares equal to the same NaN
        t = torch.as_tensor(v).detach().cpu()
        return t.view(torch.int64 if t.dtype == torch.float64 else torch.int32)

    assert torch.equal(bits(list(a["p1"].values())), bits(list(b["p1"].values())))
    assert torch.equal(bits(a["after"]["metrics"]), bits(b["after"]["metrics"]))
    assert torch.equal(bits([a["p2"]["trav_w"]]), bits([b["p2"]["trav_w"]]))
    for k in ("conf", "grads"):
        assert torch.equal(bits(a["p2"][k][:n]), bits(b["p2"][k][:n])), k
    for k in ("params", "m", "v"):
        assert torch.equal(bits(a["after"][k]), bits(b["after"][k])), k


@pytest.mark.gpu
@pytest.mark.parametrize("bound", [True, False], ids=["bound", "private"])
@pytest.mark.parametrize("method", ["moving_average", "running_mean", "kalman_filter"])
def test_regrowth_keeps_the_generator(method, bound):
    """A step that outgrows max_rows replaces the handle: the generator (moving_average's window and, when private,
    var and the running sums) must continue exactly as on a trainer created large enough."""
    D = 384
    small, large = (Trainer(make_model(D, 64, 32), mr, method, bound=bound) for mr in (256, 4096))
    for s, R in enumerate([200, 230, 180, 600, 210, 190, 1500]):
        x, y, yv = rows(R, D, 80 + s, scale=1.0 + 0.3 * s)
        small.tr.step(x, y, yv)
        large.tr.step(x, y, yv)
        for k in ("cg_mean", "cg_std", "metrics", "exp_avg"):
            assert torch.equal(getattr(small.tr, k), getattr(large.tr, k)), f"step {s}: {k}"
        assert torch.equal(small.model.flat_params, large.model.flat_params), f"step {s}: params"
        if bound:
            assert torch.equal(small.var, large.var) and torch.equal(small.running, large.running), f"step {s}"
    assert small.tr.max_rows >= 1500 and small.tr.max_rows < large.tr.max_rows


# ------------------------------------------------------------------------------------------------ CPU: the reference
ORACLE_SHAPES = [(384, 64, 32, 300), (1, 4, 1, 65), (33, 68, 17, 129), (90, 256, 31, 64), (1024, 16, 1, 17)]


@pytest.mark.parametrize("D,h1,h2,R", ORACLE_SHAPES, ids=[f"{d}x{a}x{b}-{r}" for d, a, b, r in ORACLE_SHAPES])
@pytest.mark.parametrize("balanced", [True, False])
@pytest.mark.parametrize("method", list(METHODS))
def test_reference_matches_autograd(method, balanced, D, h1, h2, R):
    """forward_ref / backward_ref against oracle/double_mlp.train_step (autograd) in float64, fed the oracle's own
    confidence and fp32 weights 1 - conf: the output, and every gradient element to 1e-12 of its tensor's largest.
    Two steps, so the generator carries state; the bounds are finite and non-negative."""
    from oracle import double_mlp as odm
    from oracle.wvn_path import ConfidenceState

    sd = {k: v.double() for k, v in odm.init(D, [h1, h2, 1], seed=5).items()}
    cg = ConfidenceState(0.5, method)
    for s in range(2):
        x, y, yv = rows(R, D, 40 + s + R, device="cpu")
        x, y = x.double(), y.double()
        P = torch.cat([v.reshape(-1) for v in sd.values()])
        fw = forward_ref(P, x, y, D, h1, h2)
        out = odm.forward(sd, x)
        assert (torch.cat([fw["t"][:, None], fw["rec"]], 1) - out).abs().max().item() <= 1e-12 * (1 + out.abs().max())
        new_sd, grads, _, aux = odm.train_step(sd, {}, x, y, yv, cg, anomaly_balanced=balanced)
        conf32 = aux["confidence"]
        n = float(yv.sum())
        g = dict(lo=0.0, hi=1.0, cmin=0.0, cmax=1.0, g_reco=0.5 * 2 / (n * D), g_trav=0.03 * 2 / R)
        bw = backward_ref(fw, x, y, yv, "latest_measurement", g, dict(CFG, anomaly_balanced=balanced),
                          w_unl=(1 - conf32).double())
        mine, bound = flat_grads(bw, 0), flat_grads(bw, 1)
        o = 0
        for name, want in grads.items():
            k = want.numel()
            err = (mine[o:o + k] - want.reshape(-1)).abs().max().item()
            assert err <= 1e-12 * want.abs().max().item() + 1e-300, (method, name, err)
            o += k
        assert o == mine.numel()
        assert bool(torch.isfinite(bound).all()) and bool((bound >= 0).all())
        sd = new_sd


def fake_record(R, seed=9, D=384, h1=64, h2=32, method="latest_measurement", drop_stats=None, corrupt=None,
                scales=None, **bad):
    """A correct record built from the float64 reference rounded to fp32, as Trainer.run would read it from a kernel
    that computes the step exactly.  bad: backward_ref's negative-control options; drop_stats: rows left out of the
    statistic sums; scales: (n_valid, n_rows) the loss scales are formed over; corrupt(rec): any other change.  Adam is
    applied to the gradient as recorded, as the kernel's Adam consumes the kernel's own gradient."""
    from oracle import double_mlp as odm

    P = torch.cat([v.reshape(-1) for v in odm.init(D, [h1, h2, 1]).values()]).double()
    x, y, yv = rows(R, D, seed, device="cpu")
    x64, y64 = x.double(), y.double()
    fw = forward_ref(P, x64, y64, D, h1, h2)
    st = stats_ref(fw, yv, drop=drop_stats)
    before = dict(params=P, m=torch.zeros_like(P), v=torch.zeros_like(P), step=0, cg_mean=0.0, cg_std=1.0, var=1.0,
                  running=[0.0, 0.0, 0.0])
    gen, _ = ts.generator_ref(method, st, before, [], CFG["std_factor"])
    mean, std = ts.f32(gen["mean"][0]), ts.f32(gen["std"][0])
    g, _ = published_view(method, mean, std, st, CFG["std_factor"])
    g["g_reco"], g["g_trav"] = loss_scales(CFG, *(scales or (st["n_valid"][0], R)), D)
    bw = backward_ref(fw, x64, y64, yv, method, g, CFG, **bad)
    p1 = {k: st[k][0] for k in ("sum_lr", "sum_lr2", "sum_raw", "n_valid", "n_rows")}
    p1.update(reserved=0.0, x_min=ts.f32(st["x_min"][0]), x_max=ts.f32(st["x_max"][0]))
    conf = torch.full((R + 7,), SENTINEL)
    conf[:R] = bw["conf"][0].float()
    p2 = dict(cg_mean=mean, cg_std=std, var=1.0, running=[0.0, 0.0, 0.0], conf=conf,
              grads=flat_grads(bw, 0).float(), trav_w=bw["trav_w"][0].item())
    rec = dict(before=before, p1=p1, p2=p2)
    if corrupt is not None:
        corrupt(rec)
    grads = rec["p2"]["grads"].double()
    (p, _), (mm, _), (vv, _) = ts.adam_ref(P, grads, before["m"], before["v"], 1, ts.f32(CFG["lr"]), ts.f32(0.9),
                                           ts.f32(0.999), ts.f32(CFG["eps"]))
    with np.errstate(all="ignore"):
        lreco = ts.f32(np.float64(p1["sum_lr"]) / p1["n_valid"])
        ltrav = ts.f32(np.float64(p1["sum_raw"]) / p1["n_rows"])
        ltc = ts.f32(np.float64(p2["trav_w"]) / p1["n_rows"])
    metrics = [ts.f32(ts.f32(0.03) * ltc + ts.f32(0.5) * lreco), ltrav, lreco, ltc, mean, std]
    rec["after"] = dict(params=p.float().double(), m=mm.float().double(), v=vv.float().double(), step=1,
                        metrics=metrics)
    return rec, x, y, yv, fw, bw


def _check(rec, x, y, yv):
    check_step("ctrl", rec, x, y, yv, 384, 64, 32, need=False)


def _rejects(rec, x, y, yv, tag):
    """The checker rejects the record, and the check that rejects it is the one the corruption is for (its tag)."""
    with pytest.raises(AssertionError, match=f"^{tag}"):
        _check(rec, x, y, yv)


def _labelled(R, i):
    return int(rows(R, 384, 9, device="cpu")[2].nonzero()[i])


def _unlabelled(R, i):
    return int((~rows(R, 384, 9, device="cpu")[2]).nonzero()[i])


CTRL_R = [1024, 4096]


@pytest.mark.parametrize("R", CTRL_R)
def test_checker_accepts_a_correct_step(R):
    rec, x, y, yv, _, _ = fake_record(R)
    _check(rec, x, y, yv)


@pytest.mark.parametrize("R", CTRL_R)
def test_checker_rejects_a_labelled_row_dropped_from_every_sum(R):
    """One labelled row left out of the statistic sums, Σ raw·w and every gradient sum (a live bound one row short):
    the fp64 statistics reject it first."""
    i = _labelled(R, R // 40)
    rec, x, y, yv, _, _ = fake_record(R, drop_stats=[i], drop=[i])
    _rejects(rec, x, y, yv, "dm_")


@pytest.mark.parametrize("R", CTRL_R)
def test_checker_rejects_a_labelled_row_dropped_from_the_gradients(R):
    """The same row left out of the gradient sums only: the gradient checks alone reject it."""
    i = _labelled(R, R // 40)
    rec, x, y, yv, _, _ = fake_record(R, drop=[i])
    _rejects(rec, x, y, yv, "dm_d")


def _row_term_over_bound(R, i):
    """The largest |term of row i| / bound over every gradient element of a correct record."""
    _, x, _, _, fw, bw = fake_record(R)
    worst = 0.0
    for k in (0, 1):
        rw, N = bw["rows"][k], fw["net"][k]
        for (lw, lb), dz, a in ((("W3", "b3"), rw["dz3"], N["a2"]), (("W2", "b2"), rw["dz2"], N["a1"]),
                                (("W1", "b1"), rw["dz1"], x.double())):
            worst = max(worst, ((dz[i][:, None] * a[i][None, :]).abs() / rw["grads"][lw][1].clamp_min(1e-300)).max(),
                        (dz[i].abs() / rw["grads"][lb][1].clamp_min(1e-300)).max())
    return float(worst)


@pytest.mark.parametrize("R", CTRL_R)
def test_checker_rejects_an_unlabelled_row_dropped_from_the_gradients(R):
    """An unlabelled row enters only net 0's gradients, through its traversability term g_trav (1 - conf) (t - y)
    t (1 - t), and Σ raw·w (net 1 reads no unlabelled row).  Net 0's sums are made of such terms only, so the row
    shows: its largest term is 25 times its bound at R = 1024 and 3.5 times at R = 4096 (net 0's dW2).  (In the
    SimpleMLP step the same row is below resolution, next to the labelled rows' reconstruction terms.)"""
    i = _unlabelled(R, R // 40)
    assert _row_term_over_bound(R, i) > 1
    rec, x, y, yv, _, _ = fake_record(R, drop=[i])
    _rejects(rec, x, y, yv, "dm_d")


@pytest.mark.parametrize("R", CTRL_R)
def test_checker_rejects_swapped_first_layer_weight_gradients(R):
    """networks.0.0.weight's gradient block exchanged with networks.1.0.weight's (the same shape)."""
    k = 64 * 384
    o1 = sum(v for v in (64 * 384, 64, 32 * 64, 32, 32, 1))

    def swap(rec):
        g = rec["p2"]["grads"].clone()
        g[:k], g[o1:o1 + k] = rec["p2"]["grads"][o1:o1 + k], rec["p2"]["grads"][:k]
        rec["p2"]["grads"] = g

    rec, x, y, yv, _, _ = fake_record(R, corrupt=swap)
    _rejects(rec, x, y, yv, "dm_dW1")


@pytest.mark.parametrize("R", CTRL_R)
def test_checker_rejects_a_bias_gradient_one_row_short(R):
    """Net 0's layer-2 bias gradient (a kBiasGrad column sum) summed over n_live - 1 rows: the last row's term is
    15 times that sum's bound at R = 1024 and 7.1 times at R = 4096.  Not every bias sum resolves one row: net 0's
    layer-3 bias (the column sum of dOut_0) holds the same row's term at 1.9 times its bound at R = 1024 but 0.96
    times at R = 4096, so at 4096 rows a row missing from that sum alone would pass."""
    rec, x, y, yv, _, _ = fake_record(R, short_db=(0, "b2"))
    _rejects(rec, x, y, yv, "dm_db2.0")


@pytest.mark.parametrize("R", CTRL_R)
def test_checker_rejects_g_trav_over_n_valid(R):
    n = int(rows(R, 384, 9, device="cpu")[2].sum())
    rec, x, y, yv, _, _ = fake_record(R, scales=(n, n))
    _rejects(rec, x, y, yv, "dm_d")


@pytest.mark.parametrize("R", CTRL_R)
def test_checker_rejects_g_reco_over_n_rows(R):
    rec, x, y, yv, _, _ = fake_record(R, scales=(R, R))
    _rejects(rec, x, y, yv, "dm_d")


@pytest.mark.parametrize("R", CTRL_R)
def test_checker_rejects_the_conf_weight_on_a_labelled_row(R):
    rec, x, y, yv, _, _ = fake_record(R, w_on=[_labelled(R, R // 40)])
    _rejects(rec, x, y, yv, "dm_")


@pytest.mark.parametrize("R", CTRL_R)
def test_checker_rejects_one_wrong_conf(R):
    def bump(rec):
        rec["p2"]["conf"][_unlabelled(R, 3)] += 1e-3

    rec, x, y, yv, _, _ = fake_record(R, corrupt=bump)
    _rejects(rec, x, y, yv, "dm_conf")


@pytest.mark.parametrize("R", CTRL_R)
def test_checker_rejects_relu_masks_of_the_other_network(R):
    rec, x, y, yv, _, _ = fake_record(R, swap_masks=True)
    _rejects(rec, x, y, yv, "dm_d")


@pytest.mark.parametrize("R", CTRL_R)
def test_checker_rejects_a_param_four_ulps_off(R):
    rec, x, y, yv, _, _ = fake_record(R)
    p = rec["after"]["params"]
    v = np.float32(p[777])
    for _ in range(4):
        v = np.nextafter(v, np.float32(np.inf))
    p[777] = float(v)
    _rejects(rec, x, y, yv, "dm_adam_p")
