"""The LinearRnvp train step (csrc/flow_train.cu) phase by phase against a one-step float64 reference: the NLL
statistics, the ConfidenceGenerator update, the per-row confidence, every element of the 24 gradient tensors and Adam,
at every tile, tail and live-row geometry of the shared fp32 GEMM (csrc/train_core.cu) and the flow's row kernels.

ops.FlowTrainer.step runs by phase_mask 1, 2 and 4 and the state is read in between:
  after 1  metrics (loss, n), cg_mean / cg_std, var and the running sums (bound to test tensors with set_confidence)
           and the confidence of every live row in compacted order;
  after 2  the flat gradient, in parameters() order (coupling 0 s, coupling 0 t, coupling 2 s, coupling 2 t; each
           Linear 0, 2, 4 weight then bias);
  after 4  params, exp_avg, exp_avg_sq and the step counter.
Every step's reference starts from the kernel's own state before that step (params, moments, step counter, generator
state), so every step is held to a one-step bound.  Three steps per case, so running_mean, kalman_filter and
moving_average carry state; the test keeps its own float64 copy of moving_average's window.

Bound: first order, on magnitudes, in float64, u = 2^-24.  A sum of n fp32 terms with S = sum |terms| gets
acc(n, S) = (C_FLOW n + 2) u S, as in test_train_step_gpu.py.

Departure from the MLP test's worst-case rule: errors of inputs are carried through W in quadrature, sqrt(e^2 W^2),
treating the roundings as independent, where the MLP test carries them through |W|.  So what this module checks is
an estimate of the error, not a bound on it.  The reason: each layer of |W| carries the bound's ratio to the value up
by about sqrt(K) (16x per layer at D = 384, h = 200), and the flow's gradients of coupling 0 lie twelve products deep.
Carried through |W|, the NLL's bound was 2.8 % of the NLL (median row, c = 0.01) and the bias gradients' 8e4 times
their value, and not one negative control showed.  In quadrature they are 8e-7 and ~1e-4 (c = 0.01), and the controls
below are rejected, at the sizes their docstrings give.  What an estimate costs:
  - the ReLU mask margin AMB is set from measurement, not derived: with 16 times a unit's bound, two dW2 elements of the
    D = 90, h = 200 case were one row's term off on the H100 (a mask the estimate did not count as ambiguous); AMB = 64;
  - C_FLOW's margin over the measured "c needed" holds for the weights, inputs and seeds measured here, not for every
    input: another model or batch may need a larger C_FLOW.
  net layer       z = a W^T + b: e_z = sqrt(e_a^2 W^2^T) + acc(K + 1, (|a| + e_a) |W|^T + |b|); ReLU is 1-Lipschitz
  s = tanh(so)    e_s = e_so + 4 u |s|               (1-Lipschitz, tanhf within 2 ulp)
  exp(s)          relative e_s + 4 u
  coupling        x = mu + (1 - m)(u e^s + t): e = m e_u + (1 - m)(e_u e^s + |u| e_es + e_t + 2 u |u e^s| + u |u e^s + t|)
  log-det         sqrt(sum (1 - m) e_s^2) + acc(D, sum (1 - m) |s|), + u |ld| per coupling
  NLL             sum z^2 / 2 + D log sqrt(2 pi) - log_det: sqrt(sum z^2 e_z^2) + (acc(D, S) + 3 u S) + e_ld + u (S + |ld|)
                  + u |nll|, S = sum (z^2 / 2 + log sqrt(2 pi))
  permutation     exact
  statistics      the NLL sums over the live rows accumulate in double: the row bounds in quadrature
  backward        dz = z / n, dld = -1 / n (1 / n rounded: relative u), dx = dz[invp] (next coupling: du[invp]),
                  gx = (1 - m) dx, dt = gx, ds = gx u e^s + (1 - m) dld, dso = ds (1 - s^2) where (1 - s^2) carries
                  2 |s| e_s + 2 u (absolute: relative would blow up where tanh saturates);
                  du = (1 - m) dx e^s + m (dx + dmu_s + dmu_t);  data gradients d = (dO W) [z > 0] as the forward,
                  a unit whose float64 pre-activation lies within AMB = 64 times its bound of 0 may take either mask
  weight grads    dW = dO^T A, db = sum dO over the n live rows: sqrt(e_dO^2^T A^2) + sqrt(dO^2^T e_A^2)
                  + acc(n, |dO|^T |A|)
  conf            L e_nll + 8 u, L the method's Lipschitz constant, from lo / hi derived from the kernel's published
                  mean / std (3 u of slack; moving_average's clipped extrema from the float64 extrema)
  Adam            test_train_step_gpu.adam_ref on the kernel's own gradient.
Entries whose bound is 0 (the weight-gradient columns of masked-out inputs, the last layers' rows of masked-out
outputs, sums over no rows) must be exactly equal, which is what a zero bound asserts.

C_FLOW is measured as C_TRAIN was: the bound is affine in c to first order, so (|err| - bound at c = 0) / (bound -
bound at c = 0) * c is the smallest c that covers an element; its maximum over a check is its "c needed", printed at
the end of the module (pytest -s) with the worst error / bound, and recorded in DESIGN.md §4.

NaN: with n = 0 (mean of an empty set) or n = 1 (std of one element) the reference's generator produces NaN; the
kernel's loss, generator and confidence must be NaN in exactly the same places, and its gradients finite.

The CPU section (no gpu mark) checks the explicit float64 reference against oracle/linear_rnvp.train_step's autograd
gradients and holds the negative controls: each corrupts a correct result in one place and the checker must reject it.
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
from test_linear_rnvp_gpu import _model  # noqa: E402

U = 2.0 ** -24
# accumulator constant of acc(n, S).  Measured over this module on one H100 80GB HBM3 (700 W), the largest c needed
# is 0.030 (dW2 at D = 90, h = 200, 1025 rows); 0.15 keeps a 5x margin, and every negative control is still rejected
C_FLOW = 0.15
METHODS = ts.METHODS
CFG = dict(std_factor=0.5, lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
LOG_SQRT_2PI = math.log(math.sqrt(2 * math.pi))
LAYERS = ("W0", "b0", "W2", "b2", "W4", "b4")
SENTINEL = 12345.0
# a ReLU unit whose float64 pre-activation lies within AMB times its bound of 0 may take either mask: the carried
# errors are root-sum-square estimates, not worst cases (module docstring), so the mask test gets a wide margin; it
# widens only the bounds that unit feeds
AMB = 64.0


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    tags = {k: v for k, v in edges._WORST.items() if k.startswith("fl_")}
    if tags:
        print(f"\nflow train step, worst error / bound at c = {C_FLOW} (c needed: the smallest c covering every element):")
        for tag in sorted(tags):
            need = ts._NEED.get(tag)
            print(f"  {tag:20s} {tags[tag][0]:.4f}   c needed {need[0] if need else 0.0:.4f}   "
                  f"worst at {ts._WHERE.get(tag, (0, '-'))[1]}")


def _one(v):
    return torch.tensor(v, dtype=torch.float64)


def check(got, ref, bound, tag, b0=None):
    ts.check(got, ref, bound, tag, b0, c=C_FLOW)


# ------------------------------------------------------------------------------------------------ float64 reference
def acc(n, S, c):
    return (c * n + 2) * U * S


def rss(e, W):
    """Carried errors e through the matrix W, added in quadrature: sqrt(e^2 W^2)."""
    return (e * e @ (W * W)).sqrt()


def rss_sum(e, dim):
    return (e * e).sum(dim).sqrt()


def unflat(P, D, h):
    """The flat parameter vector -> [coupling 0 s, coupling 0 t, coupling 2 s, coupling 2 t], each {layer: view}."""
    nets, o = [], 0
    for _ in range(4):
        net = {}
        for name, shape in zip(LAYERS, ((h, D), (h,), (h, h), (h,), (D, h), (D,))):
            k = math.prod(shape)
            net[name] = P[o:o + k].view(shape)
            o += k
        nets.append(net)
    return nets


def buffers(model, device):
    f = model.flows
    return dict(m=[f[0].mask.to(device, torch.float64), f[2].mask.to(device, torch.float64)],
                p=[f[1].p.to(device), f[3].p.to(device)], invp=[f[1].invp.to(device), f[3].invp.to(device)])


def _net_fwd(net, mu, e_mu, c):
    W0, b0, W2, b2, W4, b4 = (net[k] for k in LAYERS)
    D, h = W0.shape[1], W0.shape[0]
    z1 = mu @ W0.T + b0
    e_z1 = rss(e_mu, W0.T) + acc(D + 1, (mu.abs() + e_mu) @ W0.abs().T + b0.abs(), c)
    a1 = torch.relu(z1)
    z2 = a1 @ W2.T + b2
    e_z2 = rss(e_z1, W2.T) + acc(h + 1, (a1 + e_z1) @ W2.abs().T + b2.abs(), c)
    a2 = torch.relu(z2)
    o = a2 @ W4.T + b4
    e_o = rss(e_z2, W4.T) + acc(h + 1, (a2 + e_z2) @ W4.abs().T + b4.abs(), c)
    return dict(z1=z1, e_z1=e_z1, a1=a1, z2=z2, e_z2=e_z2, a2=a2, o=o, e_o=e_o)


def forward_ref(P, x, bufs, D, h, c=C_FLOW):
    """Both couplings, the permutations and the per-row NLL in float64, each value with its bound.  x: the live rows."""
    nets = unflat(P, D, h)
    u, e_u = x, torch.zeros_like(x)
    ld, e_ld = x.new_zeros(x.shape[0]), x.new_zeros(x.shape[0])
    cpl = []
    for ci in (0, 1):
        m = bufs["m"][ci]
        om = 1 - m
        mu, e_mu = u * m, e_u * m
        ns, nt = _net_fwd(nets[2 * ci], mu, e_mu, c), _net_fwd(nets[2 * ci + 1], mu, e_mu, c)
        s = torch.tanh(ns["o"])
        e_s = ns["e_o"] + 4 * U * s.abs()
        es = torch.exp(s)
        e_es = es * (e_s + 4 * U)
        ue = u * es
        xs = mu + om * (ue + nt["o"])
        e_xs = m * e_u + om * (e_u * es + u.abs() * e_es + nt["e_o"] + 2 * U * ue.abs() + U * (ue + nt["o"]).abs())
        ld = ld + (om * s).sum(1)
        e_ld = e_ld + rss_sum(om * e_s, 1) + acc(D, (om * s.abs()).sum(1), c) + U * ld.abs()
        cpl.append(dict(m=m, u=u, e_u=e_u, mu=mu, e_mu=e_mu, s=s, e_s=e_s, es=es, e_es=e_es, nets=(ns, nt)))
        u, e_u = xs[:, bufs["p"][ci]], e_xs[:, bufs["p"][ci]]
    sq = u * u / 2 + LOG_SQRT_2PI
    S = sq.sum(1)
    nll = S - ld
    e_nll = (rss_sum(u * e_u, 1) + acc(D, S, c) + 3 * U * S + e_ld + U * (S + ld.abs()) + U * nll.abs())
    return dict(nets=nets, cpl=cpl, z=u, e_z=e_u, nll=nll, e_nll=e_nll)


def _relu_back(da, e_da, z, e_z):
    on, amb = z > 0, z.abs() <= AMB * e_z
    dz = torch.where(on, da, torch.zeros_like(da))
    e_dz = torch.where(on, e_da, torch.zeros_like(da)) + torch.where(amb, da.abs() + e_da, torch.zeros_like(da))
    return dz, e_dz


def backward_ref(fw, bufs, c=C_FLOW, inv_n=None, dld_sign=1.0, perm=False, drop=None):
    """The 24 gradient tensors (in parameters() order) of mean_r NLL_r, each with its bound, and the per-row data
    gradients of every net.  Negative controls: inv_n (in place of 1 / n), dld_sign, perm (read p where the backward
    reads invp), drop (row indices left out of every weight-gradient sum)."""
    z, e_z = fw["z"], fw["e_z"]
    n = z.shape[0]
    g = (1.0 / n if n else float("inf")) if inv_n is None else inv_n
    e_g = U * g
    dld = -g * dld_sign
    keep = torch.ones(n, dtype=z.dtype, device=z.device)
    if drop is not None:
        keep[drop] = 0
    grads, rows = [None] * 4, {}
    du = e_du = None
    for ci in (1, 0):
        C = fw["cpl"][ci]
        m, s, e_s, es, e_es = C["m"], C["s"], C["e_s"], C["es"], C["e_es"]
        om = 1 - m
        ip = bufs["p" if perm else "invp"][ci]
        if ci == 1:
            src, e_src = z * g, e_z * g + z.abs() * e_g + U * (z * g).abs()
        else:
            src, e_src = du, e_du
        dx, e_dx = src[:, ip], e_src[:, ip]
        gx, e_gx = om * dx, om * e_dx
        ue = C["u"] * es
        e_ue = C["e_u"] * es + C["u"].abs() * e_es
        ds = gx * ue + om * dld
        e_ds = gx.abs() * e_ue + e_gx * ue.abs() + om * e_g + 3 * U * (gx * ue).abs() + 2 * U * om * abs(dld)
        one_s2 = 1 - s * s
        dso = ds * one_s2
        e_dso = e_ds * one_s2 + ds.abs() * (2 * s.abs() * e_s + 2 * U) + U * dso.abs()
        dmu = []
        for k, (dO, e_dO) in enumerate(((dso, e_dso), (gx, e_gx))):
            N, W = C["nets"][k], fw["nets"][2 * ci + k]
            D, h = W["W0"].shape[1], W["W0"].shape[0]
            da2 = dO @ W["W4"]
            d2, e_d2 = _relu_back(da2, rss(e_dO, W["W4"]) + acc(D, dO.abs() @ W["W4"].abs(), c), N["z2"], N["e_z2"])
            da1 = d2 @ W["W2"]
            d1, e_d1 = _relu_back(da1, rss(e_d2, W["W2"]) + acc(h, d2.abs() @ W["W2"].abs(), c), N["z1"], N["e_z1"])
            out = {}
            for (lw, lb), dz, e_dz, a, e_a in ((("W4", "b4"), dO, e_dO, N["a2"], N["e_z2"]),
                                               (("W2", "b2"), d2, e_d2, N["a1"], N["e_z1"]),
                                               (("W0", "b0"), d1, e_d1, C["mu"], C["e_mu"])):
                dzk, e_dzk = dz * keep[:, None], e_dz * keep[:, None]
                out[lw] = (dzk.T @ a, rss(e_dzk.T, a) + rss(dzk.T, e_a) + acc(n, dzk.abs().T @ a.abs(), c))
                out[lb] = (dzk.sum(0), rss_sum(e_dzk, 0) + acc(n, dzk.abs().sum(0), c))
            grads[2 * ci + k] = out
            rows[(ci, k)] = dict(dO=dO, d2=d2, d1=d1)
            if ci == 1:
                dmu.append((d1 @ W["W0"], rss(e_d1, W["W0"]) + acc(h, d1.abs() @ W["W0"].abs(), c)))
        if ci == 1:
            (ms, e_ms), (mt, e_mt) = dmu
            du = om * dx * es + m * (dx + ms + mt)
            e_du = (om * (e_dx * es + dx.abs() * e_es + 2 * U * (dx * es).abs())
                    + m * (e_dx + e_ms + e_mt + 2 * U * (dx.abs() + ms.abs() + mt.abs())))
    return dict(grads=grads, rows=rows)


def flat_grads(bw, i):
    """Value (i = 0) or bound (i = 1) of every gradient as one vector in parameters() order."""
    return torch.cat([bw["grads"][q][k][i].reshape(-1) for q in range(4) for k in LAYERS])


def stats_ref(fw):
    v, e = fw["nll"], fw["e_nll"]
    n = v.numel()
    s1, s2 = v.sum().item(), (v * v).sum().item()
    emax = e.max().item() if n else 0.0
    return dict(n_valid=(float(n), 0.0), sum_lr=(s1, rss_sum(e, 0).item() + 2.0 ** -50 * abs(s1)),
                sum_lr2=(s2, rss_sum(2 * v * e, 0).item() + (e * e).sum().item() + 2.0 ** -50 * s2),
                x_min=(v.min().item() if n else float("inf"), emax), x_max=(v.max().item() if n else -float("inf"), emax))


def conf_ref(method, fw, st, mean, std, f):
    """The confidence of every live row from the kernel's published mean / std -> (conf, bound)."""
    m, sd = np.float64(mean), np.float64(std)
    with np.errstate(all="ignore"):
        if method == "kalman_filter":
            lo, hi, cmin, cmax, e_lohi = m, 1 / (sd * f), 0.0, 0.0, 0.0
        elif method == "moving_average":
            lo, hi = m - 2 * sd, m + 2 * sd
            e_lohi = 3 * U * (abs(m) + 2 * abs(sd))
            cmin = float(np.fmin(np.fmax(st["x_min"][0], lo), hi))
            cmax = float(np.fmin(np.fmax(st["x_max"][0], lo), hi))
            e_lohi = max(e_lohi, st["x_min"][1])
        else:
            lo, hi = float(np.fmax(m + sd * f - sd, 0.0)), m + sd * f + sd
            cmin = cmax = 0.0
            e_lohi = 3 * U * (abs(m) + (f + 1) * abs(sd))
    conf, L = ts.row_conf_ref(method, fw["nll"], float(lo), float(hi), cmin, cmax)
    return conf, L * (fw["e_nll"] + 3 * e_lohi) + 8 * U


# ------------------------------------------------------------------------------------------------ the checker
def check_step(tag, rec, x, yv, bufs, D, h, method="latest_measurement", window=None, where="", need=True):
    """Every phase of one recorded step against the float64 reference started from the kernel's state before it.
    rec: what Flow.run read (or fake_record made).  need: also take the reference at c = 0, for "c needed".
    Returns moving_average's new window."""
    b, dev = rec["before"], x.device
    P = b["params"].to(dev)
    xl = x[yv].double()
    n, f = xl.shape[0], CFG["std_factor"]
    ts._CTX[0] = f"{tag} {method} D={D} h={h} R={x.shape[0]} n={n} {where}".strip()
    fw = forward_ref(P, xl, bufs, D, h)
    fw0 = forward_ref(P, xl, bufs, D, h, c=0.0) if need else None
    st = stats_ref(fw)
    p1 = rec["p1"]
    met = p1["metrics"]
    # ---- phase 1: loss, generator, confidence
    assert met[3] == n, f"{tag}: metrics[3] = {met[3]}, {n} live rows"
    assert met[1] == 0 and met[2] == 0, f"{tag}: loss_trav / loss_reco {met[1:3]}"
    with np.errstate(all="ignore"):
        loss = float(np.float64(st["sum_lr"][0]) / n)
        e_loss = float(np.float64(st["sum_lr"][1]) / n) + U * abs(loss)
        e_loss0 = (float(np.float64(stats_ref(fw0)["sum_lr"][1]) / n) + U * abs(loss)) if need else None
    check(_one([met[0]]), _one([loss]), _one([e_loss]), "fl_loss", None if e_loss0 is None else _one([e_loss0]))
    gen, window = ts.generator_ref(method, st, b, window or [], f)
    check(_one([p1["cg_mean"]]), _one([gen["mean"][0]]), _one([gen["mean"][1]]), "fl_gen_mean")
    if not (method == "running_mean" and abs(gen["var"][0]) <= gen["var"][1] and math.isnan(p1["cg_std"])):
        # running_mean's var = sum_sq / n - mean^2 with mean in fp32: a variance of 0 within its bound (one labelled row
        # so far) may round below 0, and its sqrtf is NaN, as in the reference's float32 generator
        check(_one([p1["cg_std"]]), _one([gen["std"][0]]), _one([gen["std"][1]]), "fl_gen_std")
    ts.same(met[4], p1["cg_mean"], f"{tag}: metrics mean")
    ts.same(met[5], p1["cg_std"], f"{tag}: metrics std")
    if "var" in gen:
        check(_one([p1["var"]]), _one([gen["var"][0]]), _one([gen["var"][1]]), "fl_gen_var")
    if method == "running_mean":
        assert p1["running"][0] == gen["running_n"][0], f"{tag}: running_n {p1['running'][0]}"
        for i, k in ((1, "running_sum"), (2, "running_sumsq")):
            check(_one([p1["running"][i]]), _one([gen[k][0]]), _one([gen[k][1]]), f"fl_gen_{k}")
    conf, e_conf = conf_ref(method, fw, st, p1["cg_mean"], p1["cg_std"], f)
    e_conf0 = conf_ref(method, fw0, stats_ref(fw0), p1["cg_mean"], p1["cg_std"], f)[1] if need else None
    check(p1["conf"][:n], conf, e_conf, "fl_conf", e_conf0)
    assert bool((p1["conf"][n:x.shape[0]] == SENTINEL).all()), f"{tag}: conf written past the {n} live rows"
    # ---- phase 2: every gradient element
    bw = backward_ref(fw, bufs)
    bw0 = backward_ref(fw0, bufs, c=0.0) if need else None
    grads = rec["grads"].to(dev).double()
    assert bool(torch.isfinite(grads).all()), f"{tag}: non-finite gradient"
    o = 0
    for q in range(4):
        for k in LAYERS:
            ref, bound = bw["grads"][q][k]
            sz = ref.numel()
            check(grads[o:o + sz].view(ref.shape), ref, bound, f"fl_d{k}", bw0["grads"][q][k][1] if need else None)
            o += sz
    assert o == grads.numel()
    # ---- phase 4: Adam on the kernel's own gradient
    a = rec["after"]
    assert a["step"] == b["step"] + 1, f"{tag}: step counter {b['step']} -> {a['step']}"
    b1, b2 = (ts.f32(v) for v in CFG["betas"])
    (p, e_p), (mm, e_m), (vv, e_v) = ts.adam_ref(P, grads, b["m"].to(dev), b["v"].to(dev), a["step"], ts.f32(CFG["lr"]),
                                                 b1, b2, ts.f32(CFG["eps"]))
    check(a["m"], mm, e_m, "fl_adam_m")
    check(a["v"], vv, e_v, "fl_adam_v")
    check(a["params"], p, e_p, "fl_adam_p")
    return window


# ------------------------------------------------------------------------------------------------ the GPU driver
class Flow:
    """ops.FlowTrainer driven phase by phase, with its generator state in tensors the test can read."""

    def __init__(self, model, max_rows, method="latest_measurement"):
        from wild_visual_navigation_b200 import ops

        self.model = model
        self.tr = ops.FlowTrainer(model, max_rows=max_rows, std_factor=CFG["std_factor"], lr=CFG["lr"],
                                  betas=CFG["betas"], eps=CFG["eps"])
        self.var = torch.ones(1, 1, device="cuda")
        self.running = torch.zeros(3, dtype=torch.float64, device="cuda")
        self.tr.set_confidence(METHODS[method], self.var, self.running[0:1], self.running[1:2], self.running[2:3])

    def state(self):
        tr = self.tr
        return dict(params=self.model.flat_params.double().clone(), m=tr.exp_avg.double().clone(),
                    v=tr.exp_avg_sq.double().clone(), step=int(tr.step_counter.item()), cg_mean=tr.cg_mean.item(),
                    cg_std=tr.cg_std.item(), var=self.var.item(), running=self.running.tolist())

    def run(self, x, yv):
        tr, rec = self.tr, {}
        tr._reserve(x.shape[0])
        rec["before"] = self.state()
        tr.conf.fill_(SENTINEL)   # conf is written at the live rows only
        tr.step(x, yv, phase_mask=1)
        rec["p1"] = dict(metrics=tr.metrics.tolist(), cg_mean=tr.cg_mean.item(), cg_std=tr.cg_std.item(),
                         var=self.var.item(), running=self.running.tolist(), conf=tr.conf.clone())
        tr.step(x, yv, phase_mask=2)
        rec["grads"] = tr.grads.clone()
        tr.step(x, yv, phase_mask=4)
        rec["after"] = self.state()
        return rec


ROWS = [1, 63, 64, 65, 130, 1025, 4096]
LABELS = ["all", "most", "one", "none"]


def inputs(R, D, seed, labels, scale=1.0, device="cuda"):
    """x ~ 0.5 N(0, 1) with about 1 % of rows x20 (tanh saturates, e^s ~ e); y_valid all set, ~60 % set, exactly one
    set, or none set."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R, D, generator=g) * 0.5 * scale
    x[torch.arange(R) % 100 == 37] *= 20
    if labels == "all":
        yv = torch.ones(R, dtype=torch.bool)
    elif labels == "most":
        yv = torch.rand(R, generator=g) < 0.6
    elif labels == "one":
        yv = torch.zeros(R, dtype=torch.bool)
        yv[R // 3] = True
    else:
        yv = torch.zeros(R, dtype=torch.bool)
    return x.to(device), yv.to(device)


def run_steps(tag, D, h, mask, method, steps, max_rows=None, seed=0):
    """steps: [(R, labels, scale)] on one trainer, each checked."""
    m = _model(D, h, mask, seed=42 + seed)
    T = Flow(m, max_rows or max(R for R, _, _ in steps), method)
    bufs, window = buffers(m, "cuda"), []
    for s, (R, labels, scale) in enumerate(steps):
        x, yv = inputs(R, D, 1000 * seed + 10 * s + R, labels, scale)
        rec = T.run(x, yv)
        window = check_step(tag, rec, x, yv, bufs, D, h, method, window, where=f"step {s} {labels}")
    return T


# ------------------------------------------------------------------------------------------------ GPU: geometry
@pytest.mark.gpu
@pytest.mark.parametrize("R", ROWS)
@pytest.mark.parametrize("method", list(METHODS))
@pytest.mark.parametrize("mask", ["odds", "half"])
def test_shipped_shape(mask, method, R):
    """LinearRnvp(384, [200]): an N tail of 8 on h (200 = 3 * 64 + 8), six M tiles on D.  Rows 1 (one block), 63 / 64
    / 65 around a 64-row tile, 130 (three tiles), 1025 (the compaction's threads scan two rows each; n > 256 in the
    statistics kernel), 4096.  Three steps with the labelled fractions rotating, so every fraction meets every
    method and step position over the row list."""
    i = ROWS.index(R)
    steps = [(R, LABELS[(i + s) % 4], 1.0) for s in range(3)]
    run_steps("shipped", 384, 200, mask, method, steps, seed=i)


GEOMETRY = [
    (90, 200, "odds"),     # STEGO code width: tails in M, N and K (90 = 64 + 26; K = 90 ends in a 10-wide chunk)
    (768, 256, "half"),    # ViT-B tokens: exact tiles, as a control
    (33, 8, "half"),       # odd D with the half mask (16 ones, 17 zeros); minimum hidden width
    (2, 8, "odds"),        # minimum D: one live input column per coupling
    (1030, 512, "odds"),   # maximum hidden width; D > 1024: the coupling kernels loop nine times
]


@pytest.mark.gpu
@pytest.mark.parametrize("D,h,mask", GEOMETRY, ids=[f"{d}x{h}-{m}" for d, h, m in GEOMETRY])
def test_geometry(D, h, mask):
    """Three steps: n_live well below the grid (the live row bound of the forward and data-gradient products, the live
    K bound of the weight-gradient products), then every row live with several K chunks and gy blocks in the bias
    sums, then a small batch."""
    run_steps("geometry", D, h, mask, "running_mean", [(1025, "most", 1.0), (4096, "all", 1.0), (65, "most", 1.0)])


@pytest.mark.gpu
def test_stale_rows_past_n_live():
    """4096 rows all labelled with x x8, then 37 of 4096 labelled on the same handle: the workspace rows past n_live
    hold large stale activations and gradients, which no product may read."""
    D, h = 384, 200
    m = _model(D, h, "odds")
    T, bufs = Flow(m, 4096), buffers(m, "cuda")
    x, yv = inputs(4096, D, 77, "all", scale=8.0)
    check_step("stale", T.run(x, yv), x, yv, bufs, D, h, where="all x8")
    x, _ = inputs(4096, D, 78, "none")
    yv = torch.zeros(4096, dtype=torch.bool, device="cuda")
    yv[torch.randperm(4096, generator=torch.Generator().manual_seed(79))[:37].cuda()] = True
    check_step("stale", T.run(x, yv), x, yv, bufs, D, h, where="37 of 4096")


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["moving_average", "kalman_filter"])
def test_growth_mid_sequence(method):
    """A handle made for 64 rows, then batches above max_rows: the handle is replaced twice, and the generator (the
    window inside the handle, the bound var) and Adam's state carry over."""
    T = run_steps("growth", 384, 200, "odds", method,
                  [(50, "all", 1.0), (1025, "most", 1.0), (200, "most", 1.0), (4096, "most", 1.0), (90, "all", 1.0)],
                  max_rows=64)
    assert T.tr.max_rows >= 4096


@pytest.mark.gpu
def test_bit_reproducible():
    """Two trainers on the same model and inputs give bit-identical gradients, parameters, confidence and metrics
    (DESIGN.md §9.12: every output element is summed in a fixed order)."""
    outs = []
    for _ in range(2):
        m = _model(384, 200, "odds")
        T = Flow(m, 4096, "moving_average")
        recs = [T.run(*inputs(4096, 384, 5 + s, "most")) for s in range(2)]
        outs.append((recs, m.flat_params.clone(), T.tr.exp_avg.clone(), T.tr.exp_avg_sq.clone()))
    (ra, pa, ma, va), (rb, pb, mb, vb) = outs
    for a, b in zip(ra, rb):
        assert torch.equal(a["grads"], b["grads"])
        assert torch.equal(a["p1"]["conf"], b["p1"]["conf"])
        assert a["p1"]["metrics"] == b["p1"]["metrics"]
    assert torch.equal(pa, pb) and torch.equal(ma, mb) and torch.equal(va, vb)


# ------------------------------------------------------------------------------------------------ CPU: the reference
@pytest.mark.parametrize("D,h,R", [(6, 8, 20), (33, 16, 40), (2, 8, 11)])
@pytest.mark.parametrize("mask", ["odds", "half"])
def test_reference_matches_autograd(D, h, R, mask):
    """forward_ref / backward_ref against oracle/linear_rnvp.train_step (autograd) in float64: the NLL, every gradient
    element to 1e-12 of its tensor's largest, and the bounds finite and non-negative.  Rows x20 saturate tanh."""
    from oracle import linear_rnvp as orn
    from oracle.wvn_path import ConfidenceState

    m = _model(D, h, mask, device="cpu")
    sd = {k: (v.detach().double() if v.is_floating_point() else v) for k, v in m.state_dict().items()}
    x, _ = inputs(R, D, D + R, "all", device="cpu")
    x[1] *= 20
    x = x.double()
    _, grads, loss, _ = orn.train_step(sd, {}, x, ConfidenceState(0.5, "latest_measurement"))
    bufs = buffers(m, "cpu")
    P = m.flat_params.detach().double()
    fw = forward_ref(P, x, bufs, D, h)
    assert (fw["nll"] - orn.nll(sd, x)).abs().max().item() <= 1e-12 * (1 + fw["nll"].abs().max().item())
    assert abs(fw["nll"].mean().item() - loss.item()) <= 1e-12 * (1 + abs(loss.item()))
    mine = flat_grads(backward_ref(fw, bufs), 0)
    want = torch.cat([g.reshape(-1) for g in grads.values()])
    assert [n for n, _ in m.named_parameters()] == list(grads)
    o = 0
    for name, g in grads.items():
        k = g.numel()
        err = (mine[o:o + k] - g.reshape(-1)).abs().max().item()
        assert err <= 1e-12 * g.abs().max().item() + 1e-300, (name, err)
        o += k
    assert o == want.numel()
    bound = flat_grads(backward_ref(fw, bufs), 1)
    assert bool(torch.isfinite(bound).all()) and bool((bound >= 0).all())


def fake_record(D, h, R, seed, mask="odds", method="latest_measurement", labels="most", corrupt=None, **bad):
    """A correct record built from the float64 reference rounded to fp32, as Flow.run would read it from a kernel that
    computes the step exactly.  bad: backward_ref's negative-control options; corrupt(grads, bw) -> grads changes the
    flat gradient.  Either way Adam is then applied to the gradient as recorded, as the kernel's Adam consumes the
    kernel's own gradient, so a corrupted gradient can only show in the gradient checks."""
    m = _model(D, h, mask, device="cpu")
    bufs = buffers(m, "cpu")
    x, yv = inputs(R, D, seed, labels, device="cpu")
    P = m.flat_params.detach().double()
    fw = forward_ref(P, x[yv].double(), bufs, D, h)
    st = stats_ref(fw)
    n = fw["nll"].numel()
    before = dict(params=P, m=torch.zeros_like(P), v=torch.zeros_like(P), step=0, cg_mean=0.0, cg_std=1.0, var=1.0,
                  running=[0.0, 0.0, 0.0])
    gen, _ = ts.generator_ref(method, st, before, [], CFG["std_factor"])
    mean, std = ts.f32(gen["mean"][0]), ts.f32(gen["std"][0])
    conf = torch.full((R,), SENTINEL)
    conf[:n] = conf_ref(method, fw, st, mean, std, CFG["std_factor"])[0].float()
    with np.errstate(all="ignore"):
        loss = ts.f32(np.float64(st["sum_lr"][0]) / n)
    p1 = dict(metrics=[loss, 0.0, 0.0, float(n), mean, std], cg_mean=mean, cg_std=std,
              var=ts.f32(gen["var"][0]) if "var" in gen else 1.0, running=[0.0, 0.0, 0.0], conf=conf)
    bw = backward_ref(fw, bufs, **bad)
    grads = flat_grads(bw, 0).float()
    if corrupt is not None:
        grads = corrupt(grads, bw)
    (p, _), (mm, _), (vv, _) = ts.adam_ref(P, grads.double(), before["m"], before["v"], 1, ts.f32(CFG["lr"]),
                                           ts.f32(0.9), ts.f32(0.999), ts.f32(CFG["eps"]))
    after = dict(params=p.float().double(), m=mm.float().double(), v=vv.float().double(), step=1)
    rec = dict(before=before, p1=p1, grads=grads, after=after)
    return rec, x, yv, bufs, bw


CTRL = dict(D=384, h=200, R=1024, seed=9)


def _check(rec, x, yv, bufs):
    check_step("ctrl", rec, x, yv, bufs, 384, 200, need=False)


def _rejects(rec, x, yv, bufs, tag):
    """The checker rejects the record, and the check that rejects it is the one the corruption is for (its tag)."""
    with pytest.raises(AssertionError, match=f"^{tag}"):
        _check(rec, x, yv, bufs)


def _offset(q, layer, D=384, h=200):
    """Offset of net q's layer in the flat vector."""
    sizes = dict(W0=h * D, b0=h, W2=h * h, b2=h, W4=D * h, b4=D)
    per = sum(sizes.values())
    return q * per + sum(sizes[k] for k in LAYERS[:LAYERS.index(layer)])


@pytest.mark.parametrize("R", [1024, 4096])
def test_checker_accepts_a_correct_step(R):
    rec, x, yv, bufs, _ = fake_record(**dict(CTRL, R=R))
    _check(rec, x, yv, bufs)


@pytest.mark.parametrize("R", [1024, 4096])
def test_checker_rejects_one_missing_row(R):
    """One labelled row left out of every weight-gradient sum (a live bound one row short).  It shows in the last
    layers' sums: in dW4 of every net one row's term exceeds the bound at 1341 to 6310 elements for R = 1024 and at
    207 to 5533 for R = 4096.  Coupling 0's s-net first-layer sums (dW0, db0) cannot resolve it on their own: there
    the term is at most 0.36 (R = 1024) and 0.03 (R = 4096) times the bound."""
    _, _, yv, _, _ = fake_record(**dict(CTRL, R=R))
    rec, x, yv, bufs, _ = fake_record(**dict(CTRL, R=R), drop=[int(yv.sum()) // 2])
    _rejects(rec, x, yv, bufs, "fl_d")


def test_checker_rejects_a_flipped_log_det_gradient():
    rec, x, yv, bufs, _ = fake_record(**CTRL, dld_sign=-1.0)
    _rejects(rec, x, yv, bufs, "fl_d")


def test_checker_rejects_p_read_for_invp():
    rec, x, yv, bufs, _ = fake_record(**CTRL, perm=True)
    _rejects(rec, x, yv, bufs, "fl_d")


def test_checker_rejects_swapped_s_and_t_gradients():
    k = _offset(1, "W0")
    rec, x, yv, bufs, _ = fake_record(**CTRL, corrupt=lambda g, bw: torch.cat([g[k:2 * k], g[:k], g[2 * k:]]))
    _rejects(rec, x, yv, bufs, "fl_d")


@pytest.mark.parametrize("R", [1024, 4096])
def test_checker_rejects_a_bias_gradient_over_one_row_fewer(R):
    """Coupling 2's t-net second-layer bias gradient (the kBiasGrad column sum) summed over n - 1 of the n live rows.
    The last row's term is 101 times that sum's bound at R = 1024 and 2.8 times at R = 4096.  Not every bias sum can
    resolve one row: for coupling 0's s-net first-layer bias the term is 0.40 times its bound at R = 1024 and 0.02
    times at R = 4096, so a missing row there would pass."""
    o = _offset(3, "b2")

    def drop_last(g, bw):
        g = g.clone()
        g[o:o + 200] = (bw["grads"][3]["b2"][0] - bw["rows"][(1, 1)]["d2"][-1]).float()
        return g

    rec, x, yv, bufs, _ = fake_record(**dict(CTRL, R=R), corrupt=drop_last)
    _rejects(rec, x, yv, bufs, "fl_db2")


def test_checker_rejects_one_over_n_minus_one():
    n = int(inputs(CTRL["R"], CTRL["D"], CTRL["seed"], "most", device="cpu")[1].sum())
    rec, x, yv, bufs, _ = fake_record(**CTRL, inv_n=1.0 / (n - 1))
    _rejects(rec, x, yv, bufs, "fl_d")


def test_checker_rejects_one_wrong_conf():
    rec, x, yv, bufs, _ = fake_record(**CTRL)
    rec["p1"]["conf"][7] += 1e-3
    _rejects(rec, x, yv, bufs, "fl_conf")
