"""The fused online train step (mlp_train_fused.cu) phase by phase against a one-step float64 reference: statistics,
ConfidenceGenerator update, per-row confidence, every gradient element, the confidence-weighted traversability sum,
Adam and the loss metrics, at every tile, split-K and padding geometry the kernels have.

Parameters after Adam cannot show a gradient's size: Adam's step does not change when a gradient is scaled by a
positive constant, and at step 1 it is lr * sign(g).  So the step runs by phase_mask 1, 2 and 4 (as ops.MlpTrainer
does without a library communicator) and the state is read in between:
  after 1  the FusedScalars (sum_lr, sum_lr2, sum_raw, n_valid, n_rows, x_min, x_max);
  after 2  mean, std, lo, hi, cmin, cmax, g_reco, g_trav, the generator state, conf per row, the flat gradient and
           the weighted traversability sum riding at its end (dOut is held through db3, its column sums);
  after 4  params, exp_avg, exp_avg_sq, metrics, and the scalars, which must be left clean bit for bit.
Every step's reference starts from the kernel's own state before that step (params, moments, step counter, generator
state), so every step is held to a one-step bound.  moving_average's window lives inside the trainer; the test keeps
the oracle's window of float64 (n, sum, sum of squares) triples, each entry with its loss bound.

Two levels, as the pixel-head test uses the kernel's own blend weights:
  (a) statistics and generator update (mean, std, var, running sums, lo / hi, cmin / cmax, extrema) against float64
      computed from float64 losses;
  (b) conf and every gradient against float64 computed from the kernel's published lo / hi / cmin / cmax / g_reco /
      g_trav (latest_measurement publishes only mean / std: lo / hi are derived from those, with 3 u of slack), so a
      1-ulp difference in std cannot show up as a gradient failure.

Bound: first order, on magnitudes, in float64, u = 2^-24.  A product or sum of n fp32 terms with S = sum |terms| gets
acc(n, S) = (C_TRAIN n + 2) u S; the + 2 covers the last roundings when n is small.  Errors of inputs are carried
through |W| and |a|:
  z1 = x W1^T + b1      e_z1 = acc(D + 1, |x||W1|^T + |b1|)                   (x and W are exact)
  z2 = a1 W2^T + b2     e_z2 = e_a1 |W2|^T + acc(h1 + 1, ...)    a = ReLU(z) is 1-Lipschitz: e_a = e_z
  z3 = a2 W3^T + b3     e_z3 = e_a2 |W3|^T + acc(h2 + 1, ...)
  trav = sigmoid(z3_0)  1/4 e_z3_0 + 6 u trav                     |sigmoid'| <= 1/4, expf + two roundings
  loss_reco = mean_d (rec - x)^2: the squares carry 2 |df| (e_rec + u |df|); their row sum (warp shuffles, then
                        shared-memory atomics in any order) gets the worst case D u sum df^2; then / D
  raw = (trav - y)^2    2 |dt| (e_trav + u |dt|) + u raw
  stats                 sums of the row bounds over the rows (the double accumulation adds < 2^-50 relative)
  conf                  L e_loss + 8 u, L the method's Lipschitz constant: 1 / (hi - lo), 1 / (cmax - cmin), or
                        hi e^-1/2 for the Kalman filter's exp(-z^2 / 2); clamps are 1-Lipschitz
  dOut_0 = g_trav w (t - y) t (1 - t): |d/dt| <= 1/4 + |t - y| |1 - 2t|; w = 1 - conf carries e_conf
  dOut_d = g_reco (rec - x)
  dH2 = (dOut W3) [z2 > 0]: e_dOut |W3| + acc(n3, |dOut||W3|); dH1 likewise over h2
  dW = dZ^T A, db = sum dZ over the R live rows: e_dZ^T |A| + |dZ|^T e_A + acc(R, |dZ|^T |A|), for any order of the
                        split-K atomics
  ReLU masks            a (row, unit) whose float64 pre-activation lies within its own bound of 0 may take either
                        mask: |dz| + e_dz of that row is added to its dz bound, and so to every gradient it feeds
  trav_w_sum            the row terms' bounds + (atomics + 2) u S, atomics = 8 per 32-row tile (R for the legacy path)
  Adam (torch's lerp form, fed the kernel's own gradient): m 3 u (|m0| + (1 - b1) |g - m0|); v 3 u v;
                        p: (lr / bc1 / denom) e_m + |update| (e_v / 2v + 8 u) + u |p|, i.e. a few ulp of p.
C_TRAIN is measured: the bound is affine in c to first order, so for every element (|err| - bound at c = 0) /
(bound - bound at c = 0) * c is the smallest c that covers it.  Over this module on one H100 80GB HBM3 (700 W) that is
0 at every element of every check: the + 2 floor and the terms carried from it already cover the real errors.
C_TRAIN = 0.01 keeps a margin above that.  The whole chain scales with c, so a larger c would blind the checks: at
c = 0.1 a dW1 element could be ~3 % of its magnitude sum off.  At c = 0.01 and 3200 rows the negative controls show the
bound rejects one missing labelled row and a conf error of 1e-3.  One missing unlabelled row is below resolution: its
dOut is only the traversability term g_trav w (t - y) t (1 - t), far below S / 3200 of the labelled rows' terms.

NaN: with n_valid = 0 (mean of an empty set) or 1 (std of one element) the reference produces NaN; the kernel's
metrics, conf and gradients must be NaN in exactly the same places.

The CPU section (no gpu mark) checks the float64 reference against oracle/wvn_path.train_step run in float64 and
holds the negative controls: each corrupts a correct result in one place and asserts that the checker rejects it.
Worst error / bound per check is printed at the end of the module (pytest -s) and recorded in DESIGN.md §4.
"""
import math
import os
import sys
from ctypes import byref, c_void_p

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_kernel_edges_gpu as edges  # noqa: E402

U = 2.0 ** -24
_NEED = {}       # tag -> (the smallest c that covers every element seen, where its worst element was)
_CTX = [""]      # what the current check_step is checking (test, method, step)
_WHERE = {}      # tag -> (worst error / bound, where)
# accumulator constant of acc(n, S).  Measured over this module on one H100 80GB HBM3 (700 W), the smallest c that
# covers every element of every check is 0 (the + 2 floor and the carried terms suffice); 0.01 keeps a margin above
# that and still rejects one missing labelled row in 3200 (DESIGN.md §4)
C_TRAIN = 0.01
METHODS = {"latest_measurement": 0, "running_mean": 1, "kalman_filter": 2, "moving_average": 3}
CFG = dict(w_trav=0.03, w_reco=0.5, std_factor=0.5, anomaly_balanced=True, lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
KF_Q, KF_R = float(np.float32(0.2)), float(np.float32(1.0))
SC_D = ["sum_lr", "sum_lr2", "sum_raw", "n_valid", "n_rows", "reserved", "x_min", "x_max"]
SC_F = ["mean", "std", "loss_total", "loss_trav", "loss_reco", "loss_trav_conf", "lo", "hi", "cmin", "cmax", "g_reco",
        "g_trav"]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    tags = {k: v for k, v in edges._WORST.items() if k.startswith("ts_")}
    if tags:
        print(f"\nfused train step, worst error / bound at c = {C_TRAIN} (c needed: the smallest c covering every element):")
        for tag in sorted(tags):
            r = tags[tag][0]
            need = _NEED.get(tag)
            print(f"  {tag:24s} {r:.4f}   c needed {need[0] if need else 0.0:.4f}   worst at {_WHERE.get(tag, (0, '-'))[1]}")


def f32(v):
    """The fp32 value of a double (numpy keeps the rounding mode of the kernels: round to nearest even)."""
    return float(np.float32(v))


def _t(v, like):
    return torch.as_tensor(v, dtype=torch.float64, device=like.device)


def check(got, ref, bound, tag, b0=None, c=C_TRAIN):
    """NaN in exactly the same places, every other element within its bound (edges.assert_within records the ratio).
    b0: the same bound at c = 0, bound itself being taken at c.  The bound is affine in c to first order, so
    (|err| - b0) / (bound - b0) * c is the smallest c that covers the element: its maximum is recorded as the c this
    check needs."""
    got, ref = torch.as_tensor(got).double(), torch.as_tensor(ref).double()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=ref.device).expand_as(ref)
    got = got.to(ref.device)
    gn, rn = torch.isnan(got), torch.isnan(ref)
    if not torch.equal(gn, rn):
        idx = tuple(int(i) for i in (gn != rn).nonzero()[0])
        raise AssertionError(f"{tag}: NaN in different places ({int((gn != rn).sum())} elements); first at {idx}: "
                             f"got {got[idx].item()} ref {ref[idx].item()}")
    ok = ~rn
    edges.assert_within(got[ok], ref[ok], bound[ok], tag)
    if bool(ok.any()):
        r = ((got[ok] - ref[ok]).abs() / bound[ok].clamp_min(1e-300))
        if r.max().item() >= _WHERE.get(tag, (0.0, ""))[0]:
            _WHERE[tag] = (r.max().item(), f"{_CTX[0]}, element {int(ok.nonzero()[int(r.argmax())][-1])}")
    if b0 is not None and bool(ok.any()):
        b0 = torch.as_tensor(b0, dtype=torch.float64, device=ref.device).expand_as(ref)[ok]
        err, span = (got[ok] - ref[ok]).abs(), (bound[ok] - b0).clamp_min(1e-300)
        need = ((err - b0).clamp_min(0) / span) * c
        i = int(need.argmax())
        if need[i].item() > _NEED.get(tag, (0.0, ""))[0]:
            _NEED[tag] = (need[i].item(), f"{_CTX[0]} element {i}")


def _one(v):
    return torch.tensor(v, dtype=torch.float64)


def same(a, b, tag):
    """Bit-identical fp32 values (NaN equal to NaN)."""
    a, b = np.float32(a), np.float32(b)
    assert (a == b) or (np.isnan(a) and np.isnan(b)), f"{tag}: {a!r} != {b!r}"


# ------------------------------------------------------------------------------------------------ float64 reference
def unflat(P, D, h1, h2):
    out, o = [], 0
    for shape in ((h1, D), (h1,), (h2, h1), (h2,), (D + 1, h2), (D + 1,)):
        n = math.prod(shape)
        out.append(P[o:o + n].view(shape))
        o += n
    return out


def acc(n, S, c):
    return (c * n + 2) * U * S


def forward_ref(P, x, y, D, h1, h2, c=C_TRAIN):
    """SimpleMLP.forward + the per-row loss terms in float64, each value with its bound (module docstring)."""
    W1, b1, W2, b2, W3, b3 = unflat(P, D, h1, h2)
    r = {}
    z1 = x @ W1.T + b1
    e_z1 = acc(D + 1, x.abs() @ W1.abs().T + b1.abs(), c)
    a1 = z1.clamp_min(0)
    z2 = a1 @ W2.T + b2
    e_z2 = e_z1 @ W2.abs().T + acc(h1 + 1, (a1 + e_z1) @ W2.abs().T + b2.abs(), c)
    a2 = z2.clamp_min(0)
    z3 = a2 @ W3.T + b3
    e_z3 = e_z2 @ W3.abs().T + acc(h2 + 1, (a2 + e_z2) @ W3.abs().T + b3.abs(), c)
    t = torch.sigmoid(z3[:, 0])
    e_t = 0.25 * e_z3[:, 0] + 6 * U * t
    rec, e_rec = z3[:, 1:], e_z3[:, 1:]
    df = rec - x
    sq = df * df
    lr = sq.mean(1)
    e_lr = ((2 * df.abs() * (e_rec + U * df.abs())).sum(1) + D * U * sq.sum(1)) / D + U * lr
    dt = t - y
    raw = dt * dt
    e_raw = 2 * dt.abs() * (e_t + U * dt.abs()) + U * raw
    r.update(W1=W1, W2=W2, W3=W3, z1=z1, e_z1=e_z1, a1=a1, z2=z2, e_z2=e_z2, a2=a2, t=t, e_t=e_t, rec=rec,
             e_rec=e_rec, lr=lr, e_lr=e_lr, raw=raw, e_raw=e_raw)
    return r


def stats_ref(fw, yv):
    lr, e = fw["lr"], fw["e_lr"]
    v = yv
    return dict(
        n_valid=(float(v.sum()), 0.0), n_rows=(float(lr.numel()), 0.0),
        sum_lr=(lr[v].sum().item(), e[v].sum().item() + 2.0 ** -50 * lr[v].sum().item()),
        sum_lr2=((lr * lr)[v].sum().item(), (2 * lr * e + e * e)[v].sum().item() + 2.0 ** -50 * (lr * lr)[v].sum().item()),
        sum_raw=(fw["raw"].sum().item(), fw["e_raw"].sum().item() + 2.0 ** -50 * fw["raw"].sum().item()),
        x_min=(lr.min().item(), e.max().item()), x_max=(lr.max().item(), e.max().item()))


def _lohi(m, em, sd, esd, f):
    """latest_measurement / running_mean: lo = max(m + f sd - sd, 0), hi = m + f sd + sd (fmaxf ignores NaN)."""
    r = 3 * U * (abs(m) + (f + 1) * sd)
    e = em + (f + 1) * esd + r
    return (float(np.fmax(m + f * sd - sd, 0.0)), e), (m + f * sd + sd, e)


def _sample_stats(n, s1, e1, s2, e2):
    """mean and unbiased std of n samples from their sums: (m, em), (sd, esd)."""
    with np.errstate(all="ignore"):
        n, s1, s2 = np.float64(n), np.float64(s1), np.float64(s2)
        m = s1 / n
        var = (s2 - n * m * m) / (n - 1.0)
        sd = np.sqrt(max(var, 0.0)) if n > 1 else np.float64("nan")
        em = e1 / n + U * abs(m)
        evar = (e2 + 2 * abs(m) * e1) / (n - 1.0) + 2.0 ** -50 * (s2 + n * m * m) / (n - 1.0)
        esd = evar / (2 * sd) + U * sd
    return (float(m), float(em)), (float(sd), float(esd))


def generator_ref(method, st, before, window, f):
    """ConfidenceGenerator.update (utils/confidence_generator.py:78-145) in float64 from the float64 sums of this step
    and the kernel's generator state before it -> {name: (value, bound)}, the new window."""
    n, _ = st["n_valid"]
    s1, e1 = st["sum_lr"]
    s2, e2 = st["sum_lr2"]
    out = {}
    if method == "latest_measurement":
        (m, em), (sd, esd) = _sample_stats(n, s1, e1, s2, e2)
        out["lo"], out["hi"] = _lohi(m, em, sd, esd, f)
    elif method == "running_mean":
        rn0, rs0, rq0 = before["running"]
        rn, rs, rq = rn0 + n, rs0 + s1, rq0 + s2
        with np.errstate(all="ignore"):   # rn = 0 (no labelled row yet): NaN, as 0 / 0 in the kernel
            m = float(np.float64(rs) / rn)
            var = float(np.float64(rq) / rn - m * m)
            em = float(e1 / np.float64(rn)) + U * abs(m)
            evar = float((e2 + 2 * abs(m) * e1) / np.float64(rn) + 3 * U * m * m + U * abs(var)
                         + 2.0 ** -50 * rq / np.float64(rn))
            sd = math.sqrt(var) if var >= 0 else float("nan")
            esd = float(evar / (2 * np.float64(sd))) + U * sd
        out.update(var=(var, evar), running_n=(rn, 0.0), running_sum=(rs, e1 + 2.0 ** -50 * abs(rs)),
                   running_sumsq=(rq, e2 + 2.0 ** -50 * rq))
        out["lo"], out["hi"] = _lohi(m, em, sd, esd, f)
    elif method == "kalman_filter":
        s0, cov0 = before["cg_mean"], before["var"]
        if n > 0:
            meas = s1 / n
            e_meas = e1 / n + U * abs(meas)
            cov = cov0 + KF_Q
            gain = cov / (cov + KF_R)
            e_gain = 4 * U * gain
            m = s0 + gain * (meas - s0)
            em = gain * e_meas + abs(meas - s0) * e_gain + 3 * U * (abs(s0) + gain * abs(meas - s0) + abs(m))
            var = (1 - gain) * cov
            evar = cov * e_gain + 3 * U * var + U * cov
        else:
            m, em, var, evar = s0, 0.0, cov0, 0.0
        sd = math.sqrt(var)
        esd = evar / (2 * sd) + U * sd
        out.update(var=(var, evar), lo=(m, em), hi=(1 / (sd * f), esd / (sd * sd * f) + 2 * U / (sd * f)))
    else:
        window = (window + [(n, s1, s2, e1, e2)])[-5:]
        N, S1, S2, E1, E2 = (sum(w[i] for w in window) for i in range(5))
        (m, em), (sd, esd) = _sample_stats(N, S1, E1, S2, E2)
        e = em + 2 * esd + 3 * U * (abs(m) + 2 * sd)
        lo, hi = m - 2 * sd, m + 2 * sd
        out.update(lo=(lo, e), hi=(hi, e))
        xm, ex = st["x_min"], st["x_max"]
        with np.errstate(all="ignore"):
            out["cmin"] = (float(np.fmin(np.fmax(xm[0], lo), hi)), max(xm[1], e))
            out["cmax"] = (float(np.fmin(np.fmax(ex[0], lo), hi)), max(ex[1], e))
    out["mean"], out["std"] = (m, em), (sd, esd)
    return out, window


def row_conf_ref(method, lr, lo, hi, cmin, cmax):
    """train_bwd_rows' row_confidence in float64 on the kernel's (fp32) lo / hi / cmin / cmax, with fmaxf / fminf
    semantics (a NaN bound is ignored) -> conf, Lipschitz constant in the loss."""
    lo, hi, cmin, cmax = (_t(v, lr) for v in (lo, hi, cmin, cmax))
    if method == "kalman_filter":
        z = (lr - lo) * hi
        return torch.where(lr < lo, torch.ones_like(lr), torch.exp(-z * z * 0.5)), hi.abs() * math.exp(-0.5)
    xc = torch.fmin(torch.fmax(lr, lo), hi)
    if method == "moving_average":
        return (xc - cmin) / (cmax - cmin), 1 / (cmax - cmin).abs()
    return 1 - (xc - lo) / (hi - lo), 1 / (hi - lo).abs()


def backward_ref(fw, x, y, yv, method, g, cfg, e_lohi=0.0, rel_g=0.0, c=C_TRAIN):
    """conf, dOut, the six gradient blocks and the weighted traversability sum in float64, with bounds.  g: lo, hi,
    cmin, cmax, g_reco, g_trav as the kernel has them (e_lohi / rel_g: their slack when derived, not read)."""
    conf, L = row_conf_ref(method, fw["lr"], g["lo"], g["hi"], g["cmin"], g["cmax"])
    e_conf = L * (fw["e_lr"] + 3 * e_lohi) + 8 * U
    full = yv | (not cfg["anomaly_balanced"])
    wgt = torch.where(full, torch.ones_like(conf), 1 - conf)
    e_wgt = torch.where(full, torch.zeros_like(conf), e_conf)
    t, e_t = fw["t"], fw["e_t"]
    q = (t - y) * t * (1 - t)
    e_q = (0.25 + (t - y).abs() * (1 - 2 * t).abs()) * e_t
    gt, gr = g["g_trav"], g["g_reco"]
    d0 = gt * wgt * q
    e_d0 = gt * (e_wgt * q.abs() + wgt * e_q) + (6 * U + 2 * rel_g) * d0.abs()
    dr = torch.where(yv[:, None], gr * (fw["rec"] - x), torch.zeros_like(x))
    e_dr = torch.where(yv[:, None], gr * fw["e_rec"] + (2 * U + 2 * rel_g) * dr.abs(), torch.zeros_like(x))
    dz3, e_dz3 = torch.cat([d0[:, None], dr], 1), torch.cat([e_d0[:, None], e_dr], 1)
    W2, W3 = fw["W2"], fw["W3"]
    R, n3, h2 = x.shape[0], W3.shape[0], W3.shape[1]

    def relu_back(da, e_da, z, e_z):
        on, amb = z > 0, z.abs() <= e_z
        dz = torch.where(on, da, torch.zeros_like(da))
        e_dz = torch.where(on, e_da, torch.zeros_like(da)) + torch.where(amb, da.abs() + e_da, torch.zeros_like(da))
        return dz, e_dz

    da2 = dz3 @ W3
    e_da2 = e_dz3 @ W3.abs() + acc(n3, dz3.abs() @ W3.abs(), c)
    dz2, e_dz2 = relu_back(da2, e_da2, fw["z2"], fw["e_z2"])
    da1 = dz2 @ W2
    e_da1 = e_dz2 @ W2.abs() + acc(h2, dz2.abs() @ W2.abs(), c)
    dz1, e_dz1 = relu_back(da1, e_da1, fw["z1"], fw["e_z1"])
    grads = {}
    for name, dz, e_dz, a, e_a in (("w3", dz3, e_dz3, fw["a2"], fw["e_z2"]), ("w2", dz2, e_dz2, fw["a1"], fw["e_z1"]),
                                   ("w1", dz1, e_dz1, x, None)):
        ref = dz.T @ a
        S = dz.abs().T @ a.abs()
        prop = e_dz.T @ a.abs() + (dz.abs().T @ e_a if e_a is not None else 0)
        grads[name] = (ref, prop + acc(R, S, c))
        b = "b" + name[1]
        Sb = dz.abs().sum(0)
        grads[b] = (dz.sum(0), e_dz.sum(0) + acc(R, Sb, c))
    tw = (fw["raw"] * wgt).sum()
    return dict(conf=(conf, e_conf), grads=grads, dz3=dz3, dz1=dz1,
                trav_w=(tw, (fw["e_raw"] * wgt + fw["raw"] * e_wgt).sum() + U * (fw["raw"] * wgt).abs().sum()))


def adam_ref(p0, g, m0, v0, t, lr, b1, b2, eps):
    """torch.optim.Adam (lerp form, no weight decay) in float64 on the kernel's fp32 operands -> (p, m, v) with bounds."""
    m = m0 + (g - m0) * (1 - b1)
    v = v0 * b2 + (1 - b2) * g * g
    bc1, bc2s = 1 - b1 ** t, math.sqrt(1 - b2 ** t)
    denom = v.sqrt() / bc2s + eps
    upd = lr / bc1 * m / denom
    p = p0 - upd
    e_m = 3 * U * (m0.abs() + (1 - b1) * (g - m0).abs())
    e_v = 3 * U * v
    rel_den = torch.where(v > 0, e_v / (2 * v), torch.zeros_like(v)) + 4 * U
    e_p = lr / bc1 * e_m / denom + upd.abs() * (rel_den + 4 * U) + 2 * U * p.abs()
    return (p, e_p), (m, e_m), (v, e_v)


# ------------------------------------------------------------------------------------------------ the checker
def check_step(tag, rec, x, y, yv, D, h1, h2, method="latest_measurement", cfg=CFG, window=None, legacy=False,
               where=""):
    """Every phase of one recorded step against the float64 reference started from the kernel's state before it.
    rec: what the driver read (Trainer.run / fake_record).  Returns moving_average's new window."""
    b, dev = rec["before"], x.device
    P, x64, y64 = b["params"].to(dev), x.double(), y.double()
    _CTX[0] = f"{tag} {method} D={D} h={h1}/{h2} R={x.shape[0]} {where}".strip()
    fw, fw0 = forward_ref(P, x64, y64, D, h1, h2), forward_ref(P, x64, y64, D, h1, h2, c=0.0)
    st, st0 = stats_ref(fw, yv), stats_ref(fw0, yv)
    sc1, sc2 = rec["sc1"], rec["sc2"]
    # ---- (a) statistics and the generator update, from the float64 losses
    keys = ["sum_lr", "sum_lr2", "sum_raw", "n_valid"] + ([] if legacy else ["n_rows", "x_min", "x_max"])
    for k in keys:
        check(_one([sc1[k]]), _one([st[k][0]]), _one([st[k][1]]), f"ts_{tag}_{k}", _one([st0[k][1]]))
    gen, window = generator_ref(method, st, b, window or [], cfg["std_factor"])
    for k in ("mean", "std") + (() if method == "latest_measurement" else ("lo", "hi")) + (
            ("cmin", "cmax") if method == "moving_average" else ()):
        check(_one([sc2[k]]), _one([gen[k][0]]), _one([gen[k][1]]), f"ts_gen_{k}")
    st2 = rec["gen_after"]
    same(st2["cg_mean"], sc2["mean"], f"{tag}: cg_mean")
    same(st2["cg_std"], sc2["std"], f"{tag}: cg_std")
    if "var" in gen:
        check(_one([st2["var"]]), _one([gen["var"][0]]), _one([gen["var"][1]]), "ts_gen_var")
    if method == "running_mean":
        for i, k in enumerate(("running_n", "running_sum", "running_sumsq")):
            check(_one([st2["running"][i]]), _one([gen[k][0]]), _one([gen[k][1]]), f"ts_gen_{k}")
    n, nr = sc1["n_valid"], sc1.get("n_rows", float(x.shape[0]))
    # ---- (b) conf, dOut and the gradients, from the kernel's own published generator values
    if method == "latest_measurement":
        m, sd, f = sc2["mean"], sc2["std"], cfg["std_factor"]
        with np.errstate(all="ignore"):
            g = dict(lo=float(np.fmax(m + sd * f - sd, 0.0)), hi=m + sd * f + sd, cmin=0.0, cmax=0.0,
                     g_reco=cfg["w_reco"] * 2 / (np.float64(n) * D), g_trav=cfg["w_trav"] * 2 / nr)
        e_lohi, rel_g = 3 * U * (abs(m) + (f + 1) * abs(sd)), 3 * U
    else:
        g = {k: sc2[k] for k in ("lo", "hi", "cmin", "cmax", "g_reco", "g_trav")}
        e_lohi, rel_g = 0.0, 0.0
        if n:
            check(_one([g["g_reco"]]), _one([cfg["w_reco"] * 2 / (n * D)]), _one([3 * U * g["g_reco"]]), "ts_g_reco")
        check(_one([g["g_trav"]]), _one([cfg["w_trav"] * 2 / nr]), _one([3 * U * g["g_trav"]]),
              "ts_g_trav")
    bw = backward_ref(fw, x64, y64, yv, method, g, cfg, e_lohi, rel_g)
    bw0 = backward_ref(fw0, x64, y64, yv, method, g, cfg, e_lohi, rel_g, c=0.0)
    R = x.shape[0]
    check(rec["conf"][:R], bw["conf"][0], bw["conf"][1], f"ts_{tag}_conf", bw0["conf"][1])
    grads = rec["grads"].to(dev).double()
    np_ = P.numel()
    o = 0
    for name, shape in zip(("w1", "b1", "w2", "b2", "w3", "b3"), [v.shape for v in unflat(P, D, h1, h2)]):
        k = math.prod(shape)
        ref, bound = bw["grads"][name]
        check(grads[o:o + k].view(shape), ref, bound, f"ts_{tag}_d{name}", bw0["grads"][name][1])
        o += k
    tw_ref, tw_b = bw["trav_w"]
    atomics = R if legacy else 8 * ((rec["rows_padded"] + 31) // 32)
    tw_b = tw_b + (atomics + 2) * U * tw_ref.abs()
    tw_b0 = bw0["trav_w"][1] + (atomics + 2) * U * tw_ref.abs()
    check(grads[np_:np_ + 1], tw_ref.reshape(1), tw_b.reshape(1), f"ts_{tag}_trav_w", tw_b0.reshape(1))
    # ---- Adam on the kernel's own gradient
    a = rec["after"]
    assert a["step"] == b["step"] + 1, f"{tag}: step counter {b['step']} -> {a['step']}"
    b1, b2 = (f32(v) for v in cfg["betas"])
    m0, v0 = rec.get("adam_in", (b["m"], b["v"]))
    (p, e_p), (mm, e_m), (vv, e_v) = adam_ref(P, grads[:np_], m0.to(dev), v0.to(dev), a["step"], f32(cfg["lr"]), b1, b2,
                                              f32(cfg["eps"]))
    check(a["m"], mm, e_m, "ts_adam_m")
    check(a["v"], vv, e_v, "ts_adam_v")
    check(a["params"], p, e_p, "ts_adam_p")
    # ---- loss metrics from the kernel's own sums; the scalars left clean for the next step
    met = rec["metrics"]
    with np.errstate(all="ignore"):
        lreco = f32(np.float64(sc1["sum_lr"]) / n)
        ltrav = f32(np.float64(sc1["sum_raw"]) / nr)
        ltc = f32(np.float64(grads[np_].item()) / nr)
    same(met[2], lreco, f"{tag}: loss_reco")
    same(met[1], ltrav, f"{tag}: loss_trav")
    same(met[3], ltc, f"{tag}: loss_trav_confidence")
    tot = cfg["w_trav"] * ltc + cfg["w_reco"] * lreco
    check(_one([met[0]]), _one([tot]), _one([3 * U * (abs(cfg["w_trav"] * ltc) + abs(cfg["w_reco"] * lreco))]),
          "ts_loss_total")
    same(met[4], sc2["mean"], f"{tag}: metrics mean")
    same(met[5], sc2["std"], f"{tag}: metrics std")
    if not legacy:
        c = rec["sc4_bits"]
        assert c[6] == 0x7FF0000000000000 and c[7] == 0, f"{tag}: x_min / x_max not reset ({c[6]:#x}, {c[7]:#x})"
        assert all(c[i] == 0 for i in range(6)), f"{tag}: statistic sums not reset: {c[:6]}"
    return window


# ------------------------------------------------------------------------------------------------ the GPU driver
def make_params(D, h1, h2, seed=42):
    from oracle import wvn_path

    return torch.cat([v.reshape(-1) for v in wvn_path.mlp_init(D, (h1, h2), seed=seed).values()]).float()


def _read_scalars(sc):
    s = sc.detach().cpu()
    d = dict(zip(SC_D, s[:8].tolist()))
    d.update(zip(SC_F, s[8:14].view(torch.float32).tolist()))
    return d


class Trainer:
    """ops.MlpTrainer driven phase by phase with its generator state in tensors the test can read."""

    def __init__(self, P0, D, h1, h2, max_rows, method="latest_measurement", cfg=CFG, legacy=False):
        from wild_visual_navigation_b200 import ops

        self.cfg, self.method, self.legacy = cfg, method, legacy
        self.tr = ops.MlpTrainer(P0.cuda().clone(), D, h1, h2, max_rows=max_rows, w_trav=cfg["w_trav"],
                                 w_reco=cfg["w_reco"], std_factor=cfg["std_factor"],
                                 anomaly_balanced=cfg["anomaly_balanced"], lr=cfg["lr"], betas=cfg["betas"],
                                 eps=cfg["eps"], legacy=legacy)
        self.var = torch.ones(1, 1, device="cuda")
        self.running = torch.zeros(3, dtype=torch.float64, device="cuda")
        if not legacy:
            self.tr.set_confidence(METHODS[method], self.var, self.running[0:1], self.running[1:2], self.running[2:3])

    def state(self):
        tr = self.tr
        return dict(params=tr.params.double().clone(), m=tr.exp_avg.double().clone(), v=tr.exp_avg_sq.double().clone(),
                    step=int(tr.step_counter.item()), cg_mean=tr.cg_mean.item(), cg_std=tr.cg_std.item(),
                    var=self.var.item(), running=self.running.tolist())

    def run(self, x, y, yv, groups=1, rpg=None, n_rows=None, before_phase4=None):
        """One step by phase_mask 1, 2, 4; x is [groups * rpg, D] (padded per group when n_rows is given)."""
        from wild_visual_navigation_b200._C import check as ccheck, lib, ptr, stream

        tr, rec = self.tr, {}
        rpg = x.shape[0] if rpg is None else rpg
        rec["before"] = self.state()
        rec["rows_padded"] = groups * rpg
        if self.legacy:
            tr.step(x, y, yv)
            s = tr.scalars.cpu()
            rec["sc1"] = dict(zip(SC_D[:4], s[:4].tolist()))
            rec["sc2"] = dict(zip(SC_F[:2], s[5:8].view(torch.float32)[:2].tolist()))
        else:
            tr.conf.fill_(12345.0)   # conf is written at the compacted rows only
            x, y, yv = x.contiguous(), y.contiguous().float(), yv.contiguous().to(torch.uint8)

            def phase(mask):
                ccheck(lib().wvn_mlp_train_step(tr._h, ptr(tr.params), ptr(tr.exp_avg), ptr(tr.exp_avg_sq),
                                                ptr(tr.step_counter), ptr(x), groups, rpg, ptr(n_rows), ptr(y), ptr(yv),
                                                ptr(tr.cg_mean), ptr(tr.cg_std), ptr(tr.conf), ptr(tr.metrics), mask,
                                                stream()))

            phase(1)
            rec["sc1"] = _read_scalars(tr.scalars)
            phase(2)
            rec["sc2"] = _read_scalars(tr.scalars)
            if before_phase4 is not None:
                before_phase4(tr)
            rec["adam_in"] = (tr.exp_avg.double().clone(), tr.exp_avg_sq.double().clone())
            phase(4)
            rec["sc4_bits"] = tr.scalars.cpu().view(torch.int64).tolist()
        rec["conf"] = tr.conf.clone()
        rec["grads"] = tr.grads.clone()
        a = self.state()
        rec["gen_after"] = a
        rec["after"] = a
        rec["metrics"] = tr.metrics.tolist()
        return rec


def supervision(R, seed, p_valid=0.2, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    yv = torch.rand(R, generator=g) < p_valid
    yv[:2] = True
    y = torch.where(yv, torch.rand(R, generator=g).clamp(min=0.001), torch.zeros(R))
    return y.to(device), yv.to(device)


def features(R, D, seed, scale=1.0, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(R, D, generator=g) * scale).to(device)


def run_and_check(tag, D, h1, h2, R, steps=1, seed=0, method="latest_measurement", cfg=CFG, legacy=False, P0=None):
    P0 = make_params(D, h1, h2) if P0 is None else P0
    T = Trainer(P0, D, h1, h2, max_rows=max(R, 32), method=method, cfg=cfg, legacy=legacy)
    window = []
    for s in range(steps):
        x = features(R, D, seed + s)
        y, yv = supervision(R, seed + 100 + s)
        rec = T.run(x, y, yv)
        window = check_step(tag, rec, x, y, yv, D, h1, h2, method, cfg, window, legacy)
    return T


# ------------------------------------------------------------------------------------------------ GPU: geometry
@pytest.mark.gpu
@pytest.mark.parametrize("D", [384, 768, 90, 1024, 255, 256, 33])
def test_widths(D):
    """DINO, DINOv2-B, STEGO and the limit; n3 = 256 / 257 around layer 3's 256-thread pass; a 1-wide K-chunk tail."""
    run_and_check("width", D, 256, 32, R=1000, steps=2, seed=D)


@pytest.mark.gpu
@pytest.mark.parametrize("h1,h2", [(4, 1), (68, 31), (252, 17)])
def test_hidden_widths(h1, h2):
    """A partial layer-1 column group j, and lanes m >= h2 in layer 2 and dH2."""
    run_and_check("hidden", 384, h1, h2, R=700, steps=2, seed=h1)


@pytest.mark.gpu
@pytest.mark.parametrize("R", [1, 31, 32, 33, 127, 128, 129, 511, 512, 2047, 2048, 2049, 3200])
def test_compacted_rows(R):
    """Split-K 1 / 2 / 4 / 8, each with and without a partial last 16-row block, and 32-row tiles with a tail."""
    T = Trainer(make_params(384, 256, 32), 384, 256, 32, max_rows=max(R, 32))
    x = features(R, 384, R)
    y, yv = supervision(R, R + 1)    # R = 1: the one row is labelled, std is NaN and so is conf, the step stays finite
    yv[-1] = True                    # a split that stops short drops the last rows: make them weigh
    check_step("rows", T.run(x, y, yv), x, y, yv, 384, 256, 32)


@pytest.mark.gpu
def test_rejected_shapes():
    from wild_visual_navigation_b200 import ops
    from wild_visual_navigation_b200._C import TrainConfig, lib

    cfg = TrainConfig(0.03, 0.5, 0.5, 1, 1e-3, 0.9, 0.999, 1e-8)
    for D, h1, h2 in ((1025, 256, 32), (384, 258, 32), (384, 66, 32), (384, 256, 33), (384, 256, 0)):
        h = c_void_p()
        assert lib().wvn_mlp_trainer_create(D, h1, h2, 64, byref(cfg), None, None, byref(h)) != 0, (D, h1, h2)
        assert not h.value
    with pytest.raises(Exception):
        ops.MlpTrainer(torch.zeros(lib().wvn_mlp_param_count(1025, 256, 32), device="cuda"), 1025, 256, 32)


def _padded(G, rpg, counts, D, pad, seed):
    x = features(G * rpg, D, seed).view(G, rpg, D)
    for g, c in enumerate(counts):
        x[g, min(c, rpg):] = pad
    live = torch.cat([x[g, :min(c, rpg)] for g, c in enumerate(counts)])
    return x.reshape(G * rpg, D), live


@pytest.mark.gpu
@pytest.mark.parametrize("pad", [float("nan"), float("inf"), float("-inf")])
@pytest.mark.parametrize("rpg", [20, 100])
def test_padded_rows(rpg, pad):
    """[G, rpg, D] with 0, 1, rpg and more than rpg live rows per group (the clamp in compact_index and the live test
    in train_wgrad), 32-row tiles that straddle groups, padding rows holding NaN / Inf that must reach no output, and
    conf written at exactly the compacted rows."""
    G, D = 37, 384
    pattern = [rpg, 0, 1, rpg + 7, 3, rpg - 1, 13 % rpg + 2]
    counts = [pattern[g % len(pattern)] for g in range(G)]
    xp, live = _padded(G, rpg, counts, D, pad, rpg)
    R = live.shape[0]
    y, yv = supervision(G * rpg, rpg + 5)    # sized for every padded row, as HotPathStep passes them; R are live
    n_rows = torch.tensor(counts, dtype=torch.int32, device="cuda")
    T = Trainer(make_params(D, 256, 32), D, 256, 32, max_rows=G * rpg)
    window = []
    for s in range(2):
        rec = T.run(xp, y, yv, groups=G, rpg=rpg, n_rows=n_rows)
        window = check_step("padded", rec, live, y[:R], yv[:R], D, 256, 32, window=window)
        assert bool((rec["conf"][R:] == 12345.0).all()), "conf written past the compacted rows"


# ------------------------------------------------------------------------------------------------ GPU: labels, NaN
LABELS = ["all", "one", "two", "zero_y", "none", "none_unbalanced", "one_of_many", "mixed_unbalanced"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", LABELS)
def test_labels_and_nan_parity(case):
    """Every row labelled; one or two; labelled rows with y = 0; none (the reference's mean of an empty set is NaN);
    one among unlabelled rows (std of one element is NaN, so conf and the unlabelled rows' weights are NaN);
    anomaly_balanced off.  Metrics, conf and gradients must be NaN exactly where the reference's are."""
    R, D = 300, 384
    cfg = dict(CFG, anomaly_balanced=not case.endswith("unbalanced"))
    y, yv = supervision(R, 7)
    if case == "all":
        yv[:] = True
    elif case == "one":
        R = 1
        y, yv = y[:1], torch.ones(1, dtype=torch.bool, device="cuda")
    elif case == "two":
        R = 2
        y, yv = y[:2], torch.ones(2, dtype=torch.bool, device="cuda")
    elif case == "zero_y":
        y[yv.nonzero()[::2, 0]] = 0.0
    elif case.startswith("none"):
        yv[:] = False
    elif case == "one_of_many":
        yv[:] = False
        yv[17] = True
    y = torch.where(yv, y, torch.zeros_like(y))
    T = Trainer(make_params(D, 256, 32), D, 256, 32, max_rows=max(R, 32), cfg=cfg)
    x = features(R, D, 3)
    rec = T.run(x, y, yv)
    check_step("labels", rec, x, y, yv, D, 256, 32, cfg=cfg)
    nan_expected = case in ("none", "one_of_many")
    assert bool(torch.isnan(rec["grads"]).any()) == nan_expected, case
    assert math.isnan(rec["metrics"][0]) == (case.startswith("none") or case == "one_of_many"), case


# ------------------------------------------------------------------------------------------------ GPU: generator methods
@pytest.mark.gpu
@pytest.mark.parametrize("method", list(METHODS))
def test_confidence_methods(method):
    """Eight steps per method with a different row count and feature scale each step: moving_average's window wraps."""
    D = 384
    T = Trainer(make_params(D, 256, 32), D, 256, 32, max_rows=2400, method=method)
    window = []
    for s in range(8):
        R = 300 + 251 * s
        x = features(R, D, 50 + s, scale=1.0 + 0.15 * s)
        y, yv = supervision(R, 60 + s, p_valid=0.1 + 0.05 * s)
        rec = T.run(x, y, yv)
        window = check_step("method", rec, x, y, yv, D, 256, 32, method=method, window=window, where=f"step {s}")


@pytest.mark.gpu
@pytest.mark.parametrize("bound", ["private", "module"])
@pytest.mark.parametrize("method", ["moving_average", "running_mean", "kalman_filter"])
def test_regrowth_keeps_the_generator(method, bound):
    """A step larger than max_rows rebuilds the trainer's handle.  The generator must keep following the float64
    generator carried across every step, within generator_ref's bounds: moving_average's window of 5 steps, and (for a
    trainer without bound state tensors) var and the running sums.  'module': the state bound to a
    TraversabilityEstimator's generator, whose var and running sums are compared as well."""
    from wild_visual_navigation_b200 import ops

    D = 384
    P0 = make_params(D, 256, 32)
    if bound == "module":
        from wild_visual_navigation_b200 import TraversabilityEstimator
        from wild_visual_navigation_b200.traversability_estimator.traversability_estimator import default_params

        params = default_params()
        params["loss"]["method"] = method
        tr = TraversabilityEstimator(params=params, device="cuda", min_samples_for_training=0, max_rows=256)._trainer
    else:
        tr = ops.MlpTrainer(P0.cuda().clone(), D, 256, 32, max_rows=256)
        tr.set_confidence(METHODS[method])
    cgm = tr._conf[1:5]   # the bound state tensors (var, running_n, running_sum, running_sum_of_squares) or None
    # the generator carried in float64 across every step, as generator_ref's 'before' state, with the bound its carried
    # value has picked up so far (each step's bound is the one-step bound plus the carried one)
    window, var, e_var, running, e_run = [], 1.0, 0.0, [0.0, 0.0, 0.0], [0.0, 0.0]
    rows = [200, 230, 180, 600, 210, 190, 220]    # the fourth step exceeds max_rows
    for s, R in enumerate(rows):
        P = tr.params.double().clone()
        before = dict(cg_mean=tr.cg_mean.item(), var=var, running=running)
        x = features(R, D, 80 + s, scale=1.0 + 0.5 * s)
        y, yv = supervision(R, 90 + s, p_valid=0.3)
        fw = forward_ref(P, x.double(), y.double(), D, 256, 32)
        st = stats_ref(fw, yv)
        st["sum_lr"] = (st["sum_lr"][0], st["sum_lr"][1] + e_run[0])
        st["sum_lr2"] = (st["sum_lr2"][0], st["sum_lr2"][1] + e_run[1])
        gen, window = generator_ref(method, st, before, window, 0.5)
        tr.step(x, y, yv)
        _CTX[0] = f"regrowth {method} {bound} step {s} R={R} max_rows={tr.max_rows}"
        got = dict(mean=tr.cg_mean.item(), std=tr.cg_std.item())
        if method == "kalman_filter":   # the carried var's error contracts by (1 - gain)^2 <= 1 per step
            if st["n_valid"][0] > 0:     # and moves the gain by at most e_var (d gain / d cov <= 1 / R = 1)
                gain = (before["var"] + KF_Q) / (before["var"] + KF_Q + KF_R)
                gen["mean"] = (gen["mean"][0], gen["mean"][1] + abs(gen["mean"][0] - before["cg_mean"]) / gain * e_var)
            gen["var"] = (gen["var"][0], gen["var"][1] + e_var)
            gen["std"] = (gen["std"][0], gen["std"][1] + e_var / (2 * gen["std"][0]))
            var, e_var = gen["var"]
            if cgm[0] is not None:
                got["var"] = cgm[0].item()
        if method == "running_mean":
            running = [gen["running_n"][0], gen["running_sum"][0], gen["running_sumsq"][0]]
            e_run = [gen["running_sum"][1], gen["running_sumsq"][1]]
            if cgm[1] is not None:
                got.update(running_sum=cgm[2].item(), running_sumsq=cgm[3].item(), var=cgm[0].item())
                assert cgm[1].item() == running[0]
        for k, v in got.items():
            check(_one([v]), _one([gen[k][0]]), _one([gen[k][1]]), f"ts_regrowth_{k}")
    assert tr.max_rows >= 600


# ------------------------------------------------------------------------------------------------ GPU: legacy, Adam
@pytest.mark.gpu
@pytest.mark.parametrize("D", [384, 90])
def test_legacy_trainer(D):
    """Round 1's three-phase kernels (mlp_train.cu, latest_measurement, compacted rows) through the same checks."""
    run_and_check("legacy", D, 256, 32, R=1500, steps=2, seed=D + 1, legacy=True)


def _crafted_adam_state(tr, step, seed):
    """Adam's state before phase 4: the step counter, moments with every regime, and a gradient with exactly-zero
    entries (with zero and with non-zero moments) and entries near eps."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = tr.params.numel()
    tr.step_counter.fill_(step)
    if step > 1:
        tr.exp_avg.copy_(torch.randn(n, generator=g, device="cuda") * 1e-3)
        tr.exp_avg_sq.copy_(torch.rand(n, generator=g, device="cuda") * 1e-6)
        tr.exp_avg[:500] = 0
        tr.exp_avg_sq[:500] = 0
    grads = tr.grads
    grads[:1000] = 0.0                                                  # zero: bit-identical params where m0 = 0
    eps = tr.cfg.eps
    grads[1000:2000] = eps * torch.logspace(-2, 2, 1000, device="cuda") * torch.sign(torch.randn(1000, generator=g, device="cuda"))


@pytest.mark.gpu
@pytest.mark.parametrize("step", [1, 2, 10, 10000])
@pytest.mark.parametrize("opt", ["default", "custom"])
def test_adam(step, opt):
    """train_apply against float64 Adam fed the kernel's own gradient: step counters 1, 2, 10, 10^4, non-default lr /
    betas / eps, exactly-zero gradients (params bit-identical where the moments are zero, moments decaying where not)
    and gradients near eps."""
    cfg = CFG if opt == "default" else dict(CFG, lr=3e-3, betas=(0.8, 0.99), eps=1e-6)
    D, R = 384, 500
    T = Trainer(make_params(D, 256, 32), D, 256, 32, max_rows=R, cfg=cfg)
    x = features(R, D, 11)
    y, yv = supervision(R, 12)
    rec = T.run(x, y, yv, before_phase4=lambda tr: _crafted_adam_state(tr, step, step))
    b = rec["before"]
    b1, b2 = (f32(v) for v in cfg["betas"])
    (m0, v0), g = rec["adam_in"], rec["grads"][:-1].double()
    a = rec["after"]
    assert a["step"] == step
    (p, e_p), (m, e_m), (v, e_v) = adam_ref(b["params"], g, m0, v0, step, f32(cfg["lr"]), b1, b2, f32(cfg["eps"]))
    check(a["m"], m, e_m, "ts_adam_m")
    check(a["v"], v, e_v, "ts_adam_v")
    check(a["params"], p, e_p, "ts_adam_p")
    zero = g == 0
    still = zero & (m0 == 0)
    assert bool(still[:500].all())
    assert torch.equal(a["params"][still], b["params"][still]), "a zero gradient with zero moments moved a parameter"
    assert bool((a["m"][zero].abs() <= m0[zero].abs()).all()) and bool((a["v"][zero] <= v0[zero]).all())


@pytest.mark.gpu
def test_dead_units_have_exactly_zero_gradients():
    """Hidden units that no row activates get exactly-zero weight and bias gradients, and their parameters stay
    bit-identical through the first Adam step."""
    D, h1, h2, R = 384, 256, 32, 640
    P0 = make_params(D, h1, h2)
    W1, b1, W2, b2, W3, b3 = unflat(P0, D, h1, h2)
    dead1, dead2 = torch.arange(0, h1, 7), torch.arange(0, h2, 5)
    b1[dead1] = -1e3
    b2[dead2] = -1e3
    T = Trainer(P0, D, h1, h2, max_rows=R)
    x = features(R, D, 21)
    y, yv = supervision(R, 22)
    rec = T.run(x, y, yv)
    check_step("dead", rec, x, y, yv, D, h1, h2)
    G = unflat(rec["grads"][:-1].cpu(), D, h1, h2)
    assert bool((G[0][dead1] == 0).all()) and bool((G[1][dead1] == 0).all()) and bool((G[2][:, dead1] == 0).all())
    assert bool((G[2][dead2] == 0).all()) and bool((G[3][dead2] == 0).all()) and bool((G[4][:, dead2] == 0).all())
    Pa = unflat(rec["after"]["params"].cpu(), D, h1, h2)
    Pb = unflat(rec["before"]["params"].cpu(), D, h1, h2)
    assert torch.equal(Pa[0][dead1], Pb[0][dead1]) and torch.equal(Pa[1][dead1], Pb[1][dead1])
    assert torch.equal(Pa[4][:, dead2], Pb[4][:, dead2])


# ------------------------------------------------------------------------------------------------ CPU: the reference
def _oracle_case(method, steps=2, D=48, h1=32, h2=8, R=150):
    from oracle import wvn_path

    sd = {k: v.double() for k, v in wvn_path.mlp_init(D, (h1, h2), seed=5).items()}
    cg = wvn_path.ConfidenceState(0.5, method)
    opt_state, window, m0, v0 = None, [], None, None
    for s in range(steps):
        x = features(R, D, 30 + s, device="cpu").double()
        y, yv = supervision(R, 40 + s, device="cpu")
        y = y.double()
        P = torch.cat([v.reshape(-1) for v in sd.values()])
        before = dict(cg_mean=cg.mean.item(), var=cg.var.item(), running=cg.running.tolist())
        sd, opt_state, ref = wvn_path.train_step(sd, opt_state, x, y, yv, lr=1e-3, cg=cg)
        fw = forward_ref(P, x, y, D, h1, h2)
        st = stats_ref(fw, yv)
        gen, window = generator_ref(method, st, before, window, 0.5)
        # the oracle keeps mean / std in float32: compare, then feed the reference the oracle's own values
        for k in ("mean", "std"):
            assert abs(gen[k][0] - ref[k]) <= gen[k][1] + 2 * U * abs(ref[k]), (method, k, gen[k][0], ref[k])
        m, sd_ = np.float32(ref["mean"]), np.float32(ref["std"])
        if method == "kalman_filter":
            g = dict(lo=float(m), hi=1 / float(sd_ * np.float32(0.5)), cmin=0.0, cmax=0.0)
        elif method == "moving_average":   # clip to mean -+ 2 std (float32), then min-max of the clipped losses
            lo, hi = float(m - np.float32(2) * sd_), float(m + np.float32(2) * sd_)
            xc = fw["lr"].clamp(lo, hi)
            g = dict(lo=lo, hi=hi, cmin=xc.min().item(), cmax=xc.max().item())
        else:
            shifted = m + sd_ * np.float32(0.5)
            g = dict(lo=float(max(shifted - sd_, np.float32(0))), hi=float(shifted + sd_), cmin=0.0, cmax=0.0)
        g.update(g_reco=0.5 * 2 / (float(yv.sum()) * D), g_trav=0.03 * 2 / R)
        bw = backward_ref(fw, x, y, yv, method, g, CFG)
        assert (bw["conf"][0] - ref["confidence"].double()).abs().max() <= 2 * U
        gk = ref["grads"]
        mine = [bw["grads"][k][0] for k in ("w1", "b1", "w2", "b2", "w3", "b3")]
        for (name, want), got in zip(gk.items(), mine):
            err = (got - want).abs().max().item()
            assert err <= 1e-6 * want.abs().max().item() + 1e-300, (method, name, err)
        gflat = torch.cat([v.reshape(-1) for v in gk.values()])
        m0 = torch.zeros_like(P) if m0 is None else m0
        v0 = torch.zeros_like(P) if v0 is None else v0
        (p, _), (m0, _), (v0, _) = adam_ref(P, gflat, m0, v0, s + 1, 1e-3, 0.9, 0.999, 1e-8)
        want = torch.cat([v.reshape(-1) for v in sd.values()])
        assert (p - want).abs().max().item() <= 1e-12, method


@pytest.mark.parametrize("method", list(METHODS))
def test_reference_matches_oracle_float64(method):
    """forward_ref / generator_ref / backward_ref / adam_ref against oracle/wvn_path.train_step (autograd + torch Adam)
    run in float64: the generator to the oracle's float32 state, conf to its final .float(), gradients to 1e-6 of
    their block's largest element (the conf rounding feeds the unlabelled rows' weights), Adam to 1e-12.
    moving_average runs 7 steps, so the window of 5 wraps."""
    _oracle_case(method, steps=7 if method == "moving_average" else 2)


def fake_record(D, h1, h2, R, seed, method="latest_measurement", drop_rows=None):
    """A correct record built from the float64 reference rounded to fp32, as the driver would read it from a kernel
    that computes the step exactly.  drop_rows: leave these rows out of every weight-gradient sum."""
    P = make_params(D, h1, h2).double()
    x = features(R, D, seed, device="cpu")
    y, yv = supervision(R, seed + 1, device="cpu")
    fw = forward_ref(P, x.double(), y.double(), D, h1, h2)
    st = stats_ref(fw, yv)
    before = dict(params=P, m=torch.zeros_like(P), v=torch.zeros_like(P), step=0, cg_mean=0.0, cg_std=1.0, var=1.0,
                  running=[0.0, 0.0, 0.0])
    gen, _ = generator_ref(method, st, before, [], 0.5)
    sc1 = {k: v[0] for k, v in st.items()}
    sc1["x_min"], sc1["x_max"] = f32(sc1["x_min"]), f32(sc1["x_max"])
    sc2 = dict(sc1, mean=f32(gen["mean"][0]), std=f32(gen["std"][0]))
    m, sd = sc2["mean"], sc2["std"]
    g = dict(lo=float(np.fmax(m + 0.5 * sd - sd, 0.0)), hi=m + 1.5 * sd, cmin=0.0, cmax=0.0,
             g_reco=0.5 * 2 / (sc1["n_valid"] * D), g_trav=0.03 * 2 / R)
    xb, yb, yvb = x.double(), y.double(), yv
    if drop_rows is not None:
        keep = torch.ones(R, dtype=torch.bool)
        keep[drop_rows] = False
        fwd = forward_ref(P, xb[keep], yb[keep], D, h1, h2)
        bw = backward_ref(fwd, xb[keep], yb[keep], yvb[keep], method, g, CFG)
        bw_full = backward_ref(fw, xb, yb, yvb, method, g, CFG)
        bw["conf"], bw["trav_w"] = bw_full["conf"], bw_full["trav_w"]
    else:
        bw = backward_ref(fw, xb, yb, yvb, method, g, CFG)
    grads = torch.cat([bw["grads"][k][0].reshape(-1) for k in ("w1", "b1", "w2", "b2", "w3", "b3")] +
                      [bw["trav_w"][0].reshape(1)]).float()
    (p, _), (mm, _), (vv, _) = adam_ref(P, grads[:-1].double(), before["m"], before["v"], 1, f32(1e-3), f32(0.9),
                                        f32(0.999), f32(1e-8))
    after = dict(params=p.float().double(), m=mm.float().double(), v=vv.float().double(), step=1)
    with np.errstate(all="ignore"):
        n, nr = sc1["n_valid"], sc1["n_rows"]
        lreco, ltrav, ltc = f32(sc1["sum_lr"] / n), f32(sc1["sum_raw"] / nr), f32(float(grads[-1]) / nr)
    metrics = [f32(0.03 * ltc + 0.5 * lreco), ltrav, lreco, ltc, sc2["mean"], sc2["std"]]
    clean = [0] * 6 + [0x7FF0000000000000, 0] + [0] * 6
    rec = dict(before=before, sc1=sc1, sc2=sc2, conf=bw["conf"][0].float(), grads=grads, after=after, metrics=metrics,
               sc4_bits=clean, rows_padded=R, gen_after=dict(cg_mean=sc2["mean"], cg_std=sc2["std"], var=1.0))
    return rec, x, y, yv


CTRL = dict(D=384, h1=256, h2=32, R=3200, seed=9)


def test_checker_accepts_a_correct_step():
    rec, x, y, yv = fake_record(**CTRL)
    check_step("ctrl", rec, x, y, yv, 384, 256, 32)


def _rejects(rec, x, y, yv):
    with pytest.raises(AssertionError):
        check_step("ctrl", rec, x, y, yv, 384, 256, 32)


def test_checker_rejects_one_missing_row():
    """One labelled row of 3200 left out of the weight-gradient sums (what a split that stops a row short does)."""
    _, _, _, yv = fake_record(**CTRL)
    rec, x, y, yv = fake_record(**CTRL, drop_rows=[int(yv.nonzero()[400])])
    _rejects(rec, x, y, yv)


def test_checker_rejects_a_scaled_bias_gradient():
    rec, x, y, yv = fake_record(**CTRL)
    o = 256 * 384 + int(rec["grads"][256 * 384:256 * 385].abs().argmax())
    rec["grads"][o] *= 2
    _rejects(rec, x, y, yv)


def test_checker_rejects_one_wrong_conf():
    rec, x, y, yv = fake_record(**CTRL)
    i = int((~yv).nonzero()[3])
    rec["conf"][i] += 1e-3
    _rejects(rec, x, y, yv)


def test_checker_rejects_nan_in_one_gradient():
    rec, x, y, yv = fake_record(**CTRL)
    rec["grads"][1234] = float("nan")
    _rejects(rec, x, y, yv)


def test_checker_rejects_a_param_four_ulps_off():
    rec, x, y, yv = fake_record(**CTRL)
    p = rec["after"]["params"]
    p[777] = float(np.nextafter(np.nextafter(np.nextafter(np.nextafter(np.float32(p[777]), 1), 1), 1), 1))
    _rejects(rec, x, y, yv)


def test_checker_rejects_a_statistic_missing_one_row():
    rec, x, y, yv = fake_record(**CTRL)
    rec["sc1"]["sum_lr"] -= rec["sc1"]["sum_lr"] / rec["sc1"]["n_valid"]   # about one row's loss
    _rejects(rec, x, y, yv)


def test_checker_rejects_scalars_not_left_clean():
    rec, x, y, yv = fake_record(**CTRL)
    rec["sc4_bits"][7] = 0x3F50000000000000
    _rejects(rec, x, y, yv)
