"""The data-parallel decomposition of the DoubleMLP and LinearRnvp train steps, in float64 on the CPU.

Two gloo ranks hold ragged shards.  Each runs the oracle's forward on its shard, all-reduces the statistic sums (SUM)
and the extrema (MIN / MAX), updates the generator from the global sums, forms its LOCAL loss with the GLOBAL
normalisers (row counts), back-propagates and all-reduces the gradient.  That must reproduce ``oracle.*.train_step`` on
the concatenated rows: the arithmetic the CUDA steps implement between their phases."""
import math
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from oracle import double_mlp as odm
from oracle import linear_rnvp as orn
from oracle.wvn_path import ConfidenceState, confidence_inference

METHODS = ("latest_measurement", "running_mean", "moving_average", "kalman_filter")
TOL = 1e-10


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class SumsGenerator(ConfidenceState):
    """ConfidenceState updated from all-reduced sums (n, sum, sum of squares, min, max of the input) instead of the
    concatenated rows; the same float32 state and casts as the oracle."""

    def update_from_sums(self, x, n, s1, s2, x_min, x_max):
        m = self.method
        if m == "latest_measurement":
            self.mean[0] = s1 / n
            self.std[0] = math.sqrt((s2 - s1 * s1 / n) / (n - 1))
            return confidence_inference(x, self.mean, self.std, self.std_factor)
        if m == "running_mean":
            self.running += torch.tensor([n, s1, s2], dtype=torch.float64)
            self.mean[0] = self.running[1] / self.running[0]
            self.var[0] = self.running[2:3] / self.running[0] - self.mean ** 2
            self.std[0] = torch.sqrt(self.var)[0, 0]
            return confidence_inference(x, self.mean, self.std, self.std_factor)
        if m == "moving_average":
            self.window = (self.window + [(n, s1, s2)])[-5:]
            N, S1, S2 = (sum(w[i] for w in self.window) for i in range(3))
            self.mean[0] = S1 / N
            self.std[0] = math.sqrt((S2 - S1 * S1 / N) / (N - 1))
            lo, hi = self.mean - 2 * self.std, self.mean + 2 * self.std
            xc = torch.clip(x, lo, hi)
            cmin, cmax = torch.clip(torch.tensor([x_min], dtype=x.dtype), lo, hi), torch.clip(torch.tensor([x_max], dtype=x.dtype), lo, hi)
            return ((xc - cmin) / (cmax - cmin)).float()
        if n != 0:   # kalman_filter
            meas = torch.tensor(s1 / n, dtype=torch.float64)
            state, cov = self.mean.clone(), self.var.clone() + self.kf_proc_cov
            gain = cov / (cov + self.kf_meas_cov)
            self.mean[0] = (state + (gain @ (meas - state).reshape(1)))[0]
            self.var[0, 0] = ((1.0 - gain) @ cov)[0, 0]
        self.std[0] = torch.sqrt(self.var)[0, 0]
        conf = torch.exp(-(((x - self.mean) / (self.std * self.std_factor)) ** 2) * 0.5)
        conf[x < self.mean] = 1.0
        return conf.float()


def _allreduce(vals, op=dist.ReduceOp.SUM):
    t = torch.tensor(vals, dtype=torch.float64)
    dist.all_reduce(t, op=op)
    return t.tolist()


def _double_rank_step(sd, x, y, yv, cg, w_trav=0.03, w_reco=0.5):
    params = {k: v.detach().clone().requires_grad_(True) for k, v in sd.items()}
    out = odm.forward(params, x)
    D = x.shape[1]
    lr = F.mse_loss(out[:, -D:], x, reduction="none").mean(dim=1)
    raw = F.mse_loss(out[:, :-D].squeeze(1), y, reduction="none")
    lv = lr.detach()[yv]
    inf = float("inf")
    s = _allreduce([lv.sum().item(), (lv ** 2).sum().item(), raw.detach().sum().item(), float(lv.numel()),
                    float(x.shape[0])])
    mn = _allreduce([lr.detach().min().item() if x.shape[0] else inf], dist.ReduceOp.MIN)[0]
    mx = _allreduce([lr.detach().max().item() if x.shape[0] else -inf], dist.ReduceOp.MAX)[0]
    S1, S2, SR, NV, NR = s
    with torch.no_grad():
        conf = cg.update_from_sums(lr.detach(), NV, S1, S2, mn, mx)
    w = torch.where(yv, torch.ones_like(raw), (1 - conf).to(raw.dtype))   # anomaly_balanced
    l_trav = (raw * w).sum() / NR
    loss = w_trav * l_trav + w_reco * lr[yv].sum() / NV
    loss.backward()
    grads = torch.cat([params[k].grad.reshape(-1) for k in sd])
    dist.all_reduce(grads)
    trav_w = _allreduce([(raw * w).detach().sum().item()])[0]
    return grads, {"loss_reco": S1 / NV, "loss_trav": SR / NR, "loss_trav_confidence": trav_w / NR,
                   "mean": cg.mean.item(), "std": cg.std.item(), "var": cg.var.item(), "running": cg.running.tolist()}


def _flow_rank_step(sd, x, cg):
    params = {k: v.detach().clone().requires_grad_(True) for k, v in sd.items() if k in orn.NETS}
    full = dict(sd)
    full.update(params)
    res = orn.forward(full, x)
    nll = -(res["logprob"].sum(1) + res["log_det"])
    v = nll.detach()
    inf = float("inf")
    S1, S2, N = _allreduce([v.sum().item(), (v ** 2).sum().item(), float(v.numel())])
    mn = _allreduce([v.min().item() if v.numel() else inf], dist.ReduceOp.MIN)[0]
    mx = _allreduce([v.max().item() if v.numel() else -inf], dist.ReduceOp.MAX)[0]
    with torch.no_grad():
        cg.update_from_sums(v, N, S1, S2, mn, mx)
    (nll.sum() / N).backward()
    grads = torch.cat([(params[k].grad if params[k].grad is not None else torch.zeros_like(params[k])).reshape(-1)
                       for k in params])
    dist.all_reduce(grads)
    return grads, {"loss": S1 / N, "mean": cg.mean.item(), "std": cg.std.item(), "var": cg.var.item(),
                   "running": cg.running.tolist()}


def _adam(sd, keys, grads, adam, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
    """torch.optim.Adam on the all-reduced flat gradient, the oracle's arithmetic."""
    adam["step"] = adam.get("step", 0) + 1
    t, (b1, b2), off, new = adam["step"], betas, 0, dict(sd)
    for k in keys:
        p = sd[k]
        g = grads[off:off + p.numel()].reshape(p.shape)
        off += p.numel()
        m = b1 * adam.setdefault("m", {}).get(k, torch.zeros_like(g)) + (1 - b1) * g
        v = b2 * adam.setdefault("v", {}).get(k, torch.zeros_like(g)) + (1 - b2) * g * g
        adam["m"][k], adam["v"][k] = m, v
        new[k] = p - (lr / (1 - b1**t)) * m / (v.sqrt() / math.sqrt(1 - b2**t) + eps)
    return new


def _worker(rank, world, port, learner, method, sd, shards, ret):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    cg = SumsGenerator(0.5, method)
    keys = list(sd) if learner == "double" else [k for k in sd if k in orn.NETS]
    adam, out = {}, []
    for shard in shards[rank]:
        if learner == "double":
            grads, m = _double_rank_step(sd, *shard, cg)
        else:
            grads, m = _flow_rank_step(sd, shard[0], cg)
        sd = _adam(sd, keys, grads, adam)
        out.append((grads, m))
    ret[rank] = {"steps": out, "params": torch.cat([sd[k].reshape(-1) for k in keys])}
    dist.destroy_process_group()


def _shards(learner, D, seed):
    g = torch.Generator().manual_seed(seed)
    sizes = ((7, 12), (5, 9), (11, 6))
    shards = [[], []]
    for step, ns in enumerate(sizes):
        for r, n in enumerate(ns):
            x = torch.randn(n, D, generator=g, dtype=torch.float64)
            yv = torch.rand(n, generator=g) < 0.5
            yv[0] = True
            if learner == "flow" and r == 1 and step == 1:
                x = x[:0]   # a rank with no labelled row this step
            y = torch.where(yv, torch.rand(n, generator=g, dtype=torch.float64), torch.zeros(n, dtype=torch.float64))
            shards[r].append((x, y[: x.shape[0]], yv[: x.shape[0]]))
    return shards


def _close(a, b):
    return abs(a - b) <= TOL * max(1.0, abs(b))


@pytest.mark.parametrize("learner", ["double", "flow"])
@pytest.mark.parametrize("method", METHODS)
def test_two_rank_decomposition_reproduces_the_oracle_step(learner, method):
    D = 12
    if learner == "double":
        sd = {k: v.double() for k, v in odm.init(D, [16, 8, 1]).items()}
    else:
        torch.manual_seed(3)
        from wild_visual_navigation_b200.model.linear_rnvp import LinearRnvp

        m = LinearRnvp(D, [16], mask_type="odds", conditioning_size=0, use_permutation=True, single_function=False)
        sd = {k: (v.detach().double() if v.is_floating_point() else v) for k, v in m.state_dict().items()}
    shards = _shards(learner, D, seed=5)
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(2, _free_port(), learner, method, sd, shards, ret), nprocs=2, join=True)

    cg = ConfidenceState(0.5, method)
    adam = {}
    cur = dict(sd)
    for step in range(3):
        x = torch.cat([shards[r][step][0] for r in (0, 1)])
        if learner == "double":
            y = torch.cat([shards[r][step][1] for r in (0, 1)])
            yv = torch.cat([shards[r][step][2] for r in (0, 1)])
            new, grads, loss, aux = odm.train_step(cur, adam, x, y, yv, cg)
            want = {"loss_reco": aux["loss_reco"].item(), "loss_trav": aux["loss_trav"].item(),
                    "loss_trav_confidence": aux["loss_trav_confidence"].item()}
            g = torch.cat([grads[k].reshape(-1) for k in cur])
        else:
            new, grads, loss, _ = orn.train_step(cur, adam, x, cg)
            want = {"loss": loss.item()}
            g = torch.cat([grads[k].reshape(-1) for k in grads])
        want.update(mean=cg.mean.item(), std=cg.std.item(), var=cg.var.item(), running=cg.running.tolist())
        for r in (0, 1):
            got_g, got = ret[r]["steps"][step]
            assert ((got_g - g).norm() / g.norm()).item() <= TOL, (step, r)
            for k, v in want.items():
                vals = zip(got[k], v) if isinstance(v, list) else [(got[k], v)]
                assert all(_close(a, b) for a, b in vals), (step, r, k, got[k], v)
        cur = new
    keys = list(cur) if learner == "double" else [k for k in cur if k in orn.NETS]
    p = torch.cat([cur[k].reshape(-1) for k in keys])
    for r in (0, 1):
        assert ((ret[r]["params"] - p).norm() / p.norm()).item() <= TOL
    assert torch.equal(ret[0]["params"], ret[1]["params"])
