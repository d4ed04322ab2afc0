"""ORACLE — the LinearRnvp anomaly-detection learner restated in plain torch, in the dtype of its inputs (float64 in the
tests): the flow forward (model/linear_rnvp.py:67-296 with flow_n = 2, use_permutation = True), the per-row NLL,
AnomalyLoss (utils/loss.py:16-54) and one TraversabilityEstimator.train() step with torch.optim.Adam's update.

State dicts use the reference's keys: ``prior_mean``, ``prior_var``, ``flows.{0,2}.mask``,
``flows.{0,2}.{s,t}.{0,2,4}.{weight,bias}``, ``flows.{1,3}.{p,invp}``.
"""
from __future__ import annotations

import math

import torch

from .wvn_path import ConfidenceState

NETS = [f"flows.{c}.{n}.{i}.{w}" for c in (0, 2) for n in ("s", "t") for i in (0, 2, 4) for w in ("weight", "bias")]


def _net(x, sd, pre):
    h = torch.relu(x @ sd[pre + ".0.weight"].T + sd[pre + ".0.bias"])
    h = torch.relu(h @ sd[pre + ".2.weight"].T + sd[pre + ".2.bias"])
    return h @ sd[pre + ".4.weight"].T + sd[pre + ".4.bias"]


def forward(sd: dict, x: torch.Tensor):
    """-> dict(z, log_det, logprob) like LinearRnvp.forward (the prior N(prior_mean, prior_var) with prior_var as the
    scale, as upstream)."""
    log_det = torch.zeros(x.shape[0], dtype=x.dtype, device=x.device)
    for c, p in ((0, 1), (2, 3)):
        m = sd[f"flows.{c}.mask"].to(x.dtype)
        mu = x * m
        s = torch.tanh(_net(mu, sd, f"flows.{c}.s"))
        t = _net(mu, sd, f"flows.{c}.t")
        x = mu + (1 - m) * (x * torch.exp(s) + t)
        log_det = log_det + ((1 - m) * s).sum(1)
        x = x[:, sd[f"flows.{p}.p"]]
    mean, scale = sd["prior_mean"].to(x.dtype), sd["prior_var"].to(x.dtype)
    logprob = -((x - mean) ** 2) / (2 * scale**2) - torch.log(scale) - math.log(math.sqrt(2 * math.pi))
    return {"z": x, "log_det": log_det, "logprob": logprob}


def bf16_operands(sd: dict) -> dict:
    """The state dict with every Linear weight rounded to bf16 (values kept in the original dtype): the weights the
    per-pixel wgmma path multiplies with."""
    return {k: (v.to(torch.bfloat16).to(v.dtype) if k.endswith(".weight") else v) for k, v in sd.items()}


def nll_bf16(sd: dict, x: torch.Tensor) -> torch.Tensor:
    """The NLL with the per-pixel path's bf16 rounding points emulated in x's dtype: weights, mu = u * mask and both
    hidden activations rounded to bf16; everything else (accumulation, coupling arithmetic) exact."""
    r = lambda t: t.to(torch.bfloat16).to(t.dtype)
    sdb = bf16_operands(sd)

    def net(mu, pre):
        h = r(torch.relu(mu @ sdb[pre + ".0.weight"].T + sdb[pre + ".0.bias"]))
        h = r(torch.relu(h @ sdb[pre + ".2.weight"].T + sdb[pre + ".2.bias"]))
        return h @ sdb[pre + ".4.weight"].T + sdb[pre + ".4.bias"]

    log_det = torch.zeros(x.shape[0], dtype=x.dtype, device=x.device)
    for c, p in ((0, 1), (2, 3)):
        m = sd[f"flows.{c}.mask"].to(x.dtype)
        mu = r(x * m)
        s = torch.tanh(net(mu, f"flows.{c}.s"))
        t = net(mu, f"flows.{c}.t")
        x = x * m + (1 - m) * (x * torch.exp(s) + t)
        log_det = log_det + ((1 - m) * s).sum(1)
        x = x[:, sd[f"flows.{p}.p"]]
    return (x * x / 2 + math.log(math.sqrt(2 * math.pi))).sum(1) - log_det


def nll(sd: dict, x: torch.Tensor) -> torch.Tensor:
    r = forward(sd, x)
    return -(r["logprob"].sum(1) + r["log_det"])


def anomaly_loss(res: dict, cg: ConfidenceState):
    """AnomalyLoss.forward: (loss, confidence); the generator is updated with x = x_positive = the per-row NLL."""
    losses = res["logprob"].sum(1) + res["log_det"]
    with torch.no_grad():
        confidence = cg.update(-losses.detach(), -losses.detach())
    return -torch.mean(losses), confidence


def train_step(sd: dict, adam: dict, x: torch.Tensor, cg: ConfidenceState, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
    """One train() step on the (already labelled-only) rows x.  ``adam``: {"step": int, "exp_avg": {k: t},
    "exp_avg_sq": {k: t}} over the 24 parameter tensors (updated in place).  Returns (new_sd, grads, loss,
    confidence); torch.optim.Adam's arithmetic (no weight decay, no amsgrad) in x's dtype."""
    params = {k: v.detach().clone().to(x.dtype).requires_grad_(True) for k, v in sd.items() if k in NETS}
    full = dict(sd)
    full.update(params)
    res = forward(full, x)
    loss, conf = anomaly_loss(res, cg)
    loss.backward()
    grads = {k: v.grad.detach().clone() for k, v in params.items()}
    adam["step"] = adam.get("step", 0) + 1
    t = adam["step"]
    b1, b2 = betas
    new_sd = dict(sd)
    for k, p in params.items():
        g = grads[k]
        m = adam.setdefault("exp_avg", {}).get(k, torch.zeros_like(g))
        v = adam.setdefault("exp_avg_sq", {}).get(k, torch.zeros_like(g))
        m = b1 * m + (1 - b1) * g
        v = b2 * v + (1 - b2) * g * g
        adam["exp_avg"][k], adam["exp_avg_sq"][k] = m, v
        denom = (v.sqrt() / math.sqrt(1 - b2**t)) + eps
        new_sd[k] = p.detach() - (lr / (1 - b1**t)) * m / denom
    return new_sd, grads, loss.detach(), conf
