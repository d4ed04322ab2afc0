"""ORACLE — float64 restatement of the DoubleMLP learner (reference: model/simple_mlp.py:42-67 with
utils/loss.py TraversabilityLoss and torch.optim.Adam): the seeded module construction, the forward, one
``TraversabilityEstimator.train()`` body.  Tests compare the CUDA kernels against it; it reproduces the goldens that
``tests/golden/make_golden_double_mlp.py`` makes from the reference's own classes."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from .wvn_path import ConfidenceState, traversability_loss


def keys(n_layers: int = 3):
    """State-dict keys in parameters() order: networks.{0,1}.{0,2,4}.{weight,bias}."""
    return [f"networks.{n}.{2 * i}.{w}" for n in range(2) for i in range(n_layers) for w in ("weight", "bias")]


def init(dim: int, hidden_sizes, seed: int = 42) -> dict:
    """``torch.manual_seed(seed); DoubleMLP(dim, hidden_sizes)``: the Linear layers of net 0, then of net 1, in the
    reference's construction order, so the same seeded init."""
    torch.manual_seed(seed)
    sd = {}
    for n, last in enumerate([hidden_sizes[-1], dim]):
        inp = dim
        for i, hs in enumerate(list(hidden_sizes[:-1]) + [last]):
            lin = torch.nn.Linear(inp, hs)
            sd[f"networks.{n}.{2 * i}.weight"] = lin.weight.detach().clone()
            sd[f"networks.{n}.{2 * i}.bias"] = lin.bias.detach().clone()
            inp = hs
    return sd


def net(sd: dict, x: torch.Tensor, n: int) -> torch.Tensor:
    h = F.relu(F.linear(x, sd[f"networks.{n}.0.weight"], sd[f"networks.{n}.0.bias"]))
    h = F.relu(F.linear(h, sd[f"networks.{n}.2.weight"], sd[f"networks.{n}.2.bias"]))
    return F.linear(h, sd[f"networks.{n}.4.weight"], sd[f"networks.{n}.4.bias"])


def forward(sd: dict, x: torch.Tensor) -> torch.Tensor:
    """cat([sigmoid(networks[0](x)), networks[1](x)], 1)."""
    return torch.cat([torch.sigmoid(net(sd, x, 0)), net(sd, x, 1)], dim=1)


def train_step(sd: dict, adam: dict, x, y, y_valid, cg: ConfidenceState, w_trav=0.03, w_reco=0.5,
               anomaly_balanced=True, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
    """One train() body: forward, TraversabilityLoss (the generator ``cg`` updated in place), backward, Adam.
    ``adam``: {"step": int, "exp_avg": {k: t}, "exp_avg_sq": {k: t}}, updated in place.  Computes in x's dtype.
    Returns (new_sd, grads, loss, aux) with aux = loss_reco, loss_trav, loss_trav_confidence, confidence, mean, std."""
    params = {k: v.detach().clone().to(x.dtype).requires_grad_(True) for k, v in sd.items()}
    res = forward(params, x)
    loss, aux = traversability_loss(res, x, y.to(x.dtype), y_valid, w_trav=w_trav, w_reco=w_reco,
                                    std_factor=cg.std_factor, anomaly_balanced=anomaly_balanced, cg=cg)
    loss.backward()
    grads = {k: v.grad.detach().clone() for k, v in params.items()}
    adam["step"] = adam.get("step", 0) + 1
    t = adam["step"]
    b1, b2 = betas
    new_sd = {}
    for k, p in params.items():
        g = grads[k]
        m = b1 * adam.setdefault("exp_avg", {}).get(k, torch.zeros_like(g)) + (1 - b1) * g
        v = b2 * adam.setdefault("exp_avg_sq", {}).get(k, torch.zeros_like(g)) + (1 - b2) * g * g
        adam["exp_avg"][k], adam["exp_avg_sq"][k] = m, v
        new_sd[k] = p.detach() - (lr / (1 - b1**t)) * m / (v.sqrt() / math.sqrt(1 - b2**t) + eps)
    return new_sd, grads, loss.detach(), {k: (v.detach() if torch.is_tensor(v) else v) for k, v in aux.items()}


def packed_simple_mlp(sd: dict) -> dict:
    """The block-structured SimpleMLP (``layers.{0,2,4}``) that computes the DoubleMLP's output: layer 1 stacks both
    nets' rows, layer 2 is block-diagonal, layer 3's row 0 reads net 0's half and rows 1..D net 1's half."""
    w1 = torch.cat([sd["networks.0.0.weight"], sd["networks.1.0.weight"]])
    b1 = torch.cat([sd["networks.0.0.bias"], sd["networks.1.0.bias"]])
    w2 = torch.block_diag(sd["networks.0.2.weight"], sd["networks.1.2.weight"])
    b2 = torch.cat([sd["networks.0.2.bias"], sd["networks.1.2.bias"]])
    w3 = torch.block_diag(sd["networks.0.4.weight"], sd["networks.1.4.weight"])
    b3 = torch.cat([sd["networks.0.4.bias"], sd["networks.1.4.bias"]])
    return {"layers.0.weight": w1, "layers.0.bias": b1, "layers.2.weight": w2, "layers.2.bias": b2,
            "layers.4.weight": w3, "layers.4.bias": b3}
