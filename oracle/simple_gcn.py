"""ORACLE — float64 restatement of the SimpleGCN learner (reference: model/simple_gcn.py with utils/loss.py
TraversabilityLoss and torch.optim.Adam), and of the torch_geometric 2.x ``GCNConv`` it was written for.

torch_geometric is not a dependency, and upstream's ``from torch_geometric.nn import GCNConv`` is commented out (so
building ``SimpleGCN`` upstream raises ``NameError``).  ``GCNConv`` below restates ``GCNConv(in, out)`` with its defaults
(``add_self_loops=True``, ``normalize=True``, ``bias=True``, ``aggr="add"``, flow source -> target) as the
torch_geometric 2.x source defines it:

* ``Y = X lin.weight^T`` with ``lin`` a bias-free Linear, ``weight`` of shape (out, in);
* ``E'`` = the edges with every ``i -> i`` removed, plus exactly one self-loop per node (``add_remaining_self_loops``);
* ``d(i)`` = 1 + the number of edges of ``E'`` minus loops whose target (``edge_index[1]``) is ``i``;
* ``out[i] = sum_{j -> i in E'} d(j)^-1/2 d(i)^-1/2 Y[j] + bias``.

Parameters: ``bias`` is the conv's own parameter and ``lin`` a sub-module, so ``state_dict`` / ``parameters()`` order
is ``bias``, then ``lin.weight``.  Init: ``Linear.__init__`` draws glorot-uniform once, then ``GCNConv.__init__``'s
``reset_parameters`` draws it again (the value kept) and zeroes the bias.  This module cannot check any of this against
a real torch_geometric (not installed here); the goldens of ``tests/golden/make_golden_gcn.py`` are made with this
restatement injected into the reference's ``simple_gcn.py``.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from .wvn_path import ConfidenceState, traversability_loss


def _glorot_(w: torch.Tensor):
    a = math.sqrt(6.0 / (w.size(-2) + w.size(-1)))
    with torch.no_grad():
        w.uniform_(-a, a)


class _Linear(torch.nn.Module):
    """torch_geometric.nn.Linear(in, out, bias=False, weight_initializer="glorot"): draws its init in __init__."""

    def __init__(self, in_channels: int, out_channels: int):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.empty(out_channels, in_channels))
        self.reset_parameters()

    def reset_parameters(self):
        _glorot_(self.weight)

    def forward(self, x):
        return F.linear(x, self.weight)


def normalized_edges(edge_index: torch.Tensor, n: int, dtype=torch.float64):
    """(src, dst, weight) of E' with weight d(src)^-1/2 d(dst)^-1/2: the input edges without self-loops, in their
    order, then one self-loop per node."""
    ei = edge_index.long()
    keep = ei[0] != ei[1]
    loop = torch.arange(n, dtype=torch.long, device=ei.device)
    src = torch.cat([ei[0][keep], loop])
    dst = torch.cat([ei[1][keep], loop])
    deg = torch.zeros(n, dtype=dtype, device=ei.device).index_add_(0, dst, torch.ones(dst.numel(), dtype=dtype,
                                                                                       device=ei.device))
    dinv = deg.pow(-0.5)
    dinv[torch.isinf(dinv)] = 0.0
    return src, dst, dinv[src] * dinv[dst]


def aggregate(y: torch.Tensor, edge_index: torch.Tensor) -> torch.Tensor:
    """The normalised aggregation D^-1/2 (A + I) D^-1/2 Y (A[i, j] = number of edges j -> i)."""
    src, dst, w = normalized_edges(edge_index, y.shape[0], y.dtype)
    return torch.zeros_like(y).index_add_(0, dst, y[src] * w[:, None])


class GCNConv(torch.nn.Module):
    def __init__(self, in_channels: int, out_channels: int):
        super().__init__()
        self.lin = _Linear(in_channels, out_channels)
        self.bias = torch.nn.Parameter(torch.empty(out_channels))
        self.reset_parameters()

    def reset_parameters(self):
        self.lin.reset_parameters()
        with torch.no_grad():
            self.bias.zero_()

    def forward(self, x, edge_index):
        return aggregate(self.lin(x), edge_index) + self.bias


def keys(n_layers: int = 3):
    """State-dict keys in parameters() order: layers.{i}.bias, layers.{i}.lin.weight."""
    return [f"layers.{i}.{w}" for i in range(n_layers) for w in ("bias", "lin.weight")]


def init(dim: int, hidden_sizes, seed: int = 42) -> dict:
    """``torch.manual_seed(seed); SimpleGCN(dim, True, hidden_sizes)`` built from the restated GCNConv."""
    torch.manual_seed(seed)
    sd, inp = {}, dim
    for j, h in enumerate(hidden_sizes):
        if j == len(hidden_sizes) - 1:
            h = h + dim
        conv = GCNConv(inp, h)
        sd[f"layers.{j}.bias"] = conv.bias.detach().clone()
        sd[f"layers.{j}.lin.weight"] = conv.lin.weight.detach().clone()
        inp = h
    return sd


def forward(sd: dict, x: torch.Tensor, edge_index: torch.Tensor, n_layers: int = 3) -> torch.Tensor:
    """SimpleGCN.forward: GCNConv layers with ReLU between them, sigmoid on column 0 of the last."""
    h = x
    for j in range(n_layers):
        h = aggregate(F.linear(h, sd[f"layers.{j}.lin.weight"]), edge_index) + sd[f"layers.{j}.bias"]
        if j != n_layers - 1:
            h = F.relu(h)
    return torch.cat([torch.sigmoid(h[:, :1]), h[:, 1:]], dim=1)


def train_step(sd: dict, adam: dict, x, edge_index, y, y_valid, cg: ConfidenceState, w_trav=0.03, w_reco=0.5,
               anomaly_balanced=True, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
    """One train() body: forward on the graph, TraversabilityLoss (``cg`` updated in place), backward, Adam.
    ``adam``: {"step": int, "exp_avg": {k: t}, "exp_avg_sq": {k: t}}, updated in place.  Computes in x's dtype.
    Returns (new_sd, grads, loss, aux) as oracle.double_mlp.train_step."""
    params = {k: v.detach().clone().to(x.dtype).requires_grad_(True) for k, v in sd.items()}
    res = forward(params, x, edge_index)
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


def padded_to_graph(feat, n_rows, edges, n_edges):
    """The batched graph a padded batch stands for: live rows of frame 0, then frame 1, ...; each frame's edges (local
    ids, ``edges [G, Emax, 2]``, the first ``n_edges[g]`` rows) offset by the frame's first row, edges with an endpoint
    outside the frame's live rows dropped.  Returns (x [N, D], edge_index [2, E])."""
    xs, eis, off = [], [], 0
    for g in range(feat.shape[0]):
        n = int(n_rows[g])
        xs.append(feat[g, :n])
        e = edges[g, : max(int(n_edges[g]), 0)].long()
        ok = (e >= 0).all(1) & (e < n).all(1)
        eis.append(e[ok].t() + off)
        off += n
    return torch.cat(xs), torch.cat(eis, 1) if eis else torch.zeros(2, 0, dtype=torch.long)
