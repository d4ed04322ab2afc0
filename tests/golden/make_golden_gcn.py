"""Generate tests/golden/gcn.pt by running the REFERENCE's own model/simple_gcn.py, TraversabilityLoss,
ConfidenceGenerator, Batch.from_data_list and torch.optim.Adam.

Run with a checkout of the reference repository:
``WVN_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_gcn.py``

Upstream's ``from torch_geometric.nn import GCNConv`` is commented out, so ``simple_gcn.py`` is loaded from its file
with the restated ``oracle.simple_gcn.GCNConv`` placed in its module namespace, where the import would put it.
torch_geometric itself is not available: equality with its GCNConv (arithmetic and init draws) is not checked.

  * ``graph``: the reference's shipped ``assets/graph/graph.pt`` (a pickled torch_geometric Data, decoded with stub
    classes): the 100-segment STEGO graph, ``x (100, 90)``, ``edge_index (2, 384)``, ``y`` / ``y_valid`` (16 labelled);
  * ``SimpleGCN(90, True, [32, 16, 1])`` under seed 42, three ``TraversabilityEstimator.train()`` bodies on that graph
    per ConfidenceGenerator method (anomaly_balanced True): per step the loss, aux, every gradient, confidence
    and generator state, the output of the first step and the state dict after the last;
  * ``synthetic``: three steps of ``SimpleGCN(24, True, [16, 8, 1])`` on a ``Batch.from_data_list`` of four seeded
    nodes with offset edges (an isolated segment, a self-loop, a duplicated edge, a node without edges);
  * one checkpoint in the reference's on-disk format and one ``.tmp_state_dict.pt`` (latest_measurement on graph.pt);
  * the init summary (per key: shape, sum, first 8 elements) of ``SimpleGCN(384, True, [256, 128, 1])`` and
    ``SimpleGCN(90, True, [256, 128, 1])`` under seed 42.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402
from oracle.simple_gcn import GCNConv  # noqa: E402

METHODS = ("latest_measurement", "running_mean", "moving_average", "kalman_filter")


def load_simple_gcn():
    name = "wild_visual_navigation.model.simple_gcn"
    spec = importlib.util.spec_from_file_location(name, os.path.join(ref_import.REF_ROOT,
                                                                     "wild_visual_navigation/model/simple_gcn.py"))
    mod = importlib.util.module_from_spec(spec)
    mod.GCNConv = GCNConv   # where the commented-out import would put it
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod.SimpleGCN


def load_graph():
    """assets/graph/graph.pt with stub torch_geometric classes (as make_golden.py decodes it)."""
    tg, tgd = types.ModuleType("torch_geometric"), types.ModuleType("torch_geometric.data")
    tgdd, tgds = types.ModuleType("torch_geometric.data.data"), types.ModuleType("torch_geometric.data.storage")

    class _Any:
        def __init__(self, *a, **k): pass
        def __setstate__(self, st): self.__dict__.update(st if isinstance(st, dict) else {"state": st})

    for m in (tgdd, tgds, tgd):
        m.__getattr__ = lambda name: type(name, (_Any,), {})  # type: ignore
    mods = {"torch_geometric": tg, "torch_geometric.data": tgd, "torch_geometric.data.data": tgdd,
            "torch_geometric.data.storage": tgds}
    sys.modules.update(mods)
    try:
        g = torch.load(os.path.join(ref_import.REF_ROOT, "assets", "graph", "graph.pt"), map_location="cpu",
                       weights_only=False)
    finally:
        for k in mods:
            sys.modules.pop(k, None)
    m = g._store._mapping
    return {k: m[k].clone() for k in ("x", "edge_index", "y", "y_valid")}


def synthetic_nodes(ns, g, D=24):
    """Four nodes: a chain with an isolated segment, one with a self-loop and a duplicated edge, one without edges
    (edge_index (2, 0)), one dense."""
    specs = [(7, [[0, 1], [1, 2], [2, 3], [4, 5]]),            # segment 6 isolated
             (5, [[0, 1], [1, 1], [2, 1], [2, 1], [3, 4]]),    # self-loop 1 -> 1, edge 2 -> 1 twice
             (4, []),                                          # no edges
             (6, [[i, j] for i in range(6) for j in range(6) if i < j])]
    out = []
    for n, e in specs:
        x = torch.randn(n, D, generator=g) * 0.8 + 0.1
        yv = torch.rand(n, generator=g) < 0.4
        yv[0] = True
        y = torch.where(yv, torch.rand(n, generator=g).clamp(min=0.001), torch.zeros(n))
        ei = torch.tensor(e, dtype=torch.long).reshape(-1, 2).t().contiguous()
        out.append(ns.Data(x=x, edge_index=ei, y=y, y_valid=yv))
    return out


def run(ns, SimpleGCN, method, data, D, hidden, steps=3):
    torch.manual_seed(42)
    model = SimpleGCN(D, True, hidden)
    model.train()
    loss_fn = ns.TraversabilityLoss(w_trav=0.03, w_reco=0.5, w_temp=0.0, anomaly_balanced=True, model=model,
                                    method=method, confidence_std_factor=0.5, log_enabled=False, log_folder="/tmp")
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    init = {k: v.clone() for k, v in model.state_dict().items()}
    rec = []
    for step in range(steps):
        graph = data(step)
        res = model(graph)
        loss, aux, _ = loss_fn(graph, res, step=step, log_step=False)
        opt.zero_grad()
        loss.backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters()}
        opt.step()
        cg = loss_fn._confidence_generator
        r = {"loss": loss.detach().clone(),
             "loss_reco": aux["loss_reco"].detach().clone(), "loss_trav": aux["loss_trav"].detach().clone(),
             "loss_trav_confidence": aux["loss_trav_confidence"].detach().clone(), "grads": grads,
             "confidence": aux["confidence"].detach().clone(), "cg_mean": cg.mean.detach().clone(),
             "cg_std": cg.std.detach().clone(), "cg_var": cg.var.detach().clone()}
        if step == 0:
            r["res"] = res.detach().clone()
        if step == steps - 1:
            r["state_dict"] = {k: v.clone() for k, v in model.state_dict().items()}
        rec.append(r)
    return {"init": init, "steps": rec}, model, opt, loss_fn


def summary(sd):
    return {k: {"shape": tuple(v.shape), "sum": v.double().sum().item(), "first": v.reshape(-1)[:8].clone()}
            for k, v in sd.items()}


def main():
    assert ref_import.available(), "set WVN_REFERENCE_ROOT to a reference checkout"
    ns = ref_import.load()
    SimpleGCN = load_simple_gcn()
    gr = load_graph()
    out = {"graph": gr, "train": {}}
    graph = ns.Data(x=gr["x"], edge_index=gr["edge_index"], y=gr["y"], y_valid=gr["y_valid"])
    for method in METHODS:
        out["train"][method], model, opt, loss_fn = run(ns, SimpleGCN, method, lambda step: graph, 90, [32, 16, 1])
        if method == "latest_measurement":
            out["checkpoint"] = {"step": 3, "model_state_dict": model.state_dict(),
                                 "optimizer_state_dict": opt.state_dict(),
                                 "traversability_loss_state_dict": loss_fn.state_dict(),
                                 "loss": out["train"][method]["steps"][-1]["loss"].item()}
            tmp = model.state_dict()
            tmp["confidence_generator"] = loss_fn._confidence_generator.get_dict()
            out["tmp_state_dict"] = tmp
    first = out["train"][METHODS[0]]["init"]
    for m in METHODS[1:]:   # the seeded init is the same for every method: stored once
        assert all(torch.equal(v, first[k]) for k, v in out["train"][m].pop("init").items())
    g = torch.Generator().manual_seed(11)
    nodes = [synthetic_nodes(ns, g) for _ in range(3)]
    out["synthetic_nodes"] = [[{"x": d.x, "edge_index": d.edge_index, "y": d.y, "y_valid": d.y_valid} for d in n]
                              for n in nodes]
    eis = out["synthetic_edge_index"] = []

    def batch(step):   # the reference's Batch.from_data_list returns the class itself: build each batch when used
        b = ns.Batch.from_data_list(nodes[step])
        eis.append(b.edge_index.clone())
        return b

    out["synthetic"], _, _, _ = run(ns, SimpleGCN, "latest_measurement", batch, 24, [16, 8, 1])
    for D in (384, 90):
        hs = [256, 128, 1]
        torch.manual_seed(42)
        big = SimpleGCN(D, True, hs)
        assert hs == [256, 128, 1]
        out[f"init{D}"] = summary(big.state_dict())
        out[f"init{D}_keys"] = list(big.state_dict())
        out[f"init{D}_param_count"] = sum(p.numel() for p in big.parameters())
    torch.save(out, os.path.join(HERE, "gcn.pt"))
    print("wrote", os.path.join(HERE, "gcn.pt"))


if __name__ == "__main__":
    main()
