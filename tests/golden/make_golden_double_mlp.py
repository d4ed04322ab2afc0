"""Generate tests/golden/double_mlp.pt by running the REFERENCE's own DoubleMLP, TraversabilityLoss and
torch.optim.Adam.

Run with a checkout of the reference repository:
``WVN_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_double_mlp.py``

  * ``DoubleMLP(32, [16, 8, 1])`` under seed 42, three ``TraversabilityEstimator.train()`` bodies (forward,
    TraversabilityLoss, zero_grad / backward / Adam step, lr 1e-3) on seeded rows, per ConfidenceGenerator method with
    anomaly_balanced True, and latest_measurement with anomaly_balanced False: per step the rows, loss, aux, every
    gradient, confidence and generator state, and the state dict after the last step;
  * one checkpoint in the reference's on-disk format (``save_checkpoint``: step, model / optimizer / loss state dicts);
  * one ``.tmp_state_dict.pt`` as the learning node writes it (wvn_learning_node.py:381-394);
  * the init summary (per key: shape, sum, first 8 elements) of ``DoubleMLP(384, [64, 32, 1])`` and
    ``DoubleMLP(90, [64, 32, 1])`` under seed 42, and that the constructor leaves ``hidden_sizes`` unchanged.
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402

METHODS = ("latest_measurement", "running_mean", "moving_average", "kalman_filter")
CASES = [(m, True) for m in METHODS] + [("latest_measurement", False)]


def rows(g, step, D=32):
    R = 40 + 8 * step
    x = torch.randn(R, D, generator=g) * 0.8 + 0.1
    yv = torch.rand(R, generator=g) < 0.35
    yv[:2] = True
    y = torch.where(yv, torch.rand(R, generator=g).clamp(min=0.001), torch.zeros(R))
    return x, y, yv


def run(ns, DoubleMLP, method, balanced, steps=3):
    torch.manual_seed(42)
    model = DoubleMLP(32, [16, 8, 1])
    model.train()
    loss_fn = ns.TraversabilityLoss(w_trav=0.03, w_reco=0.5, w_temp=0.0, anomaly_balanced=balanced, model=model,
                                    method=method, confidence_std_factor=0.5, log_enabled=False, log_folder="/tmp")
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    init = {k: v.clone() for k, v in model.state_dict().items()}
    g = torch.Generator().manual_seed(5)
    rec = []
    for step in range(steps):
        x, y, yv = rows(g, step)
        graph = ns.Data(x=x, y=y, y_valid=yv)
        res = model(graph)
        loss, aux, _ = loss_fn(graph, res, step=step, log_step=False)
        opt.zero_grad()
        loss.backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters()}
        opt.step()
        cg = loss_fn._confidence_generator
        r = {"x": x, "y": y, "y_valid": yv, "res": res.detach().clone(), "loss": loss.detach().clone(),
             "loss_reco": aux["loss_reco"].detach().clone(), "loss_trav": aux["loss_trav"].detach().clone(),
             "loss_trav_confidence": aux["loss_trav_confidence"].detach().clone(), "grads": grads,
             "confidence": aux["confidence"].detach().clone(), "cg_mean": cg.mean.detach().clone(),
             "cg_std": cg.std.detach().clone(), "cg_var": cg.var.detach().clone()}
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
    DoubleMLP = sys.modules["wild_visual_navigation.model.simple_mlp"].DoubleMLP
    out = {"train": {}}
    for method, balanced in CASES:
        out["train"][(method, balanced)], model, opt, loss_fn = run(ns, DoubleMLP, method, balanced)
        if (method, balanced) == ("latest_measurement", True):
            out["checkpoint"] = {"step": 3, "model_state_dict": model.state_dict(),
                                 "optimizer_state_dict": opt.state_dict(),
                                 "traversability_loss_state_dict": loss_fn.state_dict(),
                                 "loss": out["train"][(method, balanced)]["steps"][-1]["loss"].item()}
            tmp = model.state_dict()
            tmp["confidence_generator"] = loss_fn._confidence_generator.get_dict()
            out["tmp_state_dict"] = tmp
    first = out["train"][CASES[0]]["init"]
    for case in CASES[1:]:   # the seeded init is the same for every case: stored once
        assert all(torch.equal(v, first[k]) for k, v in out["train"][case].pop("init").items())
    for D in (384, 90):
        hs = [64, 32, 1]
        torch.manual_seed(42)
        big = DoubleMLP(D, hs)
        assert hs == [64, 32, 1] and big.output_features == 1 + D
        out[f"init{D}"] = summary(big.state_dict())
        out[f"init{D}_keys"] = list(big.state_dict())
        out[f"init{D}_param_count"] = sum(p.numel() for p in big.parameters())
    torch.save(out, os.path.join(HERE, "double_mlp.pt"))
    print("wrote", os.path.join(HERE, "double_mlp.pt"))


if __name__ == "__main__":
    main()
