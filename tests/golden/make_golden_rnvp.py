"""Generate tests/golden/linear_rnvp.pt by running the REFERENCE's own LinearRnvp, AnomalyLoss and torch.optim.Adam.

Run with a checkout of the reference repository:
``WVN_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_rnvp.py``

  * ``LinearRnvp(32, [16], mask_type=m, use_permutation=True)`` under ``seed_everything(42)``-equivalent seeding, three
    ``TraversabilityEstimator.train()`` bodies (model forward, AnomalyLoss, zero_grad / backward / Adam step, lr 1e-3)
    on seeded rows, per ConfidenceGenerator method (mask "odds"; latest_measurement also with mask "half"): per step the
    loss, log_det, gradients, confidence and generator state, the forward outputs of step 0 and the state dict
    after the last step;
  * one checkpoint in the reference's on-disk format (``save_checkpoint``: step, model / optimizer / loss state dicts);
  * the init summary (per key: sum and first 8 elements) of ``LinearRnvp(384, [200])`` under seed 42.
"""
from __future__ import annotations

import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402

CFG = dict(coupling_topology=[16], conditioning_size=0, use_permutation=True, single_function=False)
METHODS = ("latest_measurement", "running_mean", "moving_average", "kalman_filter")


def seed_everything(seed):
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)


def load():
    ns = ref_import.load()
    rnvp = ref_import._load("wild_visual_navigation.model.linear_rnvp", "wild_visual_navigation/model/linear_rnvp.py")
    loss = sys.modules["wild_visual_navigation.utils.loss"]
    return ns, rnvp.LinearRnvp, loss.AnomalyLoss


def run(LinearRnvp, AnomalyLoss, Data, method, mask_type, steps=3):
    seed_everything(42)
    model = LinearRnvp(input_size=32, mask_type=mask_type, **CFG)
    model.train()
    loss_fn = AnomalyLoss(confidence_std_factor=0.5, method=method, log_enabled=False, log_folder="/tmp")
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    init = {k: v.clone() for k, v in model.state_dict().items()}
    g = torch.Generator().manual_seed(7)
    rec = []
    for step in range(steps):
        x = torch.randn(24 + 4 * step, 32, generator=g) * 0.7 + 0.2
        res = model(Data(x=x))
        loss, aux, conf = loss_fn(Data(x=x), res, step=step)
        opt.zero_grad()
        loss.backward()
        grads = {k: p.grad.clone() for k, p in model.named_parameters()}
        opt.step()
        cg = loss_fn._confidence_generator
        r = {"x": x, "log_det": res["log_det"].detach().clone(), "loss": loss.detach().clone(), "grads": grads,
             "confidence": conf.clone(), "cg_mean": cg.mean.detach().clone(), "cg_std": cg.std.detach().clone(),
             "cg_var": cg.var.detach().clone()}
        if step == 0:   # the forward outputs once; the parameters after the last step (fixtures stay small)
            r["z"], r["logprob"] = res["z"].detach().clone(), res["logprob"].detach().clone()
        if step == steps - 1:
            r["state_dict"] = {k: v.clone() for k, v in model.state_dict().items()}
        rec.append(r)
    return {"init": init, "steps": rec}, model, opt, loss_fn


def main():
    assert ref_import.available(), "set WVN_REFERENCE_ROOT to a reference checkout"
    ns, LinearRnvp, AnomalyLoss = load()
    out = {"train": {}}
    for method in METHODS:
        out["train"][(method, "odds")], model, opt, loss_fn = run(LinearRnvp, AnomalyLoss, ns.Data, method, "odds")
        if method == "latest_measurement":
            out["checkpoint"] = {"step": 3, "model_state_dict": model.state_dict(),
                                 "optimizer_state_dict": opt.state_dict(),
                                 "traversability_loss_state_dict": loss_fn.state_dict(),
                                 "loss": out["train"][(method, "odds")]["steps"][-1]["loss"].item()}
    out["train"][("latest_measurement", "half")] = run(LinearRnvp, AnomalyLoss, ns.Data, "latest_measurement", "half")[0]
    for method in METHODS[1:]:   # the seeded init is the same for every method: stored once per mask type
        assert all(torch.equal(v, out["train"][(METHODS[0], "odds")]["init"][k])
                   for k, v in out["train"][(method, "odds")].pop("init").items())
    seed_everything(42)
    big = LinearRnvp(input_size=384, mask_type="odds", coupling_topology=[200], conditioning_size=0,
                     use_permutation=True, single_function=False)
    out["init384"] = {k: {"shape": tuple(v.shape), "dtype": str(v.dtype), "sum": v.double().sum().item(),
                          "first": v.reshape(-1)[:8].clone()} for k, v in big.state_dict().items()}
    out["init384_keys"] = list(big.state_dict())
    torch.save(out, os.path.join(HERE, "linear_rnvp.pt"))
    print("wrote", os.path.join(HERE, "linear_rnvp.pt"))


if __name__ == "__main__":
    main()
