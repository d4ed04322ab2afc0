"""CPU tests of the DoubleMLP learner: the float64 oracle (oracle/double_mlp.py) against goldens made by the
reference's own DoubleMLP / TraversabilityLoss / torch.optim.Adam (tests/golden/make_golden_double_mlp.py), the
module's state-dict layout and seeded init, the registry, and the shapes and options that are refused."""
import os

import pytest
import torch

from oracle import double_mlp as odm
from oracle.wvn_path import ConfidenceState

METHODS = ("latest_measurement", "running_mean", "moving_average", "kalman_filter")
CASES = [(m, True) for m in METHODS] + [("latest_measurement", False)]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "double_mlp.pt"), weights_only=False)


def _init(golden):
    return golden["train"][CASES[0]]["init"]


def _close(a, b, rtol, atol):
    a, b = a.double(), b.double()
    return bool(((a - b).abs() <= atol + rtol * b.abs()).all())


def _replay(golden, method, balanced, grad_scale=None):
    """The oracle's three steps from the golden's init and rows (float64)."""
    sd = {k: v.double() for k, v in _init(golden).items()}
    cg, adam, out = ConfidenceState(0.5, method), {}, []
    for st in golden["train"][(method, balanced)]["steps"]:
        res = odm.forward(sd, st["x"].double())
        sd, grads, loss, aux = odm.train_step(sd, adam, st["x"].double(), st["y"], st["y_valid"], cg,
                                              anomaly_balanced=balanced)
        if grad_scale:
            grads[grad_scale] = grads[grad_scale] * 1.01
        out.append((res, loss, aux, grads))
    return out, sd


def _matches(golden, method, balanced, out, sd):
    ok = True
    for (res, loss, aux, grads), st in zip(out, golden["train"][(method, balanced)]["steps"]):
        ok &= _close(res, st["res"], 1e-5, 1e-6)
        ok &= _close(loss, st["loss"], 1e-5, 1e-7)
        for k in ("loss_reco", "loss_trav", "loss_trav_confidence"):
            ok &= _close(aux[k], st[k], 1e-5, 1e-7)
        for k, g in grads.items():
            ok &= _close(g, st["grads"][k], 1e-4, 1e-6 * (1 + st["grads"][k].abs().max().item()))
        ok &= _close(aux["confidence"], st["confidence"], 1e-4, 1e-4)
        std_tol = 1e-5 + 4 * 2.0**-24 * float(st["cg_mean"]) ** 2 / float(st["cg_std"])
        ok &= _close(aux["mean"], st["cg_mean"], 1e-5, 1e-6) and _close(aux["std"], st["cg_std"], 0, std_tol)
    # Adam's step m / (sqrt(v) + eps) is insensitive to a gradient's size except where |g| is near eps = 1e-8: there the
    # fp32 and float64 gradients (relative difference ~1e-4 at such tiny sizes) move a parameter differently by up to
    # ~lr * 1e-3 per step
    for k, v in golden["train"][(method, balanced)]["steps"][-1]["state_dict"].items():
        ok &= _close(sd[k], v, 0, 5e-6)
    return ok


@pytest.mark.parametrize("method,balanced", CASES)
def test_oracle_reproduces_reference_training(golden, method, balanced):
    out, sd = _replay(golden, method, balanced)
    assert _matches(golden, method, balanced, out, sd)


def test_negative_controls_fail(golden):
    """A scaled bias gradient and swapped networks each break the match."""
    out, sd = _replay(golden, *CASES[0], grad_scale="networks.1.2.bias")
    assert not _matches(golden, *CASES[0], out, sd)
    swapped = {k.replace("networks.0", "networks.T").replace("networks.1", "networks.0").replace("networks.T", "networks.1"): v
               for k, v in _init(golden).items() if not k.startswith("networks.0.4") and not k.startswith("networks.1.4")}
    sd0 = {k: v.double() for k, v in _init(golden).items()}
    sd0.update({k: v.double() for k, v in swapped.items()})
    x = golden["train"][CASES[0]]["steps"][0]["x"].double()
    assert not _close(odm.forward(sd0, x), golden["train"][CASES[0]]["steps"][0]["res"], 1e-3, 1e-3)


@pytest.mark.parametrize("D", [384, 90])
def test_module_layout_and_seeded_init(golden, D):
    """get_model builds the reference's module: keys in order, shapes, seed-42 init bit for bit, output_features,
    and the caller's hidden_sizes untouched."""
    from wild_visual_navigation_b200 import DoubleMLP, get_model

    hs = [64, 32, 1]
    torch.manual_seed(42)
    m = get_model({"name": "DoubleMLP", "double_mlp_cfg": {"input_size": D, "hidden_sizes": hs}})
    assert isinstance(m, DoubleMLP) and hs == [64, 32, 1] and m.output_features == 1 + D
    sd = m.state_dict()
    assert list(sd) == golden[f"init{D}_keys"] == odm.keys()
    assert sum(p.numel() for p in m.parameters()) == golden[f"init{D}_param_count"] == m.flat_params.numel()
    ref_sd = odm.init(D, hs)
    for k, s in golden[f"init{D}"].items():
        assert tuple(sd[k].shape) == s["shape"]
        assert torch.equal(sd[k].reshape(-1)[:8], s["first"]) and sd[k].double().sum().item() == s["sum"]
        assert torch.equal(ref_sd[k], sd[k])
    # every parameter is a view of flat_params, in parameters() order, also after a move (.to rebuilds the buffer)
    for mm in (m, m.to(torch.float32).to("cpu")):
        off = 0
        for p in mm.parameters():
            assert p.data_ptr() == mm.flat_params.data_ptr() + 4 * off
            off += p.numel()


def test_default_params_carry_the_reference_double_mlp_cfg():
    from wild_visual_navigation_b200.traversability_estimator.traversability_estimator import default_params

    assert default_params()["model"]["double_mlp_cfg"] == {"input_size": 384, "hidden_sizes": [64, 32, 1]}


@pytest.mark.parametrize("D,hs", [(32, [16, 8, 2]), (32, [16, 1]), (32, [16, 8, 4, 1]), (1100, [16, 8, 1]),
                                  (32, [18, 8, 1]), (32, [260, 8, 1]), (32, [16, 33, 1])])
def test_unsupported_shapes_are_refused(D, hs):
    """The module can be built (as in the reference), but the trainer and the inference handle refuse the shape."""
    from wild_visual_navigation_b200 import DoubleMLP, ops

    m = DoubleMLP(D, hs)
    assert m.shape_error() is not None
    with pytest.raises(ValueError):
        ops.DoubleMlpTrainer(m)
    with pytest.raises(ValueError):
        m.check_supported()


def test_cpu_parameters_are_refused():
    from wild_visual_navigation_b200 import DoubleMLP, ops

    m = DoubleMLP(32, [16, 8, 1])
    assert m.shape_error() is None
    with pytest.raises(ValueError):
        ops.DoubleMlpTrainer(m)


def test_process_group_is_refused():
    from wild_visual_navigation_b200 import TraversabilityEstimator
    from wild_visual_navigation_b200.traversability_estimator.traversability_estimator import default_params

    p = default_params()
    p["model"]["name"] = "DoubleMLP"
    with pytest.raises(ValueError, match="process_group"):
        TraversabilityEstimator(params=p, process_group=object())


def test_reference_checkpoint_format(golden):
    """The reference's checkpoint: model keys, Adam state over the 12 tensors in parameters() order, and the loss
    state dict carrying the model as ``_model.networks.*`` next to the generator."""
    ck = golden["checkpoint"]
    assert list(ck["model_state_dict"]) == odm.keys()
    st = ck["optimizer_state_dict"]["state"]
    assert sorted(st) == list(range(12))
    for i, k in enumerate(odm.keys()):
        assert st[i]["exp_avg"].shape == ck["model_state_dict"][k].shape
    lk = list(ck["traversability_loss_state_dict"])
    assert [k for k in lk if k.startswith("_model.")] == ["_model." + k for k in odm.keys()]
    assert any(k.startswith("_confidence_generator.") for k in lk)
    assert list(golden["tmp_state_dict"])[-2] == "networks.1.4.bias"
