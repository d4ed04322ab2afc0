"""CPU tests of the LinearRnvp anomaly-detection learner: the float64 oracle (oracle/linear_rnvp.py) against goldens made
by the reference's own LinearRnvp / AnomalyLoss / torch.optim.Adam (tests/golden/make_golden_rnvp.py), the module's
state-dict layout and seeded init, the registry, the rejected options, and the reference checkpoint's format."""
import os

import pytest
import torch

from oracle import linear_rnvp as orn
from oracle.wvn_path import ConfidenceState

METHODS = ("latest_measurement", "running_mean", "moving_average", "kalman_filter")
CASES = [(m, "odds") for m in METHODS] + [("latest_measurement", "half")]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "linear_rnvp.pt"), weights_only=False)


def _init(golden, mask):
    return golden["train"][("latest_measurement", mask)]["init"]


def _d(sd):
    return {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}


def _close(a, b, rtol, atol):
    a, b = a.double(), b.double()
    return bool(((a - b).abs() <= atol + rtol * b.abs()).all())


def _replay(golden, method, mask, mutate=None):
    """The oracle's three steps from the golden's init and rows; returns per step (loss, grads, conf, cg) and the
    final state dict."""
    rec = golden["train"][(method, mask)]
    sd = _d(_init(golden, mask))
    if mutate:
        sd = mutate(sd)
    cg = ConfidenceState(0.5, method)
    adam, out = {}, []
    for st in rec["steps"]:
        x = st["x"].double()
        fwd = orn.forward(sd, x)
        sd, grads, loss, conf = orn.train_step(sd, adam, x, cg)
        out.append((fwd, loss, grads, conf, cg.mean.clone(), cg.std.clone()))
    return out, sd


def _matches(golden, method, mask, out, sd):
    rec = golden["train"][(method, mask)]
    ok = True
    for (fwd, loss, grads, conf, mean, std), st in zip(out, rec["steps"]):
        ok &= _close(fwd["log_det"], st["log_det"], 1e-5, 1e-5)
        ok &= _close(loss, st["loss"], 1e-5, 1e-5)
        for k, g in grads.items():
            ok &= _close(g, st["grads"][k], 1e-4, 1e-6 * (1 + st["grads"][k].abs().max().item()))
        ok &= _close(conf, st["confidence"], 1e-4, 1e-4)
        # running_mean's var = sum_sq / n - mean^2 with mean rounded to fp32 (confidence_generator.py:94-115): the fp32
        # rounding of mean (u |mean|) moves var by 2 u mean^2, i.e. std by u mean^2 / std; 4x that is allowed
        std_tol = 1e-5 + 4 * 2.0**-24 * float(st["cg_mean"]) ** 2 / float(st["cg_std"])
        ok &= _close(mean, st["cg_mean"], 1e-5, 1e-5) and _close(std, st["cg_std"], 0, std_tol)
    z0 = rec["steps"][0]
    if "z" in z0:
        fwd0 = out[0][0]
        ok &= _close(fwd0["z"], z0["z"], 1e-5, 1e-5) and _close(fwd0["logprob"], z0["logprob"], 1e-5, 1e-5)
    final = rec["steps"][-1]["state_dict"]
    for k, v in final.items():
        ok &= _close(sd[k], v, 0, 1e-6) if v.is_floating_point() else torch.equal(sd[k], v)
    return ok


@pytest.mark.parametrize("method,mask", CASES)
def test_oracle_reproduces_reference_training(golden, method, mask):
    out, sd = _replay(golden, method, mask)
    assert _matches(golden, method, mask, out, sd)


def test_negative_controls_fail(golden):
    """One corrupted thing each: a permutation dropped, a reversed mask.  (s and t start as copies of each other, so a
    swap of the two nets is invisible at init; the GPU tests swap them on trained weights.)"""
    def drop_perm(sd):
        sd = dict(sd)
        sd["flows.1.p"] = torch.arange(sd["flows.1.p"].numel())
        return sd

    def flip_mask(sd):
        sd = dict(sd)
        sd["flows.2.mask"] = 1 - sd["flows.2.mask"]
        return sd

    for mutate in (drop_perm, flip_mask):
        out, sd = _replay(golden, "latest_measurement", "odds", mutate)
        assert not _matches(golden, "latest_measurement", "odds", out, sd), mutate.__name__


def test_small_model_seeded_init_and_layout(golden):
    from wild_visual_navigation_b200 import LinearRnvp

    for mask in ("odds", "half"):
        torch.manual_seed(42)
        m = LinearRnvp(32, [16], mask_type=mask, conditioning_size=0, use_permutation=True, single_function=False)
        want = _init(golden, mask)
        sd = m.state_dict()
        assert list(sd) == list(want)
        for k, v in want.items():
            assert sd[k].dtype == v.dtype and torch.equal(sd[k], v), k
        # parameters are views into the flat buffer in parameters() order (the Adam state's order)
        assert m.flat_params.numel() == sum(p.numel() for p in m.parameters())
        off = 0
        for p in m.parameters():
            assert p.data_ptr() == m.flat_params.data_ptr() + 4 * off
            off += p.numel()


def test_init_384_matches_reference_summary(golden):
    from wild_visual_navigation_b200 import LinearRnvp

    torch.manual_seed(42)
    m = LinearRnvp(384, [200], mask_type="odds", conditioning_size=0, use_permutation=True, single_function=False)
    sd = m.state_dict()
    assert list(sd) == golden["init384_keys"]
    for k, s in golden["init384"].items():
        assert tuple(sd[k].shape) == s["shape"] and str(sd[k].dtype) == s["dtype"], k
        assert torch.equal(sd[k].reshape(-1)[:8], s["first"]), k
        assert abs(sd[k].double().sum().item() - s["sum"]) <= 1e-9 * max(1.0, abs(s["sum"])), k
    assert m.flat_params.numel() == 777_536 and len(list(m.parameters())) == 24


def test_get_model_and_rejected_options():
    from wild_visual_navigation_b200 import LinearRnvp, get_model

    cfg = {"input_size": 90, "coupling_topology": [200], "mask_type": "odds", "conditioning_size": 0,
           "use_permutation": True, "single_function": False}
    m = get_model({"name": "LinearRnvp", "linear_rnvp_cfg": cfg})
    assert isinstance(m, LinearRnvp) and m.input_size == 90 and m.hidden == 200
    bad = [dict(conditioning_size=4), dict(single_function=True), dict(batch_norm=True), dict(use_permutation=False),
           dict(coupling_topology=[200, 200]), dict(coupling_topology=[100, 200]), dict(coupling_topology=[]),
           dict(coupling_topology=[203]), dict(coupling_topology=[1024]), dict(mask_type="evens"), dict(flow_n=3),
           dict(input_size=1)]
    for b in bad:
        with pytest.raises(ValueError):
            LinearRnvp(**{**cfg, **b})
    with pytest.raises(NotImplementedError):
        m.sample(3)
    with pytest.raises(NotImplementedError):
        m.backward(torch.zeros(1, 90))
    with pytest.raises(RuntimeError):   # no CPU fallback
        m.forward(type("D", (), {"x": torch.zeros(2, 90)})())


def test_prior_must_be_standard_normal():
    from wild_visual_navigation_b200 import LinearRnvp

    m = LinearRnvp(16, [8], use_permutation=True)
    sd = m.state_dict()
    m.load_state_dict(sd)
    for k, v in (("prior_mean", 0.5), ("prior_var", 2.0)):
        bad = dict(sd)
        bad[k] = torch.full_like(sd[k], v)
        with pytest.raises(ValueError):
            m.load_state_dict(bad)


def test_reference_checkpoint_loads_into_model_and_loss(golden):
    from wild_visual_navigation_b200 import AnomalyLoss, LinearRnvp

    ck = golden["checkpoint"]
    assert set(ck) == {"step", "model_state_dict", "optimizer_state_dict", "traversability_loss_state_dict", "loss"}
    m = LinearRnvp(32, [16], use_permutation=True)
    loss = AnomalyLoss(0.5, "latest_measurement")
    m.load_state_dict(ck["model_state_dict"])             # strict
    loss.load_state_dict(ck["traversability_loss_state_dict"])   # strict
    assert list(loss.state_dict()) == ["_confidence_generator.mean", "_confidence_generator.var",
                                       "_confidence_generator.std"]
    ps = list(m.parameters())
    st = ck["optimizer_state_dict"]["state"]
    assert len(st) == len(ps) == 24
    assert all(st[i]["exp_avg"].shape == p.shape for i, p in enumerate(ps))
    assert torch.equal(m.flat_params[: 16 * 32].view(16, 32), ck["model_state_dict"]["flows.0.s.0.weight"])


def test_anomaly_loss_matches_oracle(golden):
    from wild_visual_navigation_b200 import AnomalyLoss

    st = golden["train"][("latest_measurement", "odds")]["steps"][0]
    res = {"logprob": st["logprob"], "log_det": st["log_det"]}
    al = AnomalyLoss(0.5, "latest_measurement")
    loss, aux, conf = al(None, res)
    assert torch.allclose(loss, st["loss"], rtol=1e-6, atol=1e-6)
    assert torch.allclose(conf, st["confidence"], atol=1e-6)
    assert aux["loss_trav"].item() == 0 and aux["loss_reco"].item() == 0
    node = type("N", (), {})()
    al.update_node_confidence(node)
    assert node.confidence == 0


def test_as_pyg_data_keeps_labelled_rows_in_anomaly_mode():
    from wild_visual_navigation_b200.traversability_estimator import MissionNode

    x = torch.arange(12.0).reshape(6, 2)
    y = torch.linspace(0, 1, 6)
    v = torch.tensor([True, False, True, True, False, False])
    n = MissionNode(x, y, v)
    d = n.as_pyg_data(anomaly_detection=True)
    assert torch.equal(d.x, x[v]) and torch.equal(d.y, y[v]) and bool(d.y_valid.all()) and d.y_valid.numel() == 3
    d = n.as_pyg_data()
    assert torch.equal(d.x, x) and torch.equal(d.y_valid, v)
