"""CPU tests of the SimpleGCN learner's restatement (oracle/simple_gcn.py) and its Python surface: the float64 oracle
reproduces tests/golden/gcn.pt (made by the reference's own simple_gcn.py with the restated GCNConv, its
TraversabilityLoss, Batch and Adam), the aggregation is the directed D^-1/2 (A + I) D^-1/2, and the model's keys,
init and bounds are the reference's."""
import os

import pytest
import torch

from oracle import simple_gcn as og
from oracle.wvn_path import ConfidenceState

METHODS = ("latest_measurement", "running_mean", "moving_average", "kalman_filter")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "gcn.pt"), weights_only=False)


def _close(a, b, rtol=2e-4, atol=1e-6):
    a, b = a.double(), b.double()
    assert torch.allclose(a, b, rtol=rtol, atol=atol), (a - b).abs().max().item()


def _replay(init, data, method, steps=3):
    sd = {k: v.double() for k, v in init.items()}
    cg, adam, out = ConfidenceState(0.5, method), {}, []
    for step in range(steps):
        x, ei, y, yv = data(step)
        res = og.forward(sd, x.double(), ei)
        sd, grads, loss, aux = og.train_step(sd, adam, x.double(), ei, y, yv, cg)
        out.append((res, grads, loss, aux, {k: v.clone() for k, v in sd.items()}, cg.mean.clone(), cg.std.clone()))
    return out


@pytest.mark.parametrize("method", METHODS)
def test_oracle_reproduces_graph_pt_goldens(golden, method):
    g = golden["graph"]
    assert g["x"].shape == (100, 90) and g["edge_index"].shape == (2, 384) and int(g["y_valid"].sum()) == 16
    init = golden["train"]["latest_measurement"]["init"]
    assert list(init) == og.keys()
    rec = golden["train"][method]["steps"]
    got = _replay(init, lambda s: (g["x"], g["edge_index"], g["y"], g["y_valid"]), method)
    for s, (res, grads, loss, aux, sd, mean, std) in enumerate(got):
        r = rec[s]
        if s == 0:
            _close(res, r["res"])
        _close(loss, r["loss"])
        _close(aux["confidence"], r["confidence"], atol=1e-4)
        _close(mean, r["cg_mean"]), _close(std, r["cg_std"])
        for k in og.keys():
            _close(grads[k], r["grads"][k], atol=1e-7)
    for k, v in rec[-1]["state_dict"].items():
        _close(got[-1][4][k], v, atol=1e-6)


def test_oracle_reproduces_synthetic_batch(golden):
    nodes, eis = golden["synthetic_nodes"], golden["synthetic_edge_index"]

    def data(s):
        x = torch.cat([d["x"] for d in nodes[s]])
        return x, eis[s], torch.cat([d["y"] for d in nodes[s]]), torch.cat([d["y_valid"] for d in nodes[s]])

    # the batch offsets each node's edges by its first row; the empty node adds none
    assert eis[0].shape[1] == 4 + 5 + 0 + 15 and eis[0][:, 4:9].min() == 7
    rec = golden["synthetic"]["steps"]
    got = _replay(golden["synthetic"]["init"], data, "latest_measurement")
    for s, (res, grads, loss, aux, sd, mean, std) in enumerate(got):
        _close(loss, rec[s]["loss"])
        for k in og.keys():
            _close(grads[k], rec[s]["grads"][k], atol=1e-7)


def test_aggregation_is_the_directed_normalised_adjacency():
    g = torch.Generator().manual_seed(3)
    n = 9
    ei = torch.tensor([[0, 1, 2, 2, 1, 5, 5, 7, 4], [1, 2, 1, 1, 1, 6, 4, 8, 5]])   # dup 2->1, loop 1->1, 3 isolated
    y = torch.randn(n, 5, generator=g, dtype=torch.float64)
    A = torch.zeros(n, n, dtype=torch.float64)
    for s, d in ei.t().tolist():
        if s != d:
            A[d, s] += 1.0          # row = target: a node aggregates from its sources
    Ah = A + torch.eye(n, dtype=torch.float64)
    dinv = Ah.sum(1).pow(-0.5)      # 1 + in-degree
    dense = dinv[:, None] * Ah * dinv[None, :]
    assert torch.allclose(og.aggregate(y, ei), dense @ y, atol=1e-14)
    # negative controls: symmetrised edges, the input's self-loop kept, the degree taken at the source
    sym = torch.cat([ei, ei.flip(0)], 1)
    assert not torch.allclose(og.aggregate(y, sym), dense @ y, atol=1e-6)
    dsrc = (A.sum(0) + 1).pow(-0.5)
    assert not torch.allclose(dsrc[:, None] * Ah * dsrc[None, :] @ y, dense @ y, atol=1e-6)
    Al = Ah.clone()
    Al[1, 1] += 1.0
    dl = Al.sum(1).pow(-0.5)
    assert not torch.allclose(dl[:, None] * Al * dl[None, :] @ y, dense @ y, atol=1e-6)


def test_two_rank_decomposition_equals_the_global_batch(golden):
    """Frames sharded over two ranks: the statistic sums and the gradient, each summed over the ranks, give the global
    batch's step (the per-rank loss is formed with the global counts and the generator update of the global sums)."""
    nodes = golden["synthetic_nodes"][0]
    sd = {k: v.double() for k, v in golden["synthetic"]["init"].items()}
    frames = [(d["x"].double(), d["edge_index"], d["y"].double(), d["y_valid"]) for d in nodes]

    def batch(fs):
        xs, eis, off = [], [], 0
        for x, ei, _, _ in fs:
            xs.append(x)
            eis.append(ei + off)
            off += x.shape[0]
        return (torch.cat(xs), torch.cat(eis, 1), torch.cat([f[2] for f in fs]), torch.cat([f[3] for f in fs]))

    x, ei, y, yv = batch(frames)
    _, g_all, loss_all, aux = og.train_step(sd, {}, x, ei, y, yv, ConfidenceState(0.5))
    conf = aux["confidence"]
    D, N, NV = x.shape[1], x.shape[0], int(yv.sum())

    def rank_grads(fs, rows):
        xr, er, yr, vr = batch(fs)
        p = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
        res = og.forward(p, xr, er)
        lr = ((res[:, 1:] - xr) ** 2).mean(1)
        raw = (res[:, 0] - yr) ** 2
        w = torch.where(vr, torch.ones_like(raw), 1 - conf[rows])
        loss = 0.03 * (raw * w).sum() / N + 0.5 * lr[vr].sum() / NV
        loss.backward()
        return {k: v.grad for k, v in p.items()}, loss.detach()

    n0 = sum(f[0].shape[0] for f in frames[:2])
    ga, la = rank_grads(frames[:2], slice(0, n0))
    gb, lb = rank_grads(frames[2:], slice(n0, N))
    assert abs((la + lb) - loss_all).item() < 1e-12
    for k in g_all:
        assert torch.allclose(ga[k] + gb[k], g_all[k], atol=1e-12)


def test_model_keys_init_and_config(golden):
    from wild_visual_navigation_b200 import SimpleGCN, get_model
    from wild_visual_navigation_b200.traversability_estimator.traversability_estimator import default_params

    cfg = default_params()["model"]["simple_gcn_cfg"]
    assert cfg == {"input_size": 384, "reconstruction": True, "hidden_sizes": [256, 128, 1]}
    for D in (384, 90):
        torch.manual_seed(42)
        hs = [256, 128, 1]
        m = get_model({"name": "SimpleGCN", "simple_gcn_cfg": {"input_size": D, "reconstruction": True,
                                                                "hidden_sizes": hs}})
        assert hs == [256, 128, 1]   # unlike SimpleMLP, the caller's list is left alone
        assert isinstance(m, SimpleGCN) and m.shape_error() is None
        sd = m.state_dict()
        assert list(sd) == golden[f"init{D}_keys"] == og.keys()
        assert m.flat_params.numel() == golden[f"init{D}_param_count"]
        for k, s in golden[f"init{D}"].items():
            assert tuple(sd[k].shape) == s["shape"] and torch.equal(sd[k].reshape(-1)[:8], s["first"])
            assert abs(sd[k].double().sum().item() - s["sum"]) < 1e-9
        want = og.init(D, [256, 128, 1])
        assert all(torch.equal(sd[k], want[k]) for k in want)
    assert golden["init384_param_count"] == 181121
    # parameters are views into the flat buffer in parameters() order, and the reference checkpoint loads strictly
    m = SimpleGCN(90, True, [32, 16, 1])
    m.load_state_dict(golden["checkpoint"]["model_state_dict"])
    off = 0
    for p in m.parameters():
        assert p.data_ptr() == m.flat_params.data_ptr() + 4 * off
        off += p.numel()
    assert len(golden["checkpoint"]["optimizer_state_dict"]["state"]) == 6
    with pytest.raises(ValueError, match="outside the H100 hot path"):
        get_model({"name": "GAT"})


@pytest.mark.parametrize("args, what", [((8, False, [4, 4, 1]), "reconstruction"), ((8, True, [4, 1]), "hidden_sizes"),
                                        ((8, True, [4, 4, 2]), "hidden_sizes"), ((1025, True, [4, 4, 1]), "range"),
                                        ((8, True, [513, 4, 1]), "range"), ((8, True, [4, 0, 1]), "range")])
def test_unsupported_shapes_raise(args, what):
    from wild_visual_navigation_b200 import SimpleGCN

    m = SimpleGCN(*args)   # builds for any shape, as upstream
    assert what in m.shape_error()
    with pytest.raises(ValueError):
        m.check_supported()


def test_missing_edges_raise():
    from wild_visual_navigation_b200 import SimpleGCN
    from wild_visual_navigation_b200.traversability_estimator import MissionNode

    m = SimpleGCN(8, True, [4, 4, 1])
    n = MissionNode(torch.zeros(3, 8), torch.zeros(3), torch.zeros(3, dtype=torch.bool))
    assert n.as_pyg_data().edge_index is None
    n.feature_edges = torch.tensor([[0], [1]])
    assert torch.equal(n.as_pyg_data().edge_index, n.feature_edges)
    with pytest.raises(ValueError):
        m.forward(n.as_pyg_data())   # on the CPU: no fallback
    from wild_visual_navigation_b200 import ops

    with pytest.raises(ValueError, match="edge_index"):
        ops._graph_as_padded(torch.zeros(3, 8), None)
    with pytest.raises(ValueError, match="edges"):
        ops._check_edges(torch.zeros(2, 4, 3, dtype=torch.long), torch.zeros(2, dtype=torch.int32), 2)
    with pytest.raises(ValueError, match="n_edges"):
        ops._check_edges(torch.zeros(2, 4, 2, dtype=torch.long), torch.zeros(2, dtype=torch.int64), 2)
