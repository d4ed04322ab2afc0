"""GPU tests of the SimpleGCN learner (csrc/gcn_train.cu): the graph build, forward and train step against the float64
oracle (oracle/simple_gcn.py) and the goldens of tests/golden/gcn.pt, the padded entry against the compacted one bit for
bit, determinism, the edge cases of the per-frame graphs, and the Python surface (estimator, checkpoints, inference)."""
import os

import pytest
import torch

from oracle import simple_gcn as og
from oracle.wvn_path import ConfidenceState

pytestmark = pytest.mark.gpu

METHODS = ("latest_measurement", "running_mean", "moving_average", "kalman_filter")
METHOD_ID = {m: i for i, m in enumerate(("latest_measurement", "running_mean", "kalman_filter", "moving_average"))}


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "gcn.pt"), weights_only=False)


def _model(D, h1, h2, sd=None, seed=42):
    from wild_visual_navigation_b200 import SimpleGCN

    torch.manual_seed(seed)
    m = SimpleGCN(D, True, [h1, h2, 1])
    if sd is not None:
        m.load_state_dict(sd)
    return m.cuda()


def _trainer(m, method="latest_measurement", **kw):
    from wild_visual_navigation_b200 import ops

    t = ops.GcnTrainer(m, **kw)
    t.set_confidence(METHOD_ID[method])
    return t


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-30)).item()


def _frames(G, S, D, seed, density=3.8, emax=None, n_rows=None):
    """G padded frames of up to S rows with random directed edges (local ids, ~density per row), some out of range and
    some self-loops; NaN padding rows.  Returns feat, n_rows, edges [G, emax, 2] int64, n_edges, y, y_valid."""
    g = torch.Generator().manual_seed(seed)
    n = n_rows if n_rows is not None else torch.randint(1, S + 1, (G,), generator=g)
    emax = emax or max(1, int(density * S))
    feat = torch.full((G, S, D), float("nan"))
    edges = torch.full((G, emax, 2), -7, dtype=torch.long)
    ne = torch.zeros(G, dtype=torch.int32)
    for f in range(G):
        k = int(n[f])
        feat[f, :k] = torch.randn(k, D, generator=g) * 0.8 + 0.1
        m = min(emax, int(density * k))
        e = torch.randint(0, k, (m, 2), generator=g)
        if m > 4:
            e[0, 1] = e[0, 0]            # a self-loop (dropped)
            e[1] = torch.tensor([0, k])  # target out of range (dropped)
        edges[f, :m] = e
        ne[f] = m
    N = int(n.sum())
    yv = torch.rand(N, generator=g) < 0.3
    yv[:2] = True   # the generator's std needs two labelled rows
    y = torch.where(yv, torch.rand(N, generator=g).clamp(min=0.001), torch.zeros(N))
    return feat, n.to(torch.int32), edges, ne, y, yv


def _cuda(*ts):
    return [t.cuda() for t in ts]


def _dense_forward(sd, x, ei, keep_loops=False, deg_at_source=False):
    """SimpleGCN's forward with a dense D^-1/2 (A + I) D^-1/2; the options build the wrong variants the negative
    controls need (the input's self-loops kept, the degree taken at the source)."""
    n = x.shape[0]
    A = torch.zeros(n, n, dtype=torch.float64)
    for s, d in ei.t().tolist():
        if s != d or keep_loops:
            A[d, s] += 1.0
    Ah = A + torch.eye(n, dtype=torch.float64)
    dinv = (Ah.sum(0) if deg_at_source else Ah.sum(1)).pow(-0.5)
    Mx = dinv[:, None] * Ah * dinv[None, :]
    h = x
    for j in range(3):
        h = Mx @ (h @ sd[f"layers.{j}.lin.weight"].t()) + sd[f"layers.{j}.bias"]
        if j < 2:
            h = torch.relu(h)
    return torch.cat([torch.sigmoid(h[:, :1]), h[:, 1:]], 1)


@pytest.mark.parametrize("method", METHODS)
def test_step_on_graph_pt_matches_goldens_and_float64(golden, method):
    g = golden["graph"]
    init = golden["train"]["latest_measurement"]["init"]
    rec = golden["train"][method]["steps"]
    m = _model(90, 32, 16, init)
    tr = _trainer(m, method)
    x, ei, y, yv = _cuda(g["x"], g["edge_index"], g["y"], g["y_valid"])
    sd64, cg, adam = {k: v.double() for k, v in init.items()}, ConfidenceState(0.5, method), {}
    for s in range(3):
        p0 = m.flat_params.clone()
        conf = tr.step(x, ei, y, yv)
        mt = tr.metrics.tolist()
        new64, g64, loss64, aux64 = og.train_step(sd64, adam, g["x"].double(), g["edge_index"], g["y"], g["y_valid"], cg)
        # gradient, in parameters() order
        grads = torch.cat([g64[k].reshape(-1) for k in og.keys()])
        assert _rel(tr.grads, grads) < 2e-4, (s, _rel(tr.grads, grads))
        assert abs(mt[0] - loss64.item()) <= 2e-5 * abs(loss64.item()) + 1e-7
        assert abs(mt[0] - rec[s]["loss"].item()) <= 2e-5 * abs(rec[s]["loss"].item()) + 1e-7
        assert (conf.cpu().double() - aux64["confidence"].double()).abs().max() < 2e-4
        assert abs(mt[4] - rec[s]["cg_mean"].item()) <= 1e-4 * abs(rec[s]["cg_mean"].item()) + 1e-7
        assert mt[6] == 0.0
        step = m.flat_params - p0
        want = torch.cat([(new64[k] - sd64[k]).reshape(-1) for k in og.keys()])
        assert _rel(step, want) < 2e-3
        sd64 = new64
    for k, v in rec[-1]["state_dict"].items():
        assert (m.state_dict()[k].cpu() - v).abs().max() < 1e-5


def test_synthetic_batch_matches_goldens(golden):
    from wild_visual_navigation_b200.traversability_estimator import MissionNode

    nodes, rec = golden["synthetic_nodes"], golden["synthetic"]["steps"]
    m = _model(24, 16, 8, golden["synthetic"]["init"])
    tr = _trainer(m)
    for s in range(3):
        # the same batch through MissionNode.as_pyg_data and Batch.from_data_list
        from wild_visual_navigation_b200 import Batch

        b = Batch.from_data_list([MissionNode(d["x"].cuda(), d["y"].cuda(), d["y_valid"].cuda(),
                                              feature_edges=d["edge_index"].cuda()).as_pyg_data() for d in nodes[s]])
        assert torch.equal(b.edge_index.cpu(), golden["synthetic_edge_index"][s])
        tr.step(b.x, b.edge_index, b.y, b.y_valid)
        grads = torch.cat([rec[s]["grads"][k].reshape(-1) for k in og.keys()])
        assert _rel(tr.grads, grads) < 2e-4
        assert abs(tr.metrics[0].item() - rec[s]["loss"].item()) <= 2e-5 * rec[s]["loss"].item()


@pytest.mark.parametrize("G, S, D, h1, h2", [(3, 1, 8, 4, 4), (3, 17, 33, 16, 8), (8, 100, 90, 32, 16),
                                              (41, 100, 384, 256, 128), (2, 2048, 64, 64, 32), (4, 96, 1024, 512, 512)])
def test_padded_step_matches_float64_and_compacted_bitwise(G, S, D, h1, h2):
    feat, n_rows, edges, ne, y, yv = _frames(G, S, D, seed=G * 1000 + S)
    x64, ei = og.padded_to_graph(feat.double(), n_rows, edges, ne)
    sd = {k: v.cpu().clone() for k, v in _model(D, h1, h2).state_dict().items()}
    sd64 = {k: v.double() for k, v in sd.items()}
    # the padded step
    m = _model(D, h1, h2, sd)
    tr = _trainer(m, max_rows=16, max_edges=16)   # grows on demand
    fc, nc, ec, nec, yc, yvc = _cuda(feat, n_rows, edges, ne, y, yv)
    conf = tr.step_padded(fc, nc, ec, nec, yc, yvc)
    _, g64, loss64, aux64 = og.train_step(sd64, {}, x64, ei, y.double(), yv, ConfidenceState(0.5))
    grads = torch.cat([g64[k].reshape(-1) for k in og.keys()])
    assert _rel(tr.grads, grads) < 5e-4, _rel(tr.grads, grads)
    assert abs(tr.metrics[0].item() - loss64.item()) <= 5e-5 * abs(loss64.item())
    N = x64.shape[0]
    assert (conf[:N].cpu().double() - aux64["confidence"]).abs().max() < 1e-3
    padded = (m.flat_params.clone(), tr.grads.clone(), tr.metrics.clone(), conf[:N].clone())
    # the same rows compacted, with the edges offset: bit-identical
    m2 = _model(D, h1, h2, sd)
    tr2 = _trainer(m2)
    conf2 = tr2.step(x64.float().cuda(), ei.cuda(), y.cuda(), yv.cuda())
    assert torch.equal(padded[0], m2.flat_params) and torch.equal(padded[1], tr2.grads)
    assert torch.equal(padded[2], tr2.metrics) and torch.equal(padded[3], conf2)
    # two runs bit-identical
    m3 = _model(D, h1, h2, sd)
    tr3 = _trainer(m3)
    tr3.step_padded(fc, nc, ec, nec, yc, yvc)
    assert torch.equal(padded[1], tr3.grads) and torch.equal(padded[0], m3.flat_params)


def test_graph_edge_cases_and_overflow_flag():
    """Frames with no edges, one row, every edge slot used, input self-loops, rows with only in- or only out-edges,
    edges out of range, dead rows between frames, and a negative edge count (overflow): the forward against float64."""
    from wild_visual_navigation_b200 import ops

    D, S, E = 12, 6, 8
    feat = torch.full((5, S, D), float("nan"))
    n_rows = torch.tensor([4, 1, 6, 0, 3], dtype=torch.int32)
    edges = torch.full((5, E, 2), 99, dtype=torch.long)
    ne = torch.tensor([0, 2, 8, 0, 3], dtype=torch.int32)
    edges[1, :2] = torch.tensor([[0, 0], [0, 1]])                                   # self-loop, out of range
    edges[2] = torch.tensor([[0, 1], [0, 2], [0, 3], [3, 3], [4, 1], [1, 5], [5, 1], [-1, 2]])  # E full
    edges[4, :3] = torch.tensor([[2, 0], [2, 1], [2, 0]])                           # 2 only out, duplicate
    g = torch.Generator().manual_seed(0)
    for f in range(5):
        feat[f, : n_rows[f]] = torch.randn(int(n_rows[f]), D, generator=g)
    m = _model(D, 8, 4)
    inf = ops.GcnInference(m)
    sd64 = {k: v.double().cpu() for k, v in m.state_dict().items()}
    x64, ei = og.padded_to_graph(feat.double(), n_rows, edges, ne)
    want = og.forward(sd64, x64, ei)
    fc, nc, ec, nec = _cuda(feat, n_rows, edges, ne)
    out, trav, conf = inf._run(fc, 5, S, nc, ec, E, nec, torch.zeros(1).cuda(), torch.ones(1).cuda(), 0.5,
                               want_out=True)
    N = x64.shape[0]
    assert (out[:N].cpu().double() - want).abs().max() < 1e-5
    live = torch.arange(S)[None, :] < n_rows[:, None].long()
    assert torch.equal(trav.view(5, S).cpu()[live], out[:N, 0].cpu())
    assert torch.isnan(trav.view(5, S).cpu()[~live]).all()
    # negative controls: reversed edges, the input self-loop kept, degree at the source
    got = out[:N].cpu().double()
    assert (got - og.forward(sd64, x64, ei.flip(0))).abs().max() > 1e-3
    assert (got - _dense_forward(sd64, x64, ei, keep_loops=True)).abs().max() > 1e-3
    assert (got - _dense_forward(sd64, x64, ei, deg_at_source=True)).abs().max() > 1e-3
    assert (got - _dense_forward(sd64, x64, ei)).abs().max() < 1e-5   # the dense form itself agrees
    # overflow: frame 2's count negative -> its edges are not read (the forward equals the oracle's without them)
    ne_bad = ne.clone()
    ne_bad[2] = -3
    out_bad, _, _ = inf._run(fc, 5, S, nc, ec, E, ne_bad.cuda(), want_out=True, want_rows=False)
    _, ei_bad = og.padded_to_graph(feat.double(), n_rows, edges, ne_bad)
    assert (out_bad[:N].cpu().double() - og.forward(sd64, x64, ei_bad)).abs().max() < 1e-5
    assert (out_bad[:N].cpu().double() - got).abs().max() > 1e-3
    # ... and the trainer flags it in metrics[6]
    tr = _trainer(m)
    ne_bad = ne.clone()
    ne_bad[2] = -3
    N = int(n_rows.sum())
    y, yv = torch.rand(N).cuda(), torch.ones(N, dtype=torch.bool).cuda()
    tr.step_padded(fc, nc, ec, ne_bad.cuda(), y, yv)
    assert tr.metrics[6].item() == 1.0
    tr.step_padded(fc, nc, ec, nec, y, yv)
    assert tr.metrics[6].item() == 0.0


def test_dead_units_get_exact_zero_gradient():
    D, h1, h2 = 16, 8, 4
    m = _model(D, h1, h2)
    with torch.no_grad():
        m.layers[0].bias[:3] = -1e4     # units 0..2 of layer 1 never fire
        m.layers[1].bias[0] = -1e4
    feat, n_rows, edges, ne, y, yv = _frames(3, 20, D, seed=5)
    tr = _trainer(m)
    tr.step_padded(*_cuda(feat, n_rows, edges, ne, y, yv))
    o, off = {}, 0
    for k, p in m.state_dict().items():
        o[k] = tr.grads[off : off + p.numel()].view_as(p)
        off += p.numel()
    assert torch.all(o["layers.0.lin.weight"][:3] == 0) and torch.all(o["layers.0.bias"][:3] == 0)
    assert torch.all(o["layers.1.lin.weight"][0] == 0) and o["layers.1.bias"][0] == 0
    assert torch.all(o["layers.1.lin.weight"][:, :3] == 0)   # inputs from dead units
    assert torch.all(o["layers.0.lin.weight"][3:].abs().sum(1) > 0)


def _params(name="SimpleGCN"):
    from wild_visual_navigation_b200.traversability_estimator.traversability_estimator import default_params

    p = default_params()
    p["model"]["name"] = name
    p["model"]["simple_gcn_cfg"] = {"input_size": 90, "reconstruction": True, "hidden_sizes": [32, 16, 1]}
    return p


def test_estimator_trains_checkpoints_and_hands_off(golden, tmp_path):
    from wild_visual_navigation_b200 import TraversabilityEstimator, TraversabilityInference
    from wild_visual_navigation_b200.traversability_estimator import MissionNode

    g = golden["graph"]
    te = TraversabilityEstimator(params=_params(), device="cuda", min_samples_for_training=0)
    assert list(te._model.state_dict()) == og.keys()
    te.add_mission_node(MissionNode(g["x"].cuda(), g["y"].cuda(), g["y_valid"].cuda(),
                                    feature_edges=g["edge_index"].cuda()))
    out = te.train()
    assert out["loss_total"] > 0
    # the first step from the seed-42 init is the golden's first step (same init, same graph)
    assert abs(out["loss_total"] - golden["train"]["latest_measurement"]["steps"][0]["loss"].item()) < 1e-5
    te.save_checkpoint(str(tmp_path), "ck.pt")
    ck = torch.load(tmp_path / "ck.pt", weights_only=False)
    ref = golden["checkpoint"]
    assert list(ck["model_state_dict"]) == list(ref["model_state_dict"])
    assert list(ck["traversability_loss_state_dict"]) == list(ref["traversability_loss_state_dict"])
    assert len(ck["optimizer_state_dict"]["state"]) == len(ref["optimizer_state_dict"]["state"]) == 6
    # a checkpoint written by the reference classes loads, and the next step continues its Adam state
    te2 = TraversabilityEstimator(params=_params(), device="cuda", min_samples_for_training=0)
    te2.load_checkpoint(_save(tmp_path, "ref_ck.pt", ref))
    for k, v in ref["model_state_dict"].items():
        assert torch.equal(te2._model.state_dict()[k].cpu(), v)
    assert int(te2._trainer.step_counter.item()) == 3
    # the hand-off file: written by the learner, read by inference
    from wild_visual_navigation_b200 import ConfidenceGenerator

    te.write_model_handoff(str(tmp_path))
    ti = TraversabilityInference(None, _model(90, 32, 16), ConfidenceGenerator(0.5, "latest_measurement").cuda())
    assert ti.load_model(str(tmp_path))
    for k, v in te._model.state_dict().items():
        assert torch.equal(ti._model.state_dict()[k], v)
    # and the one the reference's learning node writes
    assert ti.load_model(_save(tmp_path, ".tmp_state_dict.pt", golden["tmp_state_dict"]))
    for k, v in golden["checkpoint"]["model_state_dict"].items():
        assert torch.equal(ti._model.state_dict()[k].cpu(), v)
    # segment-wise prediction on the frame's graph against float64
    seg = torch.randint(0, 100, (1, 8, 8)).cuda()
    trav, conf = ti.predict_segments(g["x"].cuda(), seg, edges=g["edge_index"].cuda())
    sd64 = {k: v.double().cpu() for k, v in ti._model.state_dict().items()}
    res = og.forward(sd64, g["x"].double(), g["edge_index"])
    assert (trav.cpu().double() - res[:, 0][seg.cpu()]).abs().max() < 1e-5
    cgm = ti._cg
    shifted = cgm.mean.double().cpu() + cgm.std.double().cpu() * 0.5
    lo, hi = (shifted - cgm.std.double().cpu()).clamp(min=0), shifted + cgm.std.double().cpu()
    lr = ((res[:, 1:] - g["x"].double()) ** 2).mean(1)
    conf64 = 1 - (lr.clamp(lo.item(), hi.item()) - lo) / (hi - lo)
    assert (conf.cpu().double() - conf64[seg.cpu()]).abs().max() < 1e-4
    with pytest.raises(ValueError):
        ti.predict_segments(g["x"].cuda(), seg)
    with pytest.raises(ValueError):
        ti.predict_from_tokens(torch.zeros(1, 4, 90).cuda(), 16)
    # a node without edges, and padded rows without edges, raise
    te.add_mission_node(MissionNode(g["x"].cuda(), g["y"].cuda(), g["y_valid"].cuda()))
    te._params["ablation_data_module"]["batch_size"] = 2
    with pytest.raises(ValueError, match="feature_edges"):
        te.train()
    with pytest.raises(ValueError, match="edges"):
        te.train_on_padded(g["x"][None].cuda(), torch.tensor([100], dtype=torch.int32).cuda(), g["y"].cuda(),
                           g["y_valid"].cuda())


def _save(tmp_path, name, obj):
    p = os.path.join(str(tmp_path), name)
    torch.save(obj, p)
    return p


def test_estimator_flags_overflowed_adjacency():
    from wild_visual_navigation_b200 import TraversabilityEstimator

    te = TraversabilityEstimator(params=_params(), device="cuda", min_samples_for_training=0)
    feat, n_rows, edges, ne, y, yv = _frames(2, 30, 90, seed=9)
    ne[1] = -1
    te.train_on_padded(*_cuda(feat, n_rows), *_cuda(y, yv), edges=edges.cuda(), n_edges=ne.cuda())
    assert te._trainer.metrics[6].item() == 1.0 and te.overflowed()
