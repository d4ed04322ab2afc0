"""The SimpleGCN learner across the deployment paths: the phased step, two gloo ranks against one process, an NCCL group
of world size 1 against no group, batched graphs split per node, the device mission graph's edge storage and
``train()``, and ``HotPathStep(model="SimpleGCN")`` eager and through ``capture`` / ``replay``."""
import os
import socket
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import simple_gcn as og

pytestmark = pytest.mark.gpu

D = 48


def _params(D=D, method="latest_measurement"):
    from wild_visual_navigation_b200.traversability_estimator.traversability_estimator import default_params

    p = default_params()
    p["model"]["name"] = "SimpleGCN"
    p["model"]["simple_gcn_cfg"] = {"input_size": D, "reconstruction": True, "hidden_sizes": [32, 16, 1]}
    p["loss"]["method"] = method
    return p


def _estimator(method="latest_measurement", pg=None, **kw):
    from wild_visual_navigation_b200 import TraversabilityEstimator

    return TraversabilityEstimator(params=_params(method=method), device="cuda", process_group=pg, max_rows=512,
                                   min_samples_for_training=0, **kw)


def _frames(n_rows, seed, S=24, E=90):
    g = torch.Generator().manual_seed(seed)
    G = len(n_rows)
    feat = torch.full((G, S, D), float("nan"))
    edges = torch.full((G, E, 2), -1, dtype=torch.long)
    ne = torch.zeros(G, dtype=torch.int32)
    for f, k in enumerate(n_rows):
        feat[f, :k] = torch.randn(k, D, generator=g) * 0.8 + 0.1
        if k > 0:
            m = min(E, int(3.8 * k))
            edges[f, :m] = torch.randint(0, k, (m, 2), generator=g)
            ne[f] = m
    N = sum(n_rows)
    yv = torch.rand(N, generator=g) < 0.4
    yv[:2] = True
    y = torch.where(yv, torch.rand(N, generator=g).clamp(min=0.001), torch.zeros(N))
    return feat, torch.tensor(n_rows, dtype=torch.int32), edges, ne, y, yv


def _cuda(*ts):
    return [t.cuda() for t in ts]


def _state(te):
    cg = te._traversability_loss._confidence_generator
    return [te._model.flat_params.detach().clone(), te._trainer.exp_avg.clone(), te._trainer.exp_avg_sq.clone(),
            te._trainer.step_counter.clone(), te._trainer.metrics.clone()] + [t.detach().clone() for t in
                                                                                cg.state_dict().values()]


def _all_equal(a, b):
    return all(torch.equal(u, v) for u, v in zip(a, b))


# ------------------------------------------------------------------------------------------------ phases
@pytest.mark.parametrize("method", ["latest_measurement", "moving_average"])
def test_phases_compose_to_the_whole_step_and_publish_float64_sums(method):
    """Phases 1 / 2 / 4 run one at a time equal the whole step bit for bit; after phase 1 the statistics block holds
    the float64 sums of the float64 oracle's forward (to fp32 rounding), after phase 2 the gradient is the oracle's."""
    from wild_visual_navigation_b200 import ops

    mid = {"latest_measurement": 0, "moving_average": 3}[method]
    feat, n_rows, edges, ne, y, yv = _cuda(*_frames([9, 0, 17, 24], seed=3))
    runs = []
    for split in (False, True):
        torch.manual_seed(42)
        from wild_visual_navigation_b200 import SimpleGCN

        m = SimpleGCN(D, True, [32, 16, 1]).cuda()
        tr = ops.GcnTrainer(m)
        tr.set_confidence(mid)
        if not split:
            tr.step_padded(feat, n_rows, edges, ne, y, yv)
        else:
            e64, E = ops._check_edges(edges, ne, 4)
            yv8 = yv.to(torch.uint8)
            for mask in (1, 2, 4):
                ops.check(ops.lib().wvn_gcn_train_step_padded(
                    tr._h, ops.ptr(m.flat_params), ops.ptr(tr.exp_avg), ops.ptr(tr.exp_avg_sq), ops.ptr(tr.step_counter),
                    ops.ptr(feat), 4, 24, ops.ptr(n_rows), ops.ptr(e64), E, ops.ptr(ne), ops.ptr(y), ops.ptr(yv8),
                    ops.ptr(tr.cg_mean), ops.ptr(tr.cg_std), ops.ptr(tr.conf), ops.ptr(tr.metrics), mask, ops.stream()))
                if mask == 1:
                    stats = tr.stats.clone()
                if mask == 2:
                    grads = tr.grads.clone()
        runs.append([m.flat_params.clone(), tr.grads.clone(), tr.metrics.clone(), tr.exp_avg.clone()])
    assert _all_equal(runs[0], runs[1])
    torch.manual_seed(42)
    sd64 = {k: v.double() for k, v in SimpleGCN(D, True, [32, 16, 1]).state_dict().items()}
    x64, ei = og.padded_to_graph(feat.cpu().double(), n_rows.cpu(), edges.cpu(), ne.cpu())
    res = og.forward(sd64, x64, ei)
    lr = ((res[:, 1:] - x64) ** 2).mean(1)
    raw = (res[:, 0] - y.cpu().double()) ** 2
    v = yv.cpu()
    want = torch.stack([lr[v].sum(), (lr[v] ** 2).sum(), raw.sum(), v.sum().double(), torch.tensor(float(len(v))),
                        torch.tensor(0.0), lr.min(), lr.max()])
    got = stats[:8].cpu()
    assert torch.equal(got[3:6], want[3:6])   # counts, and no overflow
    assert ((got - want).abs() <= 1e-5 * want.abs() + 1e-7).all(), (got, want)
    from oracle.wvn_path import ConfidenceState

    _, g64, _, _ = og.train_step(sd64, {}, x64, ei, y.cpu().double(), v, ConfidenceState(0.5, method))
    g = torch.cat([g64[k].reshape(-1) for k in og.keys()])
    assert ((grads.cpu().double() - g).abs().max() / g.abs().max()).item() < 5e-4


# ------------------------------------------------------------------------------------------------ batched graphs
def test_batch_split_per_node_is_bit_identical_to_one_frame():
    from wild_visual_navigation_b200 import Batch, Data, SimpleGCN, ops

    feat, n_rows, edges, ne, y, yv = _frames([7, 0, 12, 5], seed=8)
    nodes = [Data(x=feat[f, : n_rows[f]].cuda(), edge_index=edges[f, : ne[f]].t().contiguous().cuda())
             for f in range(4)]
    b = Batch.from_data_list(nodes)
    outs = []
    for ptr in (None, b.ptr):
        torch.manual_seed(42)
        m = SimpleGCN(D, True, [32, 16, 1]).cuda()
        tr = ops.GcnTrainer(m)
        conf = tr.step(b.x, b.edge_index, y.cuda(), yv.cuda(), ptr=ptr)
        outs.append([m.flat_params.clone(), tr.grads.clone(), tr.metrics.clone(), conf.clone()])
    assert _all_equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------------ two ranks over gloo
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_worker(rank, world, port, method, shards, ret):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(0)
    te = _estimator(method, pg=dist.group.WORLD)
    out = []
    for fr in shards[rank]:
        feat, n_rows, edges, ne, y, yv = _cuda(*fr)
        conf = te.train_on_padded(feat, n_rows, y, yv, edges=edges, n_edges=ne)
        out.append({"metrics": te._trainer.metrics.cpu().clone(), "conf": conf[: int(n_rows.sum())].cpu().clone()})
    torch.cuda.synchronize()
    ret[rank] = {"params": te._model.flat_params.detach().cpu().clone(), "steps": out}
    dist.destroy_process_group()


@pytest.mark.parametrize("method", ["latest_measurement", "moving_average"])
def test_two_ranks_equal_one_process(method):
    shapes = ([5, 0, 11], [9, 16])
    shards = [[], []]
    for step in range(3):
        for r in (0, 1):
            fr = list(_frames(shapes[r], seed=100 * step + r))
            if step == 1 and r == 1:
                fr[3][1] = -1    # an overflowed frame on rank 1: every rank must see the flag
            shards[r].append(fr)
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_rank_worker, args=(2, _free_port(), method, shards, ret), nprocs=2, join=True)
    single = _estimator(method)
    for step in range(3):
        parts = [shards[r][step] for r in (0, 1)]
        feat = torch.cat([p[0] for p in parts])
        cat = [feat, torch.cat([p[1] for p in parts]), torch.cat([p[2] for p in parts]), torch.cat([p[3] for p in parts]),
               torch.cat([p[4] for p in parts]), torch.cat([p[5] for p in parts])]
        feat, n_rows, edges, ne, y, yv = _cuda(*cat)
        conf = single.train_on_padded(feat, n_rows, y, yv, edges=edges, n_edges=ne)
        m = single._trainer.metrics.cpu()
        assert m[6].item() == (1.0 if step == 1 else 0.0)
        off = 0
        for r in (0, 1):
            got = ret[r]["steps"][step]
            assert got["metrics"][6].item() == m[6].item()
            assert ((got["metrics"] - m).abs() <= 2e-5 * m.abs().clamp(min=1)).all(), (step, r, got["metrics"], m)
            n = got["conf"].numel()
            assert ((got["conf"] - conf[off : off + n].cpu()).abs() <= 2e-5).all()
            off += n
    p = single._model.flat_params.detach().cpu()
    for r in (0, 1):
        assert ((ret[r]["params"] - p).norm() / p.norm()).item() <= 2e-5
    assert torch.equal(ret[0]["params"], ret[1]["params"])


def _nccl_worker(rank, port, ret):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", rank=0, world_size=1)
    states = []
    for pg in (None, dist.group.WORLD):
        te = _estimator("moving_average", pg=pg)
        assert te._trainer._lib_comm == (pg is not None)
        for step in range(3):
            feat, n_rows, edges, ne, y, yv = _cuda(*_frames([5, 0, 11, 24], seed=40 + step))
            te.train_on_padded(feat, n_rows, y, yv, edges=edges, n_edges=ne)
        torch.cuda.synchronize()
        states.append([t.cpu() for t in _state(te)] + [te._trainer.stats.cpu().clone()])
    ret[0] = _all_equal(*states)
    dist.destroy_process_group()


def test_nccl_world_one_library_communicator_is_bit_identical():
    if not dist.is_nccl_available():
        pytest.skip("torch.distributed was built without NCCL")
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_nccl_worker, args=(_free_port(), ret), nprocs=1, join=True)
    assert ret[0]


# ------------------------------------------------------------------------------------------------ mission graph
def test_mission_graph_stores_gathers_and_trains_from_edges():
    import random

    feat, n_rows, edges, ne, y, yv = _frames([9, 14, 20, 6, 24], seed=21)
    B, H, W = 5, 16, 16
    seg = torch.randint(0, 6, (B, H, W))
    ne_over = ne.clone()
    r = {"seg": seg.cuda(), "feat": torch.nan_to_num(feat).cuda(), "n_segments": n_rows.cuda(), "edges": edges.cuda(),
         "n_edges": ne.cuda()}
    K = torch.eye(4)
    poses = torch.eye(4).repeat(B, 1, 1)
    poses[:, 0, 3] = torch.arange(B, dtype=torch.float32)
    te, ref = _estimator(mission_graph_smax=24), _estimator(mission_graph_smax=24)
    assert te.add_mission_frames(r, poses, K, [float(i) for i in range(B)]) == B
    g = te._mission_graph
    assert g.edges.shape == (g.capacity, 16 * 24, 2) and g.edges.dtype == torch.int32
    # labels as a propagation would leave them
    g.y[:B].copy_(torch.rand(B, 24))
    g.y_valid[:B].copy_((torch.rand(B, 24) < 0.5).to(torch.uint8))
    g.y_valid[:B, :2] = 1
    g.slot_valid[:B] = 1
    g._meta_host = None
    ge, gn = g.gather_edges(g.get_nodes())
    assert torch.equal(gn.cpu(), ne)
    for f in range(B):
        assert torch.equal(ge[f, : ne[f]].cpu(), edges[f, : ne[f]])
    random.seed(5)
    out = te.train()
    assert out["loss_total"] > 0
    nodes = te.last_sampled_nodes
    fe, nr, yy, yvv = g.gather(nodes)
    e2, n2 = g.gather_edges(nodes)
    ref.train_on_padded(fe, nr, yy, yvv, edges=e2, n_edges=n2)
    assert torch.equal(te._model.flat_params, ref._model.flat_params)
    assert torch.equal(te._trainer.metrics, ref._trainer.metrics)
    # an overflowed frame is stored with a negative count and train() raises
    ne_over[2] = 10_000
    r2 = dict(r, n_edges=ne_over.cuda())
    poses2 = poses.clone()
    poses2[:, 1, 3] = 50.0
    te.add_mission_frames(r2, poses2, K, [float(10 + i) for i in range(B)])
    assert int(g.n_edges[g.get_nodes()[-3].slot]) == -1
    for nd in g.get_nodes():
        g.slot_valid[nd.slot] = 1
        g.y_valid[nd.slot, :2] = 1
    g._meta_host = None
    te._params["ablation_data_module"]["batch_size"] = 64
    with pytest.raises(ValueError, match="overflowed"):
        te.train()


# ------------------------------------------------------------------------------------------------ HotPathStep
@pytest.fixture(scope="module")
def weights():
    import bench

    cfg, sd, hd = bench.make_weights()
    return sd, hd


def _hot_path(weights):
    from wild_visual_navigation_b200 import HotPathStep

    return HotPathStep("cuda", weights[0], weights[1], batch=3, input_size=224, chunk=32, flip_tta=False,
                       run_clustering=True, n_image_clusters=20, model="SimpleGCN")


def _img(seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(3, 3, 224, 224, generator=g).cuda()


def _labels(hp, seed):
    g = torch.Generator().manual_seed(seed)
    n = 3 * hp.smax
    yv = torch.rand(n, generator=g) < 0.3
    yv[:2] = True
    return torch.where(yv, torch.rand(n, generator=g).clamp(min=0.001), torch.zeros(n)).cuda(), yv.cuda()


def test_hot_path_step_equals_composed_work(weights):
    a, b = _hot_path(weights), _hot_path(weights)
    for step in range(2):
        img = _img(step)
        y, yv = _labels(a, 50 + step)
        ra = a.step(img, y, yv)
        # the same work by hand on a's pooled rows and graph (segment pooling uses float atomics: two extractions of
        # the same frames may differ in the last bits)
        tb, cb = b.ti.predict_frames(ra["feat"], ra["n_segments"], ra["edges"], ra["n_edges"], ra["seg"])
        crow = b.te.train_on_padded(ra["feat"], ra["n_segments"], y, yv, edges=ra["edges"], n_edges=ra["n_edges"])
        assert torch.equal(ra["trav"], tb) and torch.equal(ra["conf"], cb)
        n = int(ra["n_segments"].sum())
        assert torch.equal(ra["confidence_rows"][:n], crow[:n])
        assert _all_equal(_state(a.te), _state(b.te))
        assert (ra["n_edges"] >= 0).all() and torch.isfinite(ra["trav"]).all()


def test_hot_path_capture_replay_equals_eager(weights):
    a, b = _hot_path(weights), _hot_path(weights)
    img0, img1 = _img(7), _img(8)
    y, yv = _labels(a, 9)
    a.capture(img0, y, yv, warmup=2)
    for _ in range(2):
        b.step(img0, y, yv)
    ra = a.replay(img1)
    rb = b.step(img1, y, yv)
    torch.cuda.synchronize()
    # segment pooling uses float atomics, so the two paths' rows may differ in the last bits
    assert (ra["trav"] - rb["trav"]).abs().max().item() <= 2e-3
    assert (ra["conf"] - rb["conf"]).abs().max().item() <= 2e-3
    sa, sb = _state(a.te), _state(b.te)
    assert torch.equal(sa[3], sb[3]) and int(sa[3]) == 3
    for u, v in zip(sa[:3], sb[:3]):
        assert ((u.double() - v.double()).norm() / v.double().norm().clamp_min(1e-30)).item() <= 1e-4
