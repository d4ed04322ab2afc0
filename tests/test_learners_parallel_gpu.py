"""The DoubleMLP and LinearRnvp learners on padded per-frame rows, data-parallel, and through ``HotPathStep``.

- ``step_padded`` on rows padded per frame (NaN in the padding) equals ``step`` on the same rows compacted, bit for bit:
  both run one launch sequence bounded by the device count of live rows.
- Two ranks sharing cuda:0 over gloo, each training ``TraversabilityEstimator(process_group=WORLD).train_on_padded`` on
  a ragged shard, reproduce one process's ``train_on_batch`` on the concatenated rows (2e-5), and stay bit-identical.
- With an NCCL group of world size 1 every trainer takes the library-communicator path and stays bit-identical to the
  same trainer without a group.
- ``HotPathStep(model="DoubleMLP")`` / ``HotPathStep(anomaly_detection=True)`` equal the same work composed by hand, and
  ``capture`` / ``replay`` equals an eager step.  Two HotPathSteps pool their segment features with float atomics, so
  their rows agree to rounding, not bit for bit: the composed twin trains on the stepped object's own rows, and the
  replayed object is held to a tolerance against an eager twin."""
import os
import socket
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

METHOD_ID = {"latest_measurement": 0, "running_mean": 1, "kalman_filter": 2, "moving_average": 3}
N_ROWS = [16, 3, 0, 9, 1]
S = 16


def _double(D, seed=42):
    from wild_visual_navigation_b200 import DoubleMLP

    torch.manual_seed(seed)
    return DoubleMLP(D, [64, 32, 1]).cuda()


def _flow(D, mask, seed=42):
    from wild_visual_navigation_b200 import LinearRnvp

    torch.manual_seed(seed)
    return LinearRnvp(D, [200], mask_type=mask, conditioning_size=0, use_permutation=True,
                      single_function=False).cuda()


def _padded(D, n_rows, seed, p_valid=0.4):
    """feat (G, S, D) with NaN in every padding row, n_rows (G,) int32, the live mask, y / y_valid (compacted)."""
    g = torch.Generator().manual_seed(seed)
    G = len(n_rows)
    feat = torch.randn(G, S, D, generator=g)
    live = torch.arange(S)[None, :] < torch.tensor(n_rows)[:, None]
    feat[~live] = float("nan")
    n = int(live.sum())
    yv = torch.rand(n, generator=g) < p_valid
    if n > 0:
        yv[0] = True
    y = torch.where(yv, torch.rand(n, generator=g).clamp(min=0.001), torch.zeros(n))
    return (feat.cuda(), torch.tensor(n_rows, dtype=torch.int32).cuda(), live.cuda(), y.cuda(), yv.cuda())


def _bind(tr, method):
    """Binds the generator's state to fresh caller tensors (so it can be compared) and returns them."""
    st = (torch.ones(1, 1, device="cuda"), torch.zeros(1, device="cuda", dtype=torch.float64),
          torch.zeros(1, device="cuda", dtype=torch.float64), torch.zeros(1, device="cuda", dtype=torch.float64))
    tr.set_confidence(METHOD_ID[method], *st)
    return st


def _state(tr, model, st, n_conf):
    return ([model.flat_params, tr.exp_avg, tr.exp_avg_sq, tr.step_counter, tr.metrics, tr.cg_mean, tr.cg_std,
             tr.conf[:n_conf]] + list(st))


def _all_equal(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------ padded == compacted
@pytest.mark.parametrize("D", [90, 384])
@pytest.mark.parametrize("method", list(METHOD_ID))
@pytest.mark.parametrize("balanced", [True, False])
def test_double_mlp_padded_step_equals_compacted_step(D, method, balanced):
    from wild_visual_navigation_b200 import ops

    runs = []
    for variant in ("padded", "compacted", "dropped"):
        m = _double(D)
        tr = ops.DoubleMlpTrainer(m, max_rows=len(N_ROWS) * S, anomaly_balanced=balanced)
        st = _bind(tr, method)
        for step in range(3):
            feat, n_rows, live, y, yv = _padded(D, N_ROWS, seed=10 + step)
            if variant == "padded":
                tr.step_padded(feat, n_rows, y, yv)
            elif variant == "compacted":
                tr.step(feat[live], y, yv)
            else:   # negative control: the last live row left out
                tr.step(feat[live][:-1], y[:-1], yv[:-1])
        n = sum(N_ROWS) - (variant == "dropped")
        runs.append(_state(tr, m, st, n))
    assert _all_equal(runs[0], runs[1])
    assert torch.isfinite(runs[0][0]).all()
    assert not torch.equal(runs[0][0], runs[2][0]), "dropping a live row must change the parameters"


@pytest.mark.parametrize("D", [90, 384])
@pytest.mark.parametrize("method", list(METHOD_ID))
@pytest.mark.parametrize("mask", ["odds", "half"])
def test_flow_padded_step_equals_compacted_step(D, method, mask):
    from wild_visual_navigation_b200 import ops

    runs = []
    for variant in ("padded", "compacted", "dropped"):
        m = _flow(D, mask)
        tr = ops.FlowTrainer(m, max_rows=len(N_ROWS) * S)
        st = _bind(tr, method)
        n_lab = 0
        for step in range(3):
            feat, n_rows, live, y, yv = _padded(D, N_ROWS, seed=20 + step)
            if variant == "padded":
                tr.step_padded(feat, n_rows, y, yv)
            elif variant == "compacted":
                tr.step(feat[live], yv)
            else:   # negative control: the first (always labelled) live row left out
                tr.step(feat[live][1:], yv[1:])
            n_lab = int(yv.sum()) - (variant == "dropped")
        runs.append(_state(tr, m, st, n_lab))
    assert _all_equal(runs[0], runs[1])
    assert torch.isfinite(runs[0][0]).all()
    assert not torch.equal(runs[0][0], runs[2][0]), "dropping a labelled row must change the parameters"


# ------------------------------------------------------------------------------------------------ two ranks over gloo
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _estimator(learner, method, D, pg=None):
    from wild_visual_navigation_b200 import TraversabilityEstimator
    from wild_visual_navigation_b200.traversability_estimator.traversability_estimator import default_params

    flow = learner == "flow"
    p = default_params(anomaly_detection=flow)
    if flow:
        p["model"]["linear_rnvp_cfg"]["input_size"] = D
        p["loss_anomaly"]["method"] = method
    else:
        p["model"]["name"] = "DoubleMLP"
        p["model"]["double_mlp_cfg"]["input_size"] = D
        p["loss"]["method"] = method
    return TraversabilityEstimator(params=p, device="cuda", anomaly_detection=flow, process_group=pg, max_rows=256)


def _generator(te):
    cg = te._traversability_loss._confidence_generator
    return torch.cat([t.detach().double().reshape(-1).cpu() for t in cg.state_dict().values()])


def _rank_worker(rank, world, port, learner, method, D, shards, ret):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(0)
    te = _estimator(learner, method, D, pg=dist.group.WORLD)
    out = []
    for feat, n_rows, y, yv in shards[rank]:
        conf = te.train_on_padded(feat.cuda(), n_rows.cuda(), y.cuda(), yv.cuda())
        n = int(yv.sum()) if learner == "flow" else int(n_rows.sum())
        out.append({"metrics": te._trainer.metrics.cpu().clone(), "conf": conf[:n].cpu().clone(),
                    "generator": _generator(te)})
    torch.cuda.synchronize()
    ret[rank] = {"params": te._model.flat_params.detach().cpu().clone(), "steps": out}
    dist.destroy_process_group()


def _close(got, want, tol=2e-5):
    scale = max(1.0, want.abs().max().item()) if want.numel() else 1.0
    nan = torch.isnan(want)
    return torch.equal(nan, torch.isnan(got)) and ((got - want)[~nan].abs().max().item() if (~nan).any() else 0.0) <= tol * scale


@pytest.mark.parametrize("learner", ["double", "flow"])
@pytest.mark.parametrize("method", ["latest_measurement", "moving_average", "running_mean"])
def test_two_ranks_equal_one_process(learner, method):
    D = 64
    # rank 0: 3 frames, one of them empty; rank 1: 2 frames.  For the flow, rank 1 has no labelled row at step 1.
    shapes = ([5, 0, 11], [9, 16])
    shards = [[], []]
    for step in range(3):
        for r in (0, 1):
            feat, n_rows, live, y, yv = _padded(D, shapes[r], seed=100 * step + r, p_valid=0.5)
            if learner == "flow" and r == 1 and step == 1:
                yv = torch.zeros_like(yv)
            shards[r].append((feat.cpu(), n_rows.cpu(), y.cpu(), yv.cpu()))
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_rank_worker, args=(2, _free_port(), learner, method, D, shards, ret), nprocs=2, join=True)

    single = _estimator(learner, method, D)
    for step in range(3):
        xs, ys, yvs = [], [], []
        for r in (0, 1):
            feat, n_rows, y, yv = shards[r][step]
            live = torch.arange(feat.shape[1])[None, :] < n_rows[:, None].long()
            xs.append(feat[live]); ys.append(y); yvs.append(yv)
        g = types.SimpleNamespace(x=torch.cat(xs).cuda(), y=torch.cat(ys).cuda(), y_valid=torch.cat(yvs).cuda())
        conf = single.train_on_batch(g)
        m = single._trainer.metrics.cpu()
        gen = _generator(single)
        off = 0
        for r in (0, 1):
            got = ret[r]["steps"][step]
            assert _close(got["metrics"], m), (step, r, got["metrics"], m)
            assert _close(got["generator"], gen), (step, r, got["generator"], gen)
            n = got["conf"].numel()
            assert _close(got["conf"], conf[off:off + n].cpu()), (step, r)
            off += n
    p = single._model.flat_params.detach().cpu()
    for r in (0, 1):
        d = ((ret[r]["params"] - p).norm() / p.norm()).item()
        assert d <= 2e-5, (r, d)
    assert torch.equal(ret[0]["params"], ret[1]["params"])   # replicas stay bit-identical


# ------------------------------------------------------------------------------------------------ NCCL, world size 1
def _nccl_worker(rank, port, ret):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", rank=0, world_size=1)
    from wild_visual_navigation_b200 import ops

    D = 90
    results = {}
    for name in ("mlp", "double", "flow"):
        states = []
        for pg in (None, dist.group.WORLD):
            if name == "mlp":
                torch.manual_seed(3)
                params = torch.randn(ops.lib().wvn_mlp_param_count(D, 256, 32), device="cuda") * 0.05
                tr = ops.MlpTrainer(params, D, 256, 32, max_rows=len(N_ROWS) * S, process_group=pg)
                model = types.SimpleNamespace(flat_params=params)
            elif name == "double":
                model = _double(D)
                tr = ops.DoubleMlpTrainer(model, max_rows=len(N_ROWS) * S, process_group=pg)
            else:
                model = _flow(D, "odds")
                tr = ops.FlowTrainer(model, max_rows=len(N_ROWS) * S, process_group=pg)
            assert tr._lib_comm == (pg is not None)
            st = _bind(tr, "moving_average")
            for step in range(3):
                feat, n_rows, live, y, yv = _padded(D, N_ROWS, seed=40 + step)
                tr.step_padded(feat, n_rows, y, yv)
            torch.cuda.synchronize()
            states.append([t.cpu() for t in _state(tr, model, st, 8)])
        results[name] = _all_equal(*states)
    ret[0] = results
    dist.destroy_process_group()


def test_nccl_world_one_library_communicator_is_bit_identical():
    if not dist.is_nccl_available():
        pytest.skip("torch.distributed was built without NCCL")
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_nccl_worker, args=(_free_port(), ret), nprocs=1, join=True)
    assert ret[0] == {"mlp": True, "double": True, "flow": True}, ret[0]


# ------------------------------------------------------------------------------------------------ HotPathStep
@pytest.fixture(scope="module")
def weights():
    import bench

    cfg, sd, hd = bench.make_weights()
    return sd, hd


def _hot_path(weights, learner):
    from wild_visual_navigation_b200 import HotPathStep

    kw = {"model": "DoubleMLP"} if learner == "double" else {"anomaly_detection": True}
    return HotPathStep("cuda", weights[0], weights[1], batch=3, input_size=224, chunk=32, flip_tta=False,
                       run_clustering=True, n_image_clusters=20, **kw)


def _frames(seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(3, 3, 224, 224, generator=g).cuda()


def _labels(hp, seed):
    g = torch.Generator().manual_seed(seed)
    n = 3 * hp.smax
    yv = torch.rand(n, generator=g) < 0.3
    return torch.where(yv, torch.rand(n, generator=g).clamp(min=0.001), torch.zeros(n)).cuda(), yv.cuda()


def _learner_state(hp):
    cg = hp.cg
    return [hp.te._model.flat_params.detach().clone(), hp.te._trainer.exp_avg.clone(),
            hp.te._trainer.step_counter.clone()] + [t.detach().clone() for t in cg.state_dict().values()]


@pytest.mark.parametrize("learner", ["double", "flow"])
def test_hot_path_step_equals_composed_work(weights, learner):
    a, b = _hot_path(weights, learner), _hot_path(weights, learner)
    for step in range(2):
        img = _frames(step)
        y, yv = _labels(a, 50 + step)
        ra = a.step(img, y, yv)
        # the same work by hand (maps from b's own tokens; the train step on a's pooled rows, see the module docstring)
        rb = b.fe.extract_batch(img)
        trav, conf = b.ti.predict_from_tokens(rb["tokens"], 224)
        live = torch.arange(a.smax, device="cuda")[None, :] < ra["n_segments"][:, None].long()
        x = ra["feat"][live]
        n = x.shape[0]
        crow = b.te.train_on_batch(types.SimpleNamespace(x=x, y=y[:n], y_valid=yv[:n]))
        b.ti.refresh_weights()
        assert torch.equal(ra["trav"], trav)
        assert (ra["conf"] is None and conf is None) if learner == "flow" else torch.equal(ra["conf"], conf)
        k = int(yv[:n].sum()) if learner == "flow" else n
        assert torch.equal(ra["confidence_rows"][:k], crow[:k])
        assert _all_equal(_learner_state(a), _learner_state(b))
        assert torch.isfinite(a.te._model.flat_params).all()


@pytest.mark.parametrize("learner", ["double", "flow"])
def test_hot_path_capture_replay_equals_eager(weights, learner):
    a, b = _hot_path(weights, learner), _hot_path(weights, learner)
    img0, img1 = _frames(7), _frames(8)
    y, yv = _labels(a, 9)
    a.capture(img0, y, yv, warmup=2)   # two eager steps on img0, then the capture
    for _ in range(2):
        b.step(img0, y, yv)
    ra = a.replay(img1)
    rb = b.step(img1, y, yv)
    torch.cuda.synchronize()
    # the maps run on bf16 copies of the weights: a last-bit difference in an fp32 weight can flip its bf16 rounding
    assert (ra["trav"] - rb["trav"]).abs().max().item() <= 2e-3
    if learner == "double":
        assert (ra["conf"] - rb["conf"]).abs().max().item() <= 2e-3
    sa, sb = _learner_state(a), _learner_state(b)
    assert torch.equal(sa[2], sb[2]) and int(sa[2]) == 3   # Adam's step counter: three steps, one of them replayed
    for u, v in zip(sa[:2] + sa[3:], sb[:2] + sb[3:]):
        assert ((u.double() - v.double()).norm() / v.double().norm().clamp_min(1e-30)).item() <= 1e-4
