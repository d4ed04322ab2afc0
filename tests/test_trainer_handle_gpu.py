"""GPU tests of the trainer handle every learner shares (wvn_trainer_t, ops._TrainerHandle): a SimpleGCN trainer that
outgrows its rows or its edges keeps its generator and its optimiser exactly, and every learner's entry point refuses
another learner's handle on the host, before it enqueues anything."""
from ctypes import byref, c_void_p

import pytest
import torch

from test_gcn_gpu import METHOD_ID, _cuda, _frames, _model

pytestmark = pytest.mark.gpu

# (frames, rows per frame) per step: the padded rows and, at ~3.8 edges per row, the padded edges grow twice mid-sequence
STEPS = [(2, 40), (3, 40), (8, 60), (2, 50), (20, 60), (3, 30)]


class _Gcn:
    """ops.GcnTrainer with its generator state private, or bound to tensors the test can read."""

    def __init__(self, method, bound, max_rows, max_edges):
        from wild_visual_navigation_b200 import ops

        self.model = _model(64, 32, 16)
        self.tr = ops.GcnTrainer(self.model, max_rows=max_rows, max_edges=max_edges)
        self.var = torch.ones(1, 1, device="cuda")
        self.running = torch.zeros(3, dtype=torch.float64, device="cuda")
        if bound:
            self.tr.set_confidence(METHOD_ID[method], self.var, self.running[0:1], self.running[1:2], self.running[2:3])
        else:
            self.tr.set_confidence(METHOD_ID[method])


@pytest.mark.parametrize("grow", ["rows", "edges"])
@pytest.mark.parametrize("bound", [True, False], ids=["bound", "private"])
@pytest.mark.parametrize("method", ["moving_average", "running_mean", "kalman_filter"])
def test_gcn_regrowth_keeps_the_generator(method, bound, grow):
    """A step that outgrows max_rows (or, separately, max_edges) replaces the handle: the generator (moving_average's
    window and, when private, var and the running sums) and Adam must continue exactly as on a trainer created large
    enough."""
    small_rows, small_edges = (128, 1 << 16) if grow == "rows" else (8192, 400)
    small = _Gcn(method, bound, small_rows, small_edges)
    large = _Gcn(method, bound, 8192, 1 << 16)
    for s, (G, S) in enumerate(STEPS):
        feat, n_rows, edges, ne, y, yv = _cuda(*_frames(G, S, 64, seed=500 + s))
        for T in (small, large):
            T.tr.step_padded(feat, n_rows, edges, ne, y, yv)
        for k in ("metrics", "cg_mean", "cg_std", "exp_avg"):
            assert torch.equal(getattr(small.tr, k), getattr(large.tr, k)), f"step {s}: {k}"
        assert torch.equal(small.model.flat_params, large.model.flat_params), f"step {s}: params"
        if bound:
            assert torch.equal(small.var, large.var) and torch.equal(small.running, large.running), f"step {s}"
    if grow == "rows":
        assert small_rows < small.tr.max_rows < large.tr.max_rows and small.tr.max_edges == small_edges
    else:
        assert small_edges < small.tr.max_edges < large.tr.max_edges and small.tr.max_rows == small_rows


# ------------------------------------------------------------------------------------------------ kind check
D, H1, H2, HIDDEN = 32, 16, 8, 16
NAMES = {"mlp": "SimpleMLP", "double": "DoubleMLP", "gcn": "SimpleGCN", "flow": "LinearRnvp"}


def _learner(kind):
    """A seeded model of `kind` and a fresh trainer on it."""
    from wild_visual_navigation_b200 import DoubleMLP, LinearRnvp, SimpleGCN, SimpleMLP, ops

    torch.manual_seed(7)
    if kind == "mlp":
        m = SimpleMLP(D, [H1, H2, 1], True).cuda()
        return m, ops.MlpTrainer(m.flat_params, dim=D, h1=H1, h2=H2, max_rows=256)
    if kind == "double":
        m = DoubleMLP(D, [H1, H2, 1]).cuda()
        return m, ops.DoubleMlpTrainer(m, max_rows=256)
    if kind == "gcn":
        m = SimpleGCN(D, True, [H1, H2, 1]).cuda()
        return m, ops.GcnTrainer(m, max_rows=256, max_edges=1024)
    m = LinearRnvp(D, [HIDDEN], use_permutation=True).cuda()
    return m, ops.FlowTrainer(m, max_rows=256)


def _valid_step(kind, tr):
    """One step on seeded rows: the confidence vector's live prefix.  Four rows: the SimpleMLP step adds its per-tile
    and per-warp sums with atomics, and only four rows (one warp of one tile) keep each of those sums to a single
    contributor, so that two runs are bit-identical."""
    g = torch.Generator(device="cuda").manual_seed(3)
    R = 4
    x = torch.randn(R, D, device="cuda", generator=g) * 0.5
    y = torch.rand(R, device="cuda", generator=g)
    yv = torch.rand(R, device="cuda", generator=g) < 0.5
    yv[:2] = True   # the generator's std needs two labelled rows
    if kind == "gcn":
        ei = torch.stack([torch.arange(R - 1), torch.arange(1, R)]).cuda()
        return tr.step(x, ei, y, yv)
    if kind == "flow":
        return tr.step(x, yv)[:int(yv.sum())]   # the labelled rows' confidences
    return tr.step(x, y, yv)


def _wrong_calls(flow_model):
    """Every learner-specific entry point that takes a trainer handle, as kind -> [(name, call(handle) -> status)],
    with arguments that would be valid for a handle of that kind."""
    from wild_visual_navigation_b200 import ops
    from wild_visual_navigation_b200._C import lib, stream

    buf = torch.zeros(4096, device="cuda")
    p = c_void_p(buf.data_ptr())
    fb = ops.flow_buffers(flow_model)
    s = stream()
    return {
        "mlp": [("wvn_mlp_train_step", lambda h: lib().wvn_mlp_train_step(
            h, p, p, p, p, p, 1, 4, None, p, p, p, p, p, p, 7, s))],
        "double": [("wvn_double_mlp_train_step_padded", lambda h: lib().wvn_double_mlp_train_step_padded(
            h, p, p, p, p, p, 1, 4, None, p, p, p, p, p, p, 7, s))],
        "gcn": [("wvn_gcn_train_step_padded", lambda h: lib().wvn_gcn_train_step_padded(
                    h, p, p, p, p, p, 1, 4, None, p, 1, p, p, p, p, p, p, p, 7, s)),
                ("wvn_gcn_infer_rows", lambda h: lib().wvn_gcn_infer_rows(
                    h, p, p, 1, 4, None, p, 1, p, p, p, 0.5, p, p, p, s))],
        "flow": [("wvn_flow_train_step", lambda h: lib().wvn_flow_train_step(
                     h, p, p, p, p, byref(fb), p, 4, None, p, p, p, p, 7, s)),
                 ("wvn_flow_train_step_padded", lambda h: lib().wvn_flow_train_step_padded(
                     h, p, p, p, p, byref(fb), p, 1, 4, None, None, p, p, p, p, 7, s))],
    }, buf


def test_entry_points_refuse_another_learners_handle():
    """Each learner's step entry point, wvn_gcn_infer_rows and wvn_trainer_copy_confidence return WVN_STATUS_INVALID,
    naming the learner they expected, for every other learner's handle, and launch nothing.  A valid step on a trainer
    whose handle went through those calls still equals a fresh trainer's bit for bit."""
    from wild_visual_navigation_b200._C import lib, stream

    kinds = list(NAMES)
    used = {k: _learner(k) for k in kinds}
    calls, keep = _wrong_calls(used["flow"][0])
    torch.cuda.synchronize()
    launches = lib().wvn_launch_count()
    for want in kinds:
        for name, call in calls[want]:
            for other in kinds:
                if other == want:
                    continue
                rc = call(used[other][1]._h)
                msg = lib().wvn_last_error().decode()
                assert rc == -1, (name, other, rc)
                assert f"expected a {NAMES[want]} trainer" in msg and NAMES[other] in msg, (name, other, msg)
        for other in kinds:
            if other != want:
                rc = lib().wvn_trainer_copy_confidence(used[want][1]._h, used[other][1]._h, stream())
                msg = lib().wvn_last_error().decode()
                assert rc == -1 and f"expected a {NAMES[want]} trainer" in msg, (want, other, rc, msg)
    torch.cuda.synchronize()
    assert lib().wvn_launch_count() == launches, "a refused call enqueued work"
    for k in kinds:
        (ma, ta), (mb, tb) = used[k], _learner(k)
        ca, cb = _valid_step(k, ta), _valid_step(k, tb)
        assert torch.equal(ma.flat_params, mb.flat_params), k
        for name in ("metrics", "exp_avg", "exp_avg_sq", "cg_mean", "cg_std"):
            assert torch.equal(getattr(ta, name), getattr(tb, name)), (k, name)
        assert torch.equal(ca, cb), k
