"""GPU tests of the LinearRnvp anomaly-detection learner (csrc/flow_train.cu) against the float64 oracle
(oracle/linear_rnvp.py) and against goldens made by the reference's own classes (tests/golden/make_golden_rnvp.py).

Bound for the fp32 row forward.  The kernels and the reference evaluate the same fp32 expressions; they differ only in
summation order (a length-K dot product has a first-order error of at most K u sum|terms|, u = 2^-24, in either order)
and in the exp / tanh implementations (a few ulp).  The fp32 torch evaluation of the oracle on the same inputs measures
the size of that error for the data at hand, so an element passes when |gpu - ref64| <= 8 |ref32 - ref64| +
64 u (1 + |ref64|): eight times the reference's own fp32 error plus a floor of 64 ulp of the value.  The negative
controls (s and t swapped on trained weights, a dropped permutation, one row shifted) must exceed it.
"""
import os

import pytest
import torch

from oracle import linear_rnvp as orn
from oracle.wvn_path import ConfidenceState, confidence_inference

pytestmark = pytest.mark.gpu
U = 2.0**-24
METHODS = ("latest_measurement", "running_mean", "moving_average", "kalman_filter")


def _model(dim, hidden, mask="odds", seed=42, spread=0.05, device="cuda"):
    """A LinearRnvp (on the GPU by default) whose t nets differ from the s nets (as after training)."""
    from wild_visual_navigation_b200 import LinearRnvp

    torch.manual_seed(seed)
    m = LinearRnvp(dim, [hidden], mask_type=mask, conditioning_size=0, use_permutation=True, single_function=False)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if ".t." in n:
                p.add_(torch.randn(p.shape, generator=g) * spread)
    return m.to(device)


def _sd64(m):
    return {k: (v.detach().double().cpu() if v.is_floating_point() else v.cpu()) for k, v in m.state_dict().items()}


def _bound(ref64, ref32):
    return 8 * (ref32.double() - ref64).abs() + 64 * U * (1 + ref64.abs())


def _ok(got, ref64, ref32, against=None):
    """got within the bound of (ref64, ref32); ``against``: compare with this tensor instead (negative controls) under
    the same bound."""
    want = ref64 if against is None else against
    return bool(((got.double().cpu() - want).abs() <= _bound(ref64, ref32)).all())


def _cfg(golden_dir):
    return torch.load(os.path.join(golden_dir, "linear_rnvp.pt"), weights_only=False)


@pytest.mark.parametrize("dim", [90, 384, 768])
@pytest.mark.parametrize("mask", ["odds", "half"])
def test_row_forward_matches_float64(dim, mask):
    from wild_visual_navigation_b200 import Data

    m = _model(dim, 200 if dim != 768 else 256, mask)
    sd64 = _sd64(m)
    sd32 = {k: (v.float() if v.is_floating_point() else v) for k, v in sd64.items()}
    g = torch.Generator().manual_seed(dim)
    for rows in (1, 37, 130):
        x = torch.randn(rows, dim, generator=g) * 0.5
        out = m(Data(x=x.cuda()))
        r64, r32 = orn.forward(sd64, x.double()), orn.forward(sd32, x)
        for k in ("z", "log_det", "logprob"):
            assert _ok(out[k], r64[k], r32[k]), (k, rows)
    # negative controls on the last rows: each corruption exceeds the bound somewhere
    swapped = dict(sd64)
    for c in (0, 2):
        for i in (0, 2, 4):
            for w in ("weight", "bias"):
                swapped[f"flows.{c}.s.{i}.{w}"], swapped[f"flows.{c}.t.{i}.{w}"] = (sd64[f"flows.{c}.t.{i}.{w}"],
                                                                                    sd64[f"flows.{c}.s.{i}.{w}"])
    noperm = dict(sd64)
    noperm["flows.3.p"] = torch.arange(dim)
    for bad in (swapped, noperm):
        assert not _ok(out["z"], r64["z"], r32["z"], against=orn.forward(bad, x.double())["z"])
    assert not _ok(out["z"], r64["z"], r32["z"], against=torch.roll(r64["z"], 1, 0))


def _load_small(golden, mask):
    from wild_visual_navigation_b200 import LinearRnvp

    m = LinearRnvp(32, [16], mask_type=mask, use_permutation=True)
    m.load_state_dict(golden["train"][("latest_measurement", mask)]["init"])
    return m.cuda()


@pytest.mark.parametrize("method,mask", [(m, "odds") for m in METHODS] + [("latest_measurement", "half")])
def test_three_train_steps_match_reference_golden(golden_dir, method, mask):
    """Phase by phase: after phase 1 the loss / confidence / generator, after phase 2 every gradient element, after
    phase 4 (three steps) the parameters, each against the reference's own fp32 run."""
    from wild_visual_navigation_b200 import ops
    from wild_visual_navigation_b200.utils import AnomalyLoss

    golden = _cfg(golden_dir)
    m = _load_small(golden, mask)
    loss = AnomalyLoss(0.5, method).cuda()
    cg = loss._confidence_generator
    tr = ops.FlowTrainer(m, max_rows=64, std_factor=0.5, lr=1e-3)
    tr.cg_mean, tr.cg_std = cg.mean.data, cg.std.data
    kf = getattr(cg, "_kalman_filter", None)
    tr.set_confidence(cg.method_id, cg.var.data, getattr(cg, "running_n", None), getattr(cg, "running_sum", None),
                      getattr(cg, "running_sum_of_squares", None),
                      kf_proc_cov=float(kf.proc_cov.item()) if kf is not None else 0.2,
                      kf_meas_cov=float(kf.meas_cov.item()) if kf is not None else 1.0)
    names = [n for n, _ in m.named_parameters()]
    for st in golden["train"][(method, mask)]["steps"]:
        x = st["x"].cuda()
        conf = tr.step(x, phase_mask=1)
        R = x.shape[0]
        assert abs(tr.metrics[0].item() - st["loss"].item()) <= 1e-5 * (1 + abs(st["loss"].item()))
        assert tr.metrics[3].item() == R
        std_tol = 1e-5 + 4 * U * float(st["cg_mean"]) ** 2 / float(st["cg_std"])   # see test_linear_rnvp_oracle.py
        assert abs(cg.mean.item() - st["cg_mean"].item()) <= 1e-5 * (1 + abs(st["cg_mean"].item()))
        assert abs(cg.std.item() - st["cg_std"].item()) <= std_tol + 1e-5 * abs(st["cg_std"].item())
        assert torch.allclose(conf[:R].cpu(), st["confidence"], atol=2e-4), (conf[:R].cpu() - st["confidence"]).abs().max()
        tr.step(x, phase_mask=2)
        off = 0
        for n, p in zip(names, m.parameters()):
            g = tr.grads[off : off + p.numel()].view_as(p).cpu()
            want = st["grads"][n]
            assert torch.allclose(g, want, rtol=1e-3, atol=1e-5 * (1 + want.abs().max().item())), n
            off += p.numel()
        tr.step(x, phase_mask=4)
    final = golden["train"][(method, mask)]["steps"][-1]["state_dict"]
    got = m.state_dict()
    for k, v in final.items():
        if v.is_floating_point():
            # Adam moves every parameter by about lr = 1e-3 per step; a gradient that is ~0 may flip sign
            assert torch.allclose(got[k].cpu(), v, atol=2e-5), (k, (got[k].cpu() - v).abs().max())
        else:
            assert torch.equal(got[k].cpu(), v)


def test_masked_gradients_exactly_zero_and_params_untouched():
    from wild_visual_navigation_b200 import ops

    m = _model(384, 200)
    before = m.flat_params.clone()
    tr = ops.FlowTrainer(m, max_rows=256)
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(150, 384, generator=g) * 0.5).cuda()
    yv = (torch.rand(150, generator=g) < 0.6).cuda()
    for _ in range(3):
        tr.step(x, yv)
    names = [n for n, _ in m.named_parameters()]
    off, grads, idx = 0, {}, {}
    for n, p in zip(names, m.parameters()):
        idx[n] = slice(off, off + p.numel())
        off += p.numel()
    for c in (0, 2):
        mask = m.flows[c].mask.bool()
        for net in ("s", "t"):
            w0 = f"flows.{c}.{net}.0.weight"
            g0 = tr.grads[idx[w0]].view(200, 384)
            assert bool((g0[:, ~mask] == 0).all()) and bool((g0[:, mask] != 0).any())
            p0 = m.flat_params[idx[w0]].view(200, 384)
            assert torch.equal(p0[:, ~mask], before[idx[w0]].view(200, 384)[:, ~mask])
            for leaf, shape in ((f"flows.{c}.{net}.4.weight", (384, 200)), (f"flows.{c}.{net}.4.bias", (384,))):
                gl = tr.grads[idx[leaf]].view(shape)
                assert bool((gl[mask] == 0).all())
                assert torch.equal(m.flat_params[idx[leaf]].view(shape)[mask], before[idx[leaf]].view(shape)[mask])


def test_labelled_row_selection_equals_compacted_rows():
    from wild_visual_navigation_b200 import ops

    g = torch.Generator().manual_seed(5)
    x = (torch.randn(90, 90, generator=g) * 0.5).cuda()
    yv = (torch.rand(90, generator=g) < 0.4).cuda()
    a, b = _model(90, 64), _model(90, 64)
    ta, tb = ops.FlowTrainer(a, max_rows=128), ops.FlowTrainer(b, max_rows=128)
    ca = ta.step(x, yv)
    cb = tb.step(x[yv].contiguous())
    n = int(yv.sum())
    assert torch.equal(ta.grads, tb.grads) and torch.equal(a.flat_params, b.flat_params)
    assert torch.equal(ca[:n], cb[:n]) and torch.equal(ta.metrics, tb.metrics)


def test_empty_and_single_row_batches():
    from wild_visual_navigation_b200 import ops

    m = _model(64, 32)
    before = m.flat_params.clone()
    tr = ops.FlowTrainer(m, max_rows=64)
    x = torch.randn(8, 64).cuda()
    tr.step(x, torch.zeros(8, dtype=torch.bool, device="cuda"))
    # torch: mean of nothing is NaN; every weight gradient is a sum over zero rows (0), so Adam moves nothing
    assert torch.isnan(tr.metrics[0]) and tr.metrics[3].item() == 0
    assert bool((tr.grads == 0).all()) and torch.equal(m.flat_params, before) and tr.step_counter.item() == 1
    one = torch.zeros(8, dtype=torch.bool, device="cuda")
    one[3] = True
    conf = tr.step(x, one)
    # one row: torch.std is NaN, and so is its confidence; the loss and gradients are finite
    assert torch.isnan(tr.cg_std).all() and torch.isnan(conf[0]) and torch.isfinite(tr.metrics[0])
    assert bool(torch.isfinite(tr.grads).all()) and bool((tr.grads != 0).any())


def test_trainer_grows_and_keeps_generator_state():
    from wild_visual_navigation_b200 import ops

    m = _model(32, 16)
    tr = ops.FlowTrainer(m, max_rows=64)
    tr.set_confidence(3)   # moving_average: the window lives in the handle
    g = torch.Generator().manual_seed(9)
    ref = ConfidenceState(0.5, "moving_average")
    sd = _sd64(m)
    adam = {}
    for rows in (20, 50, 200, 30):
        x = torch.randn(rows, 32, generator=g) * 0.5
        conf = tr.step(x.cuda())
        sd, _, _, want = orn.train_step(sd, adam, x.double(), ref)
        assert torch.allclose(conf[:rows].cpu(), want.float(), atol=1e-3)
        assert abs(tr.cg_mean.item() - ref.mean.item()) <= 1e-4 * (1 + abs(ref.mean.item()))
    assert tr.max_rows >= 200


def test_estimator_anomaly_mode_trains_and_checkpoints(golden_dir, tmp_path):
    from wild_visual_navigation_b200 import TraversabilityEstimator
    from wild_visual_navigation_b200.traversability_estimator import MissionNode, default_params

    with pytest.raises(ValueError):
        TraversabilityEstimator(device="cuda", anomaly_detection=True, process_group=object())
    with pytest.raises(ValueError):
        TraversabilityEstimator(params=default_params(False), device="cuda", anomaly_detection=True)
    te = TraversabilityEstimator(device="cuda", anomaly_detection=True, min_samples_for_training=0)
    g = torch.Generator().manual_seed(1)
    for _ in range(4):
        x = torch.randn(40, 384, generator=g).cuda()
        yv = (torch.rand(40, generator=g) < 0.4).cuda()
        te.add_mission_node(MissionNode(x, torch.where(yv, 1.0, 0.0), yv))
    out = te.train()
    assert out["loss_trav"] == 0 and out["loss_reco"] == 0 and out["loss_total"] == out["loss_total"]
    te.save_checkpoint(str(tmp_path), "ck.pt")
    ck = torch.load(tmp_path / "ck.pt", weights_only=False)
    assert len(ck["optimizer_state_dict"]["state"]) == 24
    assert list(ck["traversability_loss_state_dict"]) == ["_confidence_generator.mean", "_confidence_generator.var",
                                                          "_confidence_generator.std"]
    # the reference's own checkpoint (LinearRnvp(32, [16]) after three steps) loads and training continues from it
    golden = _cfg(golden_dir)
    torch.save(golden["checkpoint"], tmp_path / "ref.pt")
    p = default_params(True)
    p["model"]["linear_rnvp_cfg"]["input_size"] = 32
    p["model"]["linear_rnvp_cfg"]["coupling_topology"] = [16]
    te2 = TraversabilityEstimator(params=p, device="cuda", anomaly_detection=True, min_samples_for_training=0)
    te2.load_checkpoint(str(tmp_path / "ref.pt"))
    ref_sd = golden["checkpoint"]["model_state_dict"]
    assert all(torch.equal(te2._model.state_dict()[k].cpu(), v) for k, v in ref_sd.items())
    assert te2._trainer.step_counter.item() == 3 and te2.step == 3
    st = golden["checkpoint"]["optimizer_state_dict"]["state"]
    assert torch.equal(te2._trainer.exp_avg[: st[0]["exp_avg"].numel()].cpu(), st[0]["exp_avg"].reshape(-1))
    te2.add_mission_node(MissionNode(torch.randn(30, 32).cuda(), torch.ones(30).cuda(),
                                     torch.ones(30, dtype=torch.bool).cuda()))
    loss = te2.train()["loss_total"]
    assert loss == loss


def test_predict_segments_is_the_row_path_scattered():
    from wild_visual_navigation_b200 import ConfidenceGenerator, TraversabilityInference

    m = _model(90, 200)
    g = torch.Generator().manual_seed(4)
    feat = (torch.randn(50, 90, generator=g) * 0.5).cuda()
    cg = ConfidenceGenerator(0.5, "latest_measurement").cuda()
    n0 = orn.nll(_sd64(m), feat.double().cpu())
    with torch.no_grad():   # a generator state that puts the rows inside its interval
        cg.mean[0], cg.std[0] = n0.mean().item() - 0.5 * n0.std().item(), n0.std().item()
    ti = TraversabilityInference(None, m, cg)
    seg = torch.randint(0, 50, (2, 64, 64), generator=g).cuda()
    trav, conf = ti.predict_segments(feat, seg)
    assert conf is None
    rows = m.nll_confidence(feat, cg)
    assert torch.equal(trav, rows[seg])
    n64 = orn.nll(_sd64(m), feat.double().cpu())
    want = confidence_inference(n64, cg.mean.double().cpu(), cg.std.double().cpu(), 0.5)
    assert (rows.cpu().double() - want).abs().max().item() <= 1e-3
    assert 0.05 < rows.mean().item() < 0.95   # the generator state puts the rows inside its interval


def test_handoff_changes_inference_and_honours_permutation(tmp_path):
    """The reference's reader compares only the last state-dict key, which for LinearRnvp is ``flows.3.invp``: weights
    from a learner with the same permutation are not picked up (the reference's rule, kept).  A learner with another
    permutation is, and the loaded permutation is used at once."""
    from wild_visual_navigation_b200 import ConfidenceGenerator, TraversabilityInference
    from wild_visual_navigation_b200.utils.handoff import read_tmp_state_dict, write_tmp_state_dict

    infer_model, learner = _model(90, 64, seed=42), _model(90, 64, seed=7)
    cg, cg_l = ConfidenceGenerator(0.5, "latest_measurement").cuda(), ConfidenceGenerator(0.5, "latest_measurement").cuda()
    feat = (torch.randn(40, 90, generator=torch.Generator().manual_seed(6)) * 0.5).cuda()
    with torch.no_grad():   # generator states that put the rows inside their intervals
        for c, mm in ((cg, infer_model), (cg_l, learner)):
            n0 = orn.nll(_sd64(mm), feat.double().cpu())
            c.mean[0], c.std[0] = n0.mean().item() - 0.5 * n0.std().item(), n0.std().item()
    ti = TraversabilityInference(None, infer_model, cg)
    seg = torch.arange(40, device="cuda").reshape(1, 5, 8)
    before = ti.predict_segments(feat, seg)[0].clone()
    same = _model(90, 64, seed=42)
    with torch.no_grad():
        same.flat_params.add_(0.01)
    write_tmp_state_dict(same, cg_l, str(tmp_path))
    assert not ti.load_model(str(tmp_path))          # same last key (flows.3.invp): not loaded, as upstream
    write_tmp_state_dict(learner, cg_l, str(tmp_path))
    assert ti.load_model(str(tmp_path))
    after = ti.predict_segments(feat, seg)[0]
    assert not torch.equal(after, before)
    assert torch.equal(after, learner.nll_confidence(feat, cg_l)[seg])
    assert torch.equal(infer_model.flows[3].p, learner.flows[3].p)
    # a permutation loaded into the buffers in place takes effect after refresh_weights (a no-op re-pack here)
    with torch.no_grad():
        infer_model.flows[1].p.copy_(torch.flip(infer_model.flows[1].p, [0]))
        infer_model.flows[1].invp.copy_(torch.argsort(infer_model.flows[1].p))
    ti.refresh_weights()
    n64 = orn.nll(_sd64(infer_model), feat.double().cpu())
    want = confidence_inference(n64, cg.mean.double().cpu(), cg.std.double().cpu(), 0.5)
    got = ti.predict_segments(feat, seg)[0].reshape(-1)
    assert (got.cpu().double() - want).abs().max().item() <= 1e-3
    assert not read_tmp_state_dict(infer_model, cg, str(tmp_path / "missing"))


class _Grid:
    """Stands in for the feature extractor: the per-pixel path reads only its token grid."""

    def __init__(self, g):
        self.grid = g


# size: a square frame from a g = size / 8 grid through TraversabilityInference, or a name in _PIXEL_GEOMETRY: a
# (gh, gw) grid to an (H, W) output through ops.FlowInference with its own pixel chunk
_PIXEL_GEOMETRY = {
    "grid28x42-224x336": (28, 42, 224, 336, 0),        # non-square grid and output: a swapped gh / gw or sy / sx shows
    "grid1x7-16x56": (1, 7, 16, 56, 0),                # degenerate grid: one token row, sy = 0
    "grid5x7-37x53-chunk384": (5, 7, 37, 53, 384),     # 1961 pixels a frame: chunks of 384 straddle the frames
}


@pytest.mark.parametrize("size,dim,batch", [(224, 384, 1), (224, 384, 3), (448, 384, 1), (448, 384, 3), (224, 90, 3),
                                            (448, 90, 1), ("grid28x42-224x336", 384, 1), ("grid1x7-16x56", 90, 2),
                                            ("grid5x7-37x53-chunk384", 384, 3)])
def test_pixel_map_matches_float64(size, dim, batch):
    """Per-pixel maps from a (B, gh*gw, D) token grid (DINO ViT-S/8 tokens: D = 384; the STEGO code: D = 90), pixel by
    pixel against float64, for square frames and for the non-square, degenerate and chunk-straddling geometries of
    _PIXEL_GEOMETRY.

    Bound.  The path rounds to bf16 at fixed points: every weight, mu = u * mask and the two hidden activations of each
    net; everything else is fp32.  ``oracle.linear_rnvp.nll_bf16`` applies exactly these roundings in float64, so
    e = |nll_bf16 - nll64| is the rounding's own effect on each pixel.  The GPU rounds values computed in fp32, so a
    value within an fp32 error of a bf16 rounding boundary can go to the other neighbour: that moves one operand by one
    bf16 ulp, the same kind of step that e sums over ~1500 operands per pixel, so its size is bounded by the frame's
    typical e.  An element passes when |nll_gpu - nll64| <= 3 e + 6 rms_frame(e) + 64 u (1 + |nll64|).  The factors
    are not derived: with 3 rms_frame(e) the worst of 602k pixels (448^2, B = 3, D = 384) measured 1.11 times the bound
    on an H100, so the flip term was doubled.  The same bound
    must reject the first permutation dropped, the map shifted by one pixel and, for a non-square grid, the tokens read
    as a (gw, gh) grid.  (Dropping the last permutation cannot show: sum(z^2) does not depend on it.  Swapping s and t
    of these nets, which differ by 0.05-sized weight noise, moves the NLL by less than the bf16 resolution; the fp32 row
    test holds the swap.)"""
    import torch.nn.functional as F

    from wild_visual_navigation_b200 import ConfidenceGenerator, TraversabilityInference, ops

    if isinstance(size, int):
        gh = gw = size // 8
        H = W = size
        seed = size + dim + batch
    else:
        gh, gw, H, W, chunk = _PIXEL_GEOMETRY[size]
        seed = H + W + dim + batch
    m = _model(dim, 200)
    gen = torch.Generator().manual_seed(seed)
    tokens = (torch.randn(batch, gh * gw, dim, generator=gen) * 0.5).cuda()
    sd = {k: (v.detach().double() if v.is_floating_point() else v) for k, v in m.state_dict().items()}

    def upsampled(rows, cols):
        return F.interpolate(tokens.double().view(batch, rows, cols, dim).permute(0, 3, 1, 2), (H, W), mode="bilinear",
                             align_corners=True).permute(0, 2, 3, 1).reshape(-1, dim)

    dense = upsampled(gh, gw)
    ref = orn.nll(sd, dense).view(batch, H, W)
    emu = orn.nll_bf16(sd, dense).view(batch, H, W)
    cg = ConfidenceGenerator(0.5, "latest_measurement").cuda()
    with torch.no_grad():
        cg.mean[0], cg.std[0] = ref.mean().item() - 0.5 * ref.std().item(), ref.std().item()
    if isinstance(size, int):
        ti = TraversabilityInference(_Grid(gh), m, cg)
        trav, conf = ti.predict_from_tokens(tokens, size)
        assert conf is None and trav.shape == (batch, H, W)
        _, nll = ti._flow_infer.pixels(m, tokens, (gh, gw), (H, W), cg.mean.data, cg.std.data, 0.5, want_nll=True)
    else:
        fi = ops.FlowInference(dim, 200, chunk_pixels=chunk)
        fi.set_params(m.flat_params)
        trav, nll = fi.pixels(m, tokens, (gh, gw), (H, W), cg.mean.data, cg.std.data, 0.5, want_nll=True)
        assert trav.shape == (batch, H, W)
    e = (emu - ref).abs()
    bound = 3 * e + 6 * e.pow(2).mean().sqrt() + 64 * U * (1 + ref.abs())
    err = (nll.double() - ref).abs()
    assert bool((err <= bound).all()), (err / bound).max().item()
    want = confidence_inference(nll.double(), cg.mean.double(), cg.std.double(), 0.5)
    assert (trav.double() - want).abs().max().item() <= 1e-5
    # negative controls under the same bound
    noperm = dict(sd)
    noperm["flows.1.p"] = torch.arange(dim, device="cuda")
    assert not bool(((nll.double() - orn.nll(noperm, dense).view(batch, H, W)).abs() <= bound).all())
    assert not bool(((nll.double() - torch.roll(ref, 1, 2)).abs() <= bound).all())
    if gh != gw:   # the tokens read as a (gw, gh) grid: what a kernel with gh and gw swapped computes
        swapped = orn.nll(sd, upsampled(gw, gh)).view(batch, H, W)
        assert not bool(((nll.double() - swapped).abs() <= bound).all())


def test_pixel_map_follows_refresh_and_loaded_permutation():
    from wild_visual_navigation_b200 import ConfidenceGenerator, TraversabilityInference

    m = _model(90, 64)
    cg = ConfidenceGenerator(0.5, "latest_measurement").cuda()
    tokens = (torch.randn(1, 28 * 28, 90, generator=torch.Generator().manual_seed(2)) * 0.5).cuda()
    ti = TraversabilityInference(_Grid(28), m, cg)
    n0 = ti._flow_infer.pixels(m, tokens, (28, 28), (224, 224), cg.mean.data, cg.std.data, 0.5, want_nll=True)[1].clone()
    with torch.no_grad():   # a permutation loaded into the buffers takes effect at once
        m.flows[3].p.copy_(torch.flip(m.flows[3].p, [0]))
        m.flows[3].invp.copy_(torch.argsort(m.flows[3].p))
    n1 = ti._flow_infer.pixels(m, tokens, (28, 28), (224, 224), cg.mean.data, cg.std.data, 0.5, want_nll=True)[1].clone()
    # the last permutation does not change sum(z^2): only the fp32 summation order of the NLL changes
    assert torch.allclose(n0, n1, rtol=1e-6, atol=1e-4)
    with torch.no_grad():
        m.flows[1].p.copy_(torch.flip(m.flows[1].p, [0]))
        m.flows[1].invp.copy_(torch.argsort(m.flows[1].p))
        m.flat_params.mul_(1.1)
    n2 = ti._flow_infer.pixels(m, tokens, (28, 28), (224, 224), cg.mean.data, cg.std.data, 0.5, want_nll=True)[1].clone()
    assert not torch.equal(n1, n2)    # permutation 1 is read from the buffer
    ti.refresh_weights()              # the weights only after the re-pack
    n3 = ti._flow_infer.pixels(m, tokens, (28, 28), (224, 224), cg.mean.data, cg.std.data, 0.5, want_nll=True)[1]
    assert not torch.equal(n2, n3)
    sd = {k: (v.detach().double() if v.is_floating_point() else v) for k, v in m.state_dict().items()}
    import torch.nn.functional as F
    dense = F.interpolate(tokens.double().view(1, 28, 28, 90).permute(0, 3, 1, 2), (224, 224), mode="bilinear",
                          align_corners=True).permute(0, 2, 3, 1).reshape(-1, 90)
    ref = orn.nll(sd, dense).view(1, 224, 224)
    e = (orn.nll_bf16(sd, dense).view(1, 224, 224) - ref).abs()
    assert bool(((n3.double() - ref).abs() <= 3 * e + 6 * e.pow(2).mean().sqrt() + 64 * U * (1 + ref.abs())).all())
