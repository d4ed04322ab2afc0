"""The DoubleMLP learner on the GPU: row forward, train step, per-pixel / per-segment inference, checkpoints and the
hand-off, each against float64 (oracle/double_mlp.py) or the reference's own fp32 run (tests/golden/double_mlp.pt).
The train step's statistics, generator update, gradients and Adam are checked phase by phase against float64 under a
derived bound in test_double_mlp_train_step_gpu.py.

Row forward bound (u = 2^-24): every layer is one fp32 fma chain over K terms plus the bias, so
|z - z64| <= e_in |W|^T + (K + 2) u ((|a| + e_in) |W|^T + |b|); ReLU is 1-Lipschitz and the sigmoid 1/4-Lipschitz
(+ 4 u for expf and the division).
"""
import math
import os
import sys
import types

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import double_mlp as odm  # noqa: E402
from oracle.wvn_path import ConfidenceState  # noqa: E402

U = 2.0**-24
METHODS = ("latest_measurement", "running_mean", "moving_average", "kalman_filter")
METHOD_ID = {m: i for i, m in enumerate(("latest_measurement", "running_mean", "kalman_filter", "moving_average"))}
CASES = [(m, True) for m in METHODS] + [("latest_measurement", False)]


def _model(D, h1, h2, seed=42, scale=1.0):
    from wild_visual_navigation_b200 import DoubleMLP

    torch.manual_seed(seed)
    m = DoubleMLP(D, [h1, h2, 1]).cuda()
    with torch.no_grad():
        m.flat_params.mul_(scale)
    return m


def _sd64(m):
    return {k: v.detach().double() for k, v in m.state_dict().items()}


def _rows(R, D, seed, p_valid=0.3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(R, D, generator=g, device="cuda") * 0.8 + 0.1
    yv = torch.rand(R, generator=g, device="cuda") < p_valid
    y = torch.where(yv, torch.rand(R, generator=g, device="cuda").clamp(min=0.001), torch.zeros(R, device="cuda"))
    return x, y, yv


def forward_bound(sd, x):
    """float64 DoubleMLP output and its element-wise bound for the fp32 kernels."""
    x = x.double()
    outs, errs = [], []
    for n in range(2):
        a, e = x, torch.zeros_like(x)
        for i in range(3):
            W, b = sd[f"networks.{n}.{2 * i}.weight"], sd[f"networks.{n}.{2 * i}.bias"]
            z = a @ W.T + b
            e = e @ W.abs().T + (W.shape[1] + 2) * U * ((a.abs() + e) @ W.abs().T + b.abs())
            a = z.clamp_min(0) if i < 2 else z
        outs.append(a), errs.append(e)
    return (torch.cat([torch.sigmoid(outs[0]), outs[1]], 1),
            torch.cat([errs[0] / 4 + 4 * U, errs[1]], 1))


def assert_within(got, ref, bound, tag):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    assert not bool(bad.any()), (f"{tag}: {int(bad.sum())} of {bad.numel()} outside; worst ratio "
                                 f"{(err / bound.clamp_min(1e-300)).max().item():.3g}")


# ------------------------------------------------------------------------------------------------ row forward
@pytest.mark.gpu
@pytest.mark.parametrize("D", [90, 384, 768])
@pytest.mark.parametrize("h1,h2", [(64, 32), (128, 32), (20, 7)])
def test_row_forward(D, h1, h2):
    from wild_visual_navigation_b200.utils import Data

    m = _model(D, h1, h2, scale=2.0)
    sd = _sd64(m)
    for R in (1, 63, 64, 65, 4097):
        x = _rows(R, D, R)[0]
        out = m(Data(x=x))
        assert out.shape == (R, 1 + D)
        ref, bound = forward_bound(sd, x)
        assert_within(out, ref, bound, f"forward D={D} [{h1},{h2}] R={R}")


@pytest.mark.gpu
def test_row_forward_negative_control():
    """The two networks' h2 activations swapped (net 1's layer 2 feeding net 0's head and the reverse) fail."""
    from wild_visual_navigation_b200.utils import Data

    m = _model(384, 64, 32, scale=2.0)
    sd = _sd64(m)
    x = _rows(65, 384, 1)[0]
    out = m(Data(x=x))
    bad = dict(sd)
    for w in ("weight", "bias"):
        bad[f"networks.0.2.{w}"], bad[f"networks.1.2.{w}"] = sd[f"networks.1.2.{w}"], sd[f"networks.0.2.{w}"]
    ref, bound = forward_bound(bad, x)
    with pytest.raises(AssertionError):
        assert_within(out, ref, bound, "swapped")


# ------------------------------------------------------------------------------------------------ train step
def _trainer(m, method, balanced, max_rows=512):
    from wild_visual_navigation_b200 import ops

    tr = ops.DoubleMlpTrainer(m, max_rows=max_rows, anomaly_balanced=balanced)
    tr.set_confidence(METHOD_ID[method])
    return tr


def _split(flat, sd):
    out, off = {}, 0
    for k, v in sd.items():
        out[k] = flat[off : off + v.numel()].view(v.shape).double()
        off += v.numel()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("method,balanced", CASES)
def test_three_steps_reproduce_the_reference_fp32_run(golden_dir, method, balanced):
    """From the golden's init and rows (D = 32, [16, 8, 1]), the same three steps as the reference's fp32 run."""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import test_double_mlp_oracle as cpu

    golden = torch.load(os.path.join(golden_dir, "double_mlp.pt"), weights_only=False)
    from wild_visual_navigation_b200 import DoubleMLP
    from wild_visual_navigation_b200.utils import Data

    m = DoubleMLP(32, [16, 8, 1])
    m.load_state_dict(cpu._init(golden))
    m = m.cuda()
    tr = _trainer(m, method, balanced)
    out = []
    for st in golden["train"][(method, balanced)]["steps"]:
        x = st["x"].cuda()
        res = m(Data(x=x)).cpu()
        sd = m.state_dict()
        conf = tr.step(x, st["y"].cuda(), st["y_valid"].cuda()).cpu()
        met = tr.metrics.cpu()
        aux = {"loss_trav": met[1], "loss_reco": met[2], "loss_trav_confidence": met[3], "confidence": conf,
               "mean": met[4:5], "std": met[5:6]}
        out.append((res, met[0], aux, {k: v.cpu() for k, v in _split(tr.grads, sd).items()}))
    assert cpu._matches(golden, method, balanced, out, {k: v.cpu().double() for k, v in m.state_dict().items()})


@pytest.mark.gpu
def test_determinism_and_dead_units():
    """Two identical two-step runs are bit-identical; net 1's first 8 hidden units are dead (bias -1e3): their
    weight / bias gradients and the layer-2 columns that read them are exactly 0 and Adam leaves them bit-identical."""
    runs = []
    for _ in range(2):
        m = _model(384, 64, 32)
        with torch.no_grad():
            m.networks[1][0].bias[:8] = -1e3
        before = {k: v.clone() for k, v in m.state_dict().items()}
        tr = _trainer(m, "moving_average", True)
        confs = []
        for s in range(2):
            x, y, yv = _rows(300, 384, 20 + s)
            confs.append(tr.step(x, y, yv).clone())
        g = _split(tr.grads, before)
        assert torch.count_nonzero(g["networks.1.0.weight"][:8]) == 0 and torch.count_nonzero(g["networks.1.0.bias"][:8]) == 0
        assert torch.count_nonzero(g["networks.1.2.weight"][:, :8]) == 0
        sd = m.state_dict()
        assert torch.equal(sd["networks.1.0.weight"][:8], before["networks.1.0.weight"][:8])
        assert torch.equal(sd["networks.1.2.weight"][:, :8], before["networks.1.2.weight"][:, :8])
        runs.append((m.flat_params.clone(), torch.cat(confs), tr.metrics.clone(), tr.grads.clone()))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("labelled", [True, False])
@pytest.mark.parametrize("method", ["latest_measurement", "moving_average"])
def test_nan_input_row_matches_the_simple_mlp_step(labelled, method):
    """A row with a NaN feature, labelled or not: the metrics, every row's confidence and whether each layer's
    gradient holds a NaN are NaN exactly where the fused SimpleMLP step (csrc/mlp_train_fused.cu) has them on the same
    rows (both steps' ReLU is fmaxf, so the NaN enters through the reconstruction error of that row only)."""
    from wild_visual_navigation_b200 import SimpleMLP, ops

    R, D = 300, 384
    x, y, yv = _rows(R, D, 8)
    row = int(yv.nonzero()[0, 0]) if labelled else int((~yv).nonzero()[0, 0])
    x[row, 5] = float("nan")
    dm = _model(D, 64, 32)
    tr = _trainer(dm, method, True)
    conf_d = tr.step(x, y, yv).clone()
    torch.manual_seed(42)
    sm = SimpleMLP(D, [256, 32, 1], True).cuda()
    ts = ops.MlpTrainer(sm.flat_params, D, 256, 32, max_rows=512)
    ts.set_confidence(METHOD_ID[method])
    conf_s = ts.step(x, y, yv).clone()
    torch.cuda.synchronize()
    assert torch.equal(torch.isnan(tr.metrics), torch.isnan(ts.metrics)), (tr.metrics, ts.metrics)
    assert torch.equal(torch.isnan(conf_d), torch.isnan(conf_s[:R]))
    gd = _split(tr.grads, dm.state_dict())
    gs = _split(ts.grads[:-1], sm.state_dict())
    for layer in ("0", "2", "4"):
        nan_d = any(bool(torch.isnan(gd[f"networks.{n}.{layer}.{w}"]).any()) for n in (0, 1) for w in ("weight", "bias"))
        nan_s = any(bool(torch.isnan(gs[f"layers.{layer}.{w}"]).any()) for w in ("weight", "bias"))
        assert nan_d == nan_s, (layer, nan_d, nan_s)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["all", "one", "two", "none", "one_of_many", "none_unbalanced"])
def test_labels_edge_cases(case):
    """Every row labelled; one or two rows; none (mean of an empty set: NaN); one among many (std of one: NaN).
    Gradients and the total loss are NaN exactly where the float64 reference's are (as for the SimpleMLP step)."""
    R, D = 300, 384
    x, y, yv = _rows(R, D, 7)
    if case == "all":
        yv[:] = True
    elif case in ("one", "two"):
        R = 1 if case == "one" else 2
        x, y, yv = x[:R], y[:R], torch.ones(R, dtype=torch.bool, device="cuda")
    elif case.startswith("none"):
        yv[:] = False
    elif case == "one_of_many":
        yv[:] = False
        yv[17] = True
    y = torch.where(yv, y, torch.zeros_like(y))
    balanced = not case.endswith("unbalanced")
    m = _model(D, 64, 32)
    sd = _sd64(m)
    _, g_ref, loss, _ = odm.train_step(sd, {}, x.double(), y, yv, ConfidenceState(0.5), anomaly_balanced=balanced)
    tr = _trainer(m, "latest_measurement", balanced)
    tr.step(x, y, yv)
    g = _split(tr.grads, sd)
    for k in g_ref:
        assert torch.equal(torch.isnan(g[k]), torch.isnan(g_ref[k])), (case, k)
    assert math.isnan(tr.metrics[0].item()) == math.isnan(loss.item()), case


# ------------------------------------------------------------------------------------------------ per-pixel maps
def _packed_sd(m):
    return {k: v.float() for k, v in odm.packed_simple_mlp(dict(m.state_dict())).items()}


def _double_infer(m, chunk_rows=0):
    from wild_visual_navigation_b200 import ops

    h = ops.MlpInference(m.input_size, m.hidden[0], m.hidden[1], chunk_rows, double=True)
    h.set_params(m.flat_params)
    return h


# unfused geometries (W % 64 != 0) and shapes outside the fused head (h1 = 256, h2 = 7)
PIXEL_CASES = {
    "224_b1_d384_h64": (28, 28, 224, 224, 1, 384, 64, 32),
    "224_b3_d90_h64": (28, 28, 224, 224, 3, 90, 64, 32),
    "nonsquare_d384_h64": (28, 36, 224, 288, 1, 384, 64, 32),
    "448_b1_d90_h256": (56, 56, 448, 448, 1, 90, 256, 32),
    "224_b1_d384_h20_7": (28, 28, 224, 224, 1, 384, 20, 7),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(PIXEL_CASES))
def test_unfused_pixel_maps_pixel_by_pixel(case):
    """wvn_mlp_infer_pixels on the DoubleMLP layout where the fused head does not apply, against the unfused path's
    float64 emulation (bf16 x, weights and activations; test_pixel_head_gpu.unfused_head_ref) of the packed
    block-structured MLP, with two negative controls: the map shifted by one pixel, and the reference built with the
    networks' h2 halves swapped."""
    import test_pixel_head_gpu as ph

    gh, gw, H, W, B, D, h1, h2 = PIXEL_CASES[case]
    m = _model(D, h1, h2, scale=3.0)
    tok = ph.make_tokens(B, gh * gw, D, "cuda")
    sd = _packed_sd(m)
    ys, es, xs = [], [], []
    for b in range(B):
        yb, eb, xb = ph.unfused_head_ref(tok[b], sd, gh, gw, H, W)
        ys.append(yb), es.append(eb), xs.append(xb)
    yv, eps, x = torch.cat(ys), torch.cat(es), torch.cat(xs)
    loss = ((yv[:, :D] - x) ** 2).mean(1)
    cg = ph.quantile_window(loss)
    ref = ph.mlp_head_ref(yv, eps, x, D, D, *cg)
    trav, conf = ph.run_pixels(_double_infer(m), tok, B, gh, gw, H, W, cg)
    ph.assert_within(trav.reshape(-1), ref["trav"], ref["trav_bound"], f"dm_{case}_trav")
    ph.assert_within(conf.reshape(-1), ref["conf"], ref["conf_bound"], f"dm_{case}_conf")
    with pytest.raises(AssertionError):
        ph.assert_within(torch.roll(trav, 1, dims=-1).reshape(-1), ref["trav"], ref["trav_bound"], "shifted")
    bad = dict(sd)
    w3 = sd["layers.4.weight"].clone()
    w3[:1], w3[1:] = torch.roll(sd["layers.4.weight"][:1], h2, 1), torch.roll(sd["layers.4.weight"][1:], h2, 1)
    bad["layers.4.weight"] = w3
    yb, eb, xb = ph.unfused_head_ref(tok[0], bad, gh, gw, H, W)
    ref_bad = ph.mlp_head_ref(yb, eb, xb, D, D, *cg)
    with pytest.raises(AssertionError):
        ph.assert_within(conf[:1].reshape(-1), ref_bad["conf"], ref_bad["conf_bound"], "swapped")


def _fused_ref(monkeypatch, m, tok, B, gh, gw, H, W):
    """test_pixel_head_gpu.fused_head_ref on the packed block-structured operands: G of both networks (2 h1), h2 of
    both (64; w0 reads net 0's half, R net 1's), so the reference follows the DoubleMLP head's own algebra."""
    import test_pixel_head_gpu as ph

    monkeypatch.setattr(ph, "H1", 2 * m.hidden[0])
    monkeypatch.setattr(ph, "H2", 2 * m.hidden[1])
    op = ph.head_operands(_packed_sd(m))
    return ph.stack_refs([ph.fused_head_ref(tok[b], op, gh, gw, H, W) for b in range(B)]), op


FUSED_CASES = {
    "448_b3_d90_h128": (56, 56, 448, 448, 3, 90, 128),
    "448_b1_d384_h64": (56, 56, 448, 448, 1, 384, 64),
    "448_b1_d384_h128": (56, 56, 448, 448, 1, 384, 128),
    "nonsquare_24x40_d384_h64": (24, 40, 194, 320, 3, 384, 64),
    "ww9_14_128_d90_h64": (14, 14, 128, 128, 9, 90, 64),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(FUSED_CASES))
def test_fused_pixel_maps_pixel_by_pixel(case, monkeypatch):
    """The fused head's DoubleMLP instantiation (pixels) against the fused head's float64 reference on the packed
    operands, under the loss window and the quantile window; negative controls: the map shifted by one pixel, and the
    reference with net 0 and net 1's roles swapped (the logit read from net 1's h2, the reconstruction from net 0's)."""
    import test_pixel_head_gpu as ph

    gh, gw, H, W, B, D, h1 = FUSED_CASES[case]
    assert ph.window_width(gh, gw, H, W) > 0
    m = _model(D, h1, 32, scale=3.0)
    tok = ph.make_tokens(B, gh * gw, D, "cuda")
    ref, op = _fused_ref(monkeypatch, m, tok, B, gh, gw, H, W)
    h = _double_infer(m)
    cg = ph.loss_window(ref["loss"].max().item())
    trav, conf = ph.run_pixels(h, tok, B, gh, gw, H, W, cg)
    ph.check_maps(trav, conf, ref, cg, f"dm_fused_{case}_losswin", regimes=False)
    cg2 = ph.quantile_window(ref["loss"])
    trav2, conf2 = ph.run_pixels(h, tok, B, gh, gw, H, W, cg2)
    ph.check_maps(trav2, conf2, ref, cg2, f"dm_fused_{case}_quantwin", regimes=True)
    assert torch.equal(trav, trav2)
    with pytest.raises(AssertionError):
        ph.check_maps(torch.roll(trav, 1, dims=-1), conf, ref, cg, "shifted", regimes=False)
    sw = dict(op)
    sw["w0"] = torch.roll(op["w0"], 32)
    sw["R"] = torch.roll(op["R"], 32, 1)
    ref_sw = ph.stack_refs([ph.fused_head_ref(tok[b], sw, gh, gw, H, W) for b in range(B)])
    with pytest.raises(AssertionError):
        ph.check_maps(trav, conf, ref_sw, cg, "swapped", regimes=False)


@pytest.mark.gpu
@pytest.mark.parametrize("h1", [64, 128])
def test_pixels_from_vit_fused(h1, monkeypatch):
    """pixels_from_vit on a DINO ViT-S/8 handle at B = 9 (npad rows per frame, a second chunk 8 frames in) equals
    pixels on the same tokens bit for bit and meets the fused reference; TraversabilityInference.predict_from_tokens
    takes it for the backbone's own tokens.  A DoubleMLP outside the fused shapes is refused there."""
    import test_pixel_head_gpu as ph
    from oracle.dino_vit import ViTConfig, synthetic_state_dict
    from wild_visual_navigation_b200 import ConfidenceGenerator, TraversabilityInference, ops
    from wild_visual_navigation_b200._C import WvnError

    cfg = ViTConfig.from_name("vit_small", 8, 448)
    vit = ops.ViTBackbone(448, 8, cfg.dim, cfg.depth, cfg.heads, cfg.mlp_dim, synthetic_state_dict(cfg, seed=3),
                          max_batch=9)
    img = torch.rand(9, 3, 448, 448, generator=torch.Generator().manual_seed(1)).cuda()
    tokens = vit.forward(img)
    m = _model(384, h1, 32, scale=3.0)
    h = _double_infer(m)
    ref, _ = _fused_ref(monkeypatch, m, tokens[:2], 2, 56, 56, 448, 448)
    cg = ph.quantile_window(ref["loss"])
    cm, cs = torch.tensor([cg[0]], device="cuda"), torch.tensor([cg[1]], device="cuda")
    tv, cv = h.pixels_from_vit(vit, 9, (448, 448), cm, cs, cg[2])
    tp, cp = h.pixels(tokens, (56, 56), (448, 448), cm, cs, cg[2])
    torch.cuda.synchronize()
    assert torch.equal(tv, tp) and torch.equal(cv, cp)
    ph.check_maps(tv[:2], cv[:2], ref, cg, f"dm_vit_h{h1}", regimes=True)
    cgm = ConfidenceGenerator(cg[2], "latest_measurement").cuda()
    with torch.no_grad():
        cgm.mean[0], cgm.std[0] = cg[0], cg[1]
    ti = TraversabilityInference(types.SimpleNamespace(grid=56, _model=vit), m, cgm)
    a = ti.predict_from_tokens(tokens, 448)
    assert torch.equal(a[0], tv) and torch.equal(a[1], cv)
    odd = _double_infer(_model(384, 20, 7))
    with pytest.raises(WvnError):
        odd.pixels_from_vit(vit, 1, (448, 448), cm, cs, 0.5)


@pytest.mark.gpu
def test_predict_segments_against_float64_rows():
    """Segment-wise mode: rows x -> bf16 -> the packed GEMM chain -> trav / conf, against the float64 emulation, and
    scattered through seg."""
    import test_pixel_head_gpu as ph
    from wild_visual_navigation_b200 import ConfidenceGenerator, TraversabilityInference

    D, S = 384, 777
    m = _model(D, 64, 32, scale=3.0)
    cg = ConfidenceGenerator(0.5, "latest_measurement").cuda()
    feat = _rows(S, D, 4)[0]
    sd = _packed_sd(m)
    xb = ph._bf(feat)
    W1, b1 = ph._bf(sd["layers.0.weight"]), sd["layers.0.bias"].double()
    W2, b2 = ph._bf(sd["layers.2.weight"]), sd["layers.2.bias"].double()
    W3, b3 = ph._bf(sd["layers.4.weight"]), sd["layers.4.bias"].double()
    W3, b3 = torch.cat([W3[1:], W3[:1]]), torch.cat([b3[1:], b3[:1]])
    z1 = xb @ W1.T + b1
    e1 = ph.C_ACC * 448 * U * (xb.abs() @ W1.abs().T + b1.abs()) + 2.0**-23 * z1.abs()
    a1, d1 = ph._relu_bf16_flip(z1, e1)
    z2 = a1 @ W2.T + b2
    e2 = d1 @ W2.abs().T + ph.C_ACC * 128 * U * ((a1.abs() + d1) @ W2.abs().T + b2.abs()) + 2.0**-23 * z2.abs()
    a2, d2 = ph._relu_bf16_flip(z2, e2)
    yv = a2 @ W3.T + b3
    eps = d2 @ W3.abs().T + ph.C_ACC * 64 * U * ((a2.abs() + d2) @ W3.abs().T + b3.abs()) + 2.0**-23 * yv.abs()
    loss = ((yv[:, :D] - xb) ** 2).mean(1)
    cgw = ph.quantile_window(loss)
    with torch.no_grad():
        cg.mean[0], cg.std[0] = cgw[0], cgw[1]
    cg.std_factor = cgw[2]
    ref = ph.mlp_head_ref(yv, eps, xb, D, D, *cgw)
    ti = TraversabilityInference(types.SimpleNamespace(grid=0, _model=None), m, cg)
    seg = torch.randint(0, S, (2, 64, 64), device="cuda")
    trav, conf = ti.predict_segments(feat, seg)
    ph.assert_within(trav.reshape(-1), ref["trav"][seg].reshape(-1), ref["trav_bound"][seg].reshape(-1), "seg_trav")
    ph.assert_within(conf.reshape(-1), ref["conf"][seg].reshape(-1), ref["conf_bound"][seg].reshape(-1), "seg_conf")


# ------------------------------------------------------------------------------------------------ estimator
def _params(D=32, hs=(16, 8, 1)):
    from wild_visual_navigation_b200.traversability_estimator.traversability_estimator import default_params

    p = default_params()
    p["model"]["name"] = "DoubleMLP"
    p["model"]["double_mlp_cfg"] = {"input_size": D, "hidden_sizes": list(hs)}
    return p


@pytest.mark.gpu
def test_estimator_default_init_is_the_reference_seed42_init(golden_dir):
    from wild_visual_navigation_b200 import TraversabilityEstimator
    from wild_visual_navigation_b200.traversability_estimator.traversability_estimator import default_params

    golden = torch.load(os.path.join(golden_dir, "double_mlp.pt"), weights_only=False)
    p = default_params()
    p["model"]["name"] = "DoubleMLP"
    est = TraversabilityEstimator(params=p)
    sd = est._model.state_dict()
    for k, s in golden["init384"].items():
        assert torch.equal(sd[k].cpu().reshape(-1)[:8], s["first"]) and sd[k].double().sum().item() == s["sum"]
    with pytest.raises(ValueError):
        est.train_on_padded(None, None, None, None)


@pytest.mark.gpu
def test_checkpoints_and_handoff(golden_dir, tmp_path):
    """The estimator loads the reference's checkpoint (weights, Adam state, generator) and writes one the reference's
    format reads back; the hand-off file round-trips and TraversabilityInference.load_model picks up new weights."""
    from wild_visual_navigation_b200 import DoubleMLP, TraversabilityEstimator, TraversabilityInference
    from wild_visual_navigation_b200.traversability_estimator import MissionNode

    golden = torch.load(os.path.join(golden_dir, "double_mlp.pt"), weights_only=False)
    ck = golden["checkpoint"]
    path = tmp_path / "ref.pt"
    torch.save(ck, path)
    est = TraversabilityEstimator(params=_params(), min_samples_for_training=0)
    est.load_checkpoint(str(path))
    for k, v in ck["model_state_dict"].items():
        assert torch.equal(est._model.state_dict()[k].cpu(), v)
    assert int(est._trainer.step_counter.item()) == 3
    est.save_checkpoint(str(tmp_path), "mine.pt")
    mine = torch.load(tmp_path / "mine.pt", weights_only=False)
    assert list(mine["model_state_dict"]) == list(ck["model_state_dict"])
    assert list(mine["traversability_loss_state_dict"]) == list(ck["traversability_loss_state_dict"])
    ref_opt = torch.optim.Adam(DoubleMLP(32, [16, 8, 1]).parameters(), lr=1e-3)
    ref_opt.load_state_dict(mine["optimizer_state_dict"])   # the reference's optimizer reads it back
    for i, st in ck["optimizer_state_dict"]["state"].items():
        assert torch.equal(mine["optimizer_state_dict"]["state"][i]["exp_avg"].cpu(), st["exp_avg"])

    # hand-off: the inference side starts from the seed-42 init, the learner trains one step and writes the file
    torch.manual_seed(42)
    infer_model = DoubleMLP(32, [16, 8, 1]).cuda()
    cg = est._traversability_loss._confidence_generator
    ti = TraversabilityInference(types.SimpleNamespace(grid=0, _model=None), infer_model, cg)
    x, y, yv = _rows(60, 32, 9)
    for _ in range(12):
        est.add_mission_node(MissionNode(x, y, yv))
    assert est.train()["loss_total"] != -1
    handoff = est.write_model_handoff(str(tmp_path))
    assert ti.load_model(handoff)
    for k, v in est._model.state_dict().items():
        assert torch.equal(infer_model.state_dict()[k], v)
    assert not ti.load_model(handoff)   # unchanged weights: no reload
