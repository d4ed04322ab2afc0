"""Segment-wise inference on the GPU: the paint kernel ``wvn_segment_maps`` against ``gather`` element by element, the
padded-row inference of every learner against ``predict_segments`` on each frame's compacted rows, and
``HotPathStep(prediction_per_pixel=False)`` / ``HotPathStep(feature_type="torchvision")`` against the same work composed
by hand, eager and through ``capture`` / ``replay``."""
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ paint kernel
def _gather_ref(seg, n_rows, v):
    """v[b, seg[b, p]] with NaN for ids outside [0, n_rows[b])."""
    B, S = v.shape
    ids = seg.reshape(B, -1).long()
    live = (ids >= 0) & (ids < n_rows.long()[:, None])
    out = v.gather(1, ids.clamp(0, S - 1))
    return torch.where(live, out, torch.full_like(out, float("nan"))).view(seg.shape)


def _identical(a, b):
    return torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(a.nan_to_num(), b.nan_to_num())


@pytest.mark.parametrize("dtype", [torch.int64, torch.int32])
@pytest.mark.parametrize("B", [1, 3, 32])
@pytest.mark.parametrize("hw", [(224, 224), (448, 448), (223, 227)])
def test_segment_maps_equals_gather(dtype, B, hw):
    from wild_visual_navigation_b200 import ops

    S = 40
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + hw[1])
    seg = torch.randint(-3, S + 3, (B, *hw), generator=g, device="cuda").to(dtype)   # negative ids and ids >= S
    n_rows = torch.randint(0, S + 1, (B,), generator=g, device="cuda").int()
    n_rows[-1] = 0 if B > 1 else n_rows[-1]                                           # a frame with no rows
    n_rows[0] = S
    trav = torch.rand(B, S, generator=g, device="cuda")
    conf = torch.rand(B, S, generator=g, device="cuda")
    tm, cm = ops.segment_maps(seg, n_rows, trav, conf)
    assert tm.shape == seg.shape and cm.shape == seg.shape
    assert _identical(tm, _gather_ref(seg, n_rows, trav)) and _identical(cm, _gather_ref(seg, n_rows, conf))
    if B > 1:
        assert torch.isnan(tm[-1]).all()
    # the LinearRnvp's form: no confidence map
    tm2, cm2 = ops.segment_maps(seg, n_rows, trav)
    assert cm2 is None and _identical(tm2, tm)


def test_segment_maps_does_not_read_padding_rows():
    """Padding rows full of garbage are never read: ids in [n_rows, smax) give NaN, not the garbage."""
    from wild_visual_navigation_b200 import ops

    seg = torch.arange(16, device="cuda").reshape(1, 4, 4)
    trav = torch.arange(16, device="cuda", dtype=torch.float32)[None].clone()
    tm, _ = ops.segment_maps(seg, torch.tensor([5], device="cuda", dtype=torch.int32), trav)
    assert torch.equal(tm.reshape(-1)[:5], trav[0, :5]) and torch.isnan(tm.reshape(-1)[5:]).all()


# ------------------------------------------------------------------------------------------------ padded rows
def _padded_frames(D, n_rows, S, seed):
    g = torch.Generator().manual_seed(seed)
    feat = torch.full((len(n_rows), S, D), float("nan"))      # padding rows hold NaN: any read of them shows
    for b, n in enumerate(n_rows):
        feat[b, :n] = torch.randn(n, D, generator=g) * 0.5
    return feat.cuda(), torch.tensor(n_rows, dtype=torch.int32).cuda()


def _frame_edges(n, seed, E=64):
    g = torch.Generator().manual_seed(seed)
    if n < 2:
        return torch.zeros(0, 2, dtype=torch.long)
    src = torch.randint(0, n, (E,), generator=g)
    dst = torch.randint(0, n, (E,), generator=g)
    keep = src != dst
    return torch.stack((src[keep], dst[keep]), 1)


def _learner(kind, D):
    from wild_visual_navigation_b200 import DoubleMLP, LinearRnvp, SimpleGCN, SimpleMLP

    torch.manual_seed(42)
    if kind == "SimpleMLP":
        return SimpleMLP(D, [256, 32, 1], True).cuda()
    if kind == "DoubleMLP":
        return DoubleMLP(D, [64, 32, 1]).cuda()
    if kind == "SimpleGCN":
        return SimpleGCN(D, True, [64, 32, 1]).cuda()
    return LinearRnvp(D, [200], mask_type="odds", conditioning_size=0, use_permutation=True,
                      single_function=False).cuda()


@pytest.mark.parametrize("kind", ["SimpleMLP", "DoubleMLP", "LinearRnvp", "SimpleGCN"])
def test_padded_rows_equal_predict_segments(kind):
    from wild_visual_navigation_b200 import ConfidenceGenerator, Data, TraversabilityInference

    D, S, n_rows = 96, 30, [30, 0, 7, 19]
    feat, n = _padded_frames(D, n_rows, S, seed=5)
    m = _learner(kind, D)
    cg = ConfidenceGenerator(0.5, "latest_measurement").cuda()
    ti = TraversabilityInference(None, m, cg, max_rows=len(n_rows) * S)
    live = torch.cat([feat[b, :k] for b, k in enumerate(n_rows)])
    with torch.no_grad():   # a generator state that puts the rows inside its interval
        if kind == "LinearRnvp":
            r = ti._flow_infer.rows(m, live)
            v = -(r["logprob"].sum(1) + r["log_det"])
        elif kind == "SimpleGCN":
            v = None   # the GCN's rows depend on the graph; the generator keeps its default state
        else:
            v = ((m.forward(Data(x=live))[:, 1:] - live) ** 2).mean(1)
        if v is not None:
            cg.mean[0], cg.std[0] = v.mean() - 0.5 * v.std(), v.std()
    edges, n_edges = None, None
    frame_edges = [_frame_edges(k, 10 + b) for b, k in enumerate(n_rows)]
    if kind == "SimpleGCN":
        E = max(e.shape[0] for e in frame_edges)
        edges = torch.zeros(len(n_rows), E, 2, dtype=torch.long)
        for b, e in enumerate(frame_edges):
            edges[b, : e.shape[0]] = e
        edges = edges.cuda()
        n_edges = torch.tensor([e.shape[0] for e in frame_edges], dtype=torch.int32).cuda()
    trav, conf = ti.predict_rows(feat, n, edges, n_edges)
    assert trav.shape == (len(n_rows), S)
    assert (conf is None) == (kind == "LinearRnvp")
    tol_t, tol_c = {"SimpleMLP": (0, 0), "DoubleMLP": (0, 0), "LinearRnvp": (1e-3, 0), "SimpleGCN": (1e-5, 1e-4)}[kind]
    for b, k in enumerate(n_rows):
        assert torch.isnan(trav[b, k:]).all() and (conf is None or torch.isnan(conf[b, k:]).all())
        if k == 0:
            continue
        seg = torch.arange(k, device="cuda")
        ref_t, ref_c = ti.predict_segments(feat[b, :k], seg, edges=frame_edges[b].T.contiguous().cuda())
        dt = (trav[b, :k] - ref_t).abs().max().item()
        dc = 0.0 if conf is None else (conf[b, :k] - ref_c).abs().max().item()
        print(f"{kind} frame {b} ({k} rows): |padded - predict_segments| trav {dt:.2e} conf {dc:.2e}")
        if tol_t == 0:
            assert torch.equal(trav[b, :k], ref_t) and torch.equal(conf[b, :k], ref_c)
        assert dt <= tol_t and dc <= tol_c
        assert torch.isfinite(trav[b, :k]).all()
    # predict_frames paints the same rows
    seg = torch.randint(0, S, (len(n_rows), 16, 16), device="cuda")
    tm, cm = ti.predict_frames(feat, n, edges, n_edges, seg)
    assert _identical(tm, _gather_ref(seg, n, trav))
    if conf is not None:
        assert _identical(cm, _gather_ref(seg, n, conf))


def test_per_pixel_calls_refuse_a_pyramid():
    from wild_visual_navigation_b200 import ConfidenceGenerator, SimpleMLP, TraversabilityInference
    from wild_visual_navigation_b200.feature_extractor import TorchVisionInterface
    from wild_visual_navigation_b200.feature_extractor import weights as W

    tv = TorchVisionInterface("cuda", "resnet18", 224, state_dict=W.synthetic_resnet_state_dict(18, seed=1), max_batch=1)
    ti = TraversabilityInference(tv, SimpleMLP(960, [256, 32, 1], True).cuda(),
                                 ConfidenceGenerator(0.5, "latest_measurement").cuda())
    with pytest.raises(ValueError, match="predict_frames"):
        ti.predict(torch.rand(1, 3, 224, 224, device="cuda"))
    with pytest.raises(ValueError, match="predict_frames"):
        ti.predict_from_tokens(torch.zeros(1, 49, 960, device="cuda"), 224)


# ------------------------------------------------------------------------------------------------ HotPathStep
@pytest.fixture(scope="module")
def weights():
    import bench

    _, sd, hd = bench.make_weights()
    return sd, hd


@pytest.fixture(scope="module")
def trunks():
    from wild_visual_navigation_b200.feature_extractor import weights as W

    return {"resnet18": W.synthetic_resnet_state_dict(18, seed=1), "resnet50": W.synthetic_resnet_state_dict(50, seed=1),
            "efficientnet_b0": W.synthetic_efficientnet_b0_state_dict(seed=1)}


def _hot_path(weights, model="SimpleMLP", anomaly=False, **kw):
    from wild_visual_navigation_b200 import HotPathStep

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return HotPathStep("cuda", weights[0], weights[1], batch=3, input_size=224, chunk=32, flip_tta=False,
                           run_clustering=True, n_image_clusters=20, model=model, anomaly_detection=anomaly, **kw)


def _img(seed):
    return torch.rand(3, 3, 224, 224, generator=torch.Generator().manual_seed(seed)).cuda()


def _labels(hp, seed):
    g = torch.Generator().manual_seed(seed)
    n = 3 * hp.smax
    yv = torch.rand(n, generator=g) < 0.3
    yv[:2] = True
    return torch.where(yv, torch.rand(n, generator=g).clamp(min=0.001), torch.zeros(n)).cuda(), yv.cuda()


def _composed(hp, r, y, yv):
    """The same work by hand on r's pooled rows: per frame predict_segments painted through seg, then train_on_padded."""
    travs, confs = [], []
    for b in range(r["seg"].shape[0]):
        k = int(r["n_segments"][b])
        edges = r["edges"][b, : int(r["n_edges"][b])].T.contiguous() if hp.gcn else None
        t, c = hp.ti.predict_segments(r["feat"][b, :k], r["seg"][b], edges=edges)
        travs.append(t)
        confs.append(c)
    crow = hp.te.train_on_padded(r["feat"], r["n_segments"], y, yv, edges=r["edges"], n_edges=r["n_edges"])
    hp.ti.refresh_weights()
    return torch.stack(travs), (None if confs[0] is None else torch.stack(confs)), crow


def _check_against_composed(a, b, img, y, yv, exact):
    ra = a.step(img, y, yv)
    # b does the same work on a's rows (segment pooling adds with float atomics: two extractions may differ in the
    # last bits, so the reference reads the step's own rows)
    tb, cb, crow = _composed(b, ra, y, yv)
    assert ra["trav"].shape == ra["seg"].shape and torch.isfinite(ra["trav"]).all()
    assert (ra["conf"] is None) == (cb is None)
    dt = (ra["trav"] - tb).abs().max().item()
    dc = 0.0 if cb is None else (ra["conf"] - cb).abs().max().item()
    print(f"step vs composed: |d| trav {dt:.2e} conf {dc:.2e}")
    if exact:
        assert torch.equal(ra["trav"], tb) and torch.equal(ra["conf"], cb)
    else:
        assert dt <= 1e-3 and dc <= 1e-4
    n = int(ra["n_segments"].sum())
    if a.te._anomaly_detection:   # the flow's confidence rows are the labelled rows'
        n = int(yv[:n].sum())
    assert torch.isfinite(ra["confidence_rows"][:n]).all()
    assert (ra["confidence_rows"][:n] - crow[:n]).abs().max().item() <= 1e-4
    return ra


LEARNERS = [("SimpleMLP", False), ("DoubleMLP", False), ("SimpleGCN", False), ("SimpleMLP", True)]


@pytest.mark.parametrize("model,anomaly", LEARNERS)
def test_segment_wise_step_equals_composed_work(weights, model, anomaly):
    a = _hot_path(weights, model, anomaly, prediction_per_pixel=False)
    b = _hot_path(weights, model, anomaly, prediction_per_pixel=False)
    y, yv = _labels(a, 3)
    p0 = a.te._model.flat_params.clone()
    _check_against_composed(a, b, _img(1), y, yv, exact=model in ("SimpleMLP", "DoubleMLP") and not anomaly)
    assert not torch.equal(a.te._model.flat_params, p0)   # the step trained


def _check_replay(a, b, y, yv):
    img0, img1 = _img(7), _img(8)
    a.capture(img0, y, yv, warmup=2)
    for _ in range(2):
        b.step(img0, y, yv)
    ra = a.replay(img1)
    rb = b.step(img1, y, yv)
    torch.cuda.synchronize()
    assert torch.isfinite(ra["trav"]).all()
    dt = (ra["trav"] - rb["trav"]).abs().max().item()
    dc = 0.0 if rb["conf"] is None else (ra["conf"] - rb["conf"]).abs().max().item()
    print(f"replay vs eager: |d| trav {dt:.2e} conf {dc:.2e}")
    # segment pooling adds with float atomics, so the two paths' rows may differ in the last bits
    assert dt <= 2e-3 and dc <= 2e-3
    # the graph's Adam steps advanced the device-side step counter as the eager steps did
    assert torch.equal(a.te._trainer.step_counter, b.te._trainer.step_counter) and int(b.te._trainer.step_counter) == 3


@pytest.mark.parametrize("model,anomaly", LEARNERS)
def test_segment_wise_capture_replay_equals_eager(weights, model, anomaly):
    a = _hot_path(weights, model, anomaly, prediction_per_pixel=False)
    b = _hot_path(weights, model, anomaly, prediction_per_pixel=False)
    y, yv = _labels(a, 9)
    _check_replay(a, b, y, yv)


TORCHVISION = [("resnet18", "stego", "SimpleMLP", False), ("resnet18", "slic", "SimpleMLP", False),
               ("resnet18", "grid", "SimpleMLP", False), ("resnet18", "stego", "SimpleGCN", False),
               ("resnet18", "slic", "SimpleGCN", False), ("resnet18", "grid", "SimpleGCN", False),
               ("resnet50", "stego", "SimpleMLP", True), ("efficientnet_b0", "stego", "SimpleMLP", True)]


def _tv_hot_path(weights, trunks, model_type, seg_type, model, anomaly):
    return _hot_path(weights, model, anomaly, feature_type="torchvision", model_type=model_type,
                     backbone_state_dict=trunks[model_type], segmentation_type=seg_type, prediction_per_pixel=False)


@pytest.mark.parametrize("model_type,seg_type,model,anomaly", TORCHVISION)
def test_torchvision_step_equals_composed_work(weights, trunks, model_type, seg_type, model, anomaly):
    a = _tv_hot_path(weights, trunks, model_type, seg_type, model, anomaly)
    b = _tv_hot_path(weights, trunks, model_type, seg_type, model, anomaly)
    assert a.fe.feature_dim == {"resnet18": 960, "resnet50": 2944, "efficientnet_b0": 2432}[model_type]
    y, yv = _labels(a, 4)
    ra = _check_against_composed(a, b, _img(2), y, yv, exact=model == "SimpleMLP" and not anomaly)
    assert ra["tokens"] is None and ra["feat"].shape[1:] == (a.smax, a.fe.feature_dim)


@pytest.mark.parametrize("model_type,seg_type,model,anomaly", [TORCHVISION[1], TORCHVISION[5], TORCHVISION[7]])
def test_torchvision_capture_replay_equals_eager(weights, trunks, model_type, seg_type, model, anomaly):
    a = _tv_hot_path(weights, trunks, model_type, seg_type, model, anomaly)
    b = _tv_hot_path(weights, trunks, model_type, seg_type, model, anomaly)
    y, yv = _labels(a, 9)
    _check_replay(a, b, y, yv)


def test_argument_checks(weights, trunks):
    from wild_visual_navigation_b200 import _C

    with pytest.raises(ValueError, match="per-pixel head"):
        _hot_path(weights, feature_type="torchvision", model_type="resnet18", backbone_state_dict=trunks["resnet18"])
    with pytest.raises(ValueError, match="segmentation_type"):
        _hot_path(weights, segmentation_type="random")
    with pytest.raises(ValueError, match="model_type"):
        _hot_path(weights, feature_type="torchvision", prediction_per_pixel=False)
    with pytest.raises(_C.WvnError, match="dim <= 1024"):
        _tv_hot_path(weights, trunks, "resnet50", "grid", "SimpleMLP", False)
