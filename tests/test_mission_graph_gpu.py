"""GPU checks of the device mission graph: ``wvn_mission_propagate`` against the composition of this library's existing
kernels (``ImageProjector.update_supervision_masks``'s fused render + fmin, then ``pool_supervision``) on the same slots,
and the whole scripted trajectory of oracle/mission_graph.py through ``TraversabilityEstimator`` against the golden the
reference's own graphs.py / nodes.py / add_supervision_node wrote.

Bars.  Kernel vs composition: masks bit-identical (the same rasteriser, shared device code), y_valid identical and y
within 1e-6 relative (stored masks hold multiples of 1/16, as labels do, so the float sums are exact in any order), and
slots outside the list untouched bit for bit.  Trajectory vs golden: the same frames added, the same propagating
events, the same sampled node timestamps in every train(), identical y_valid and y within 1e-6 relative except where a
pixel next to a footprint edge falls on the other side (the projection differs from the CPU reference in the last bits,
see tests/test_footprint_gpu.py): such a segment's label moves by at most a few pixels' share of its mean (5e-3 absolute
here), and at most 1 % of the compared labels may do so.  Training from the graph is checked against
``train_on_padded`` on a batch the test assembles itself from the scenario's features and the sampled nodes' labels:
the loss metrics to 1e-4 relative (a wrong or missing row moves them far more) and the parameters to 5e-3 absolute
(Adam's first steps move each parameter by about lr = 1e-3 whatever the gradient's size).
"""
import os
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu


def _slots_case(n, H, smax, seed):
    from oracle import image_projector as oip

    g = torch.Generator().manual_seed(seed)
    cap = n + 5
    start = cap - 2 if n > 1 else 3                     # the list wraps around the end of the ring
    slots = [(start + k) % cap for k in range(n)]
    K, poses, fp = oip.synthetic_footprints(cap, seed=seed, image=H)
    seg = torch.randint(-2, smax + 3, (cap, H, H), generator=g, dtype=torch.int32)
    if smax > 8:
        seg[seg % 7 == 3] = 5                           # segment ids that never occur: empty segments
    mask = torch.randint(0, 17, (cap, H, H), generator=g).float() / 16
    mask[torch.rand(cap, H, H, generator=g) < 0.5] = float("nan")
    restart = torch.tensor([k % 3 == 1 for k in range(n)], dtype=torch.uint8)
    return cap, slots, K, poses, fp[0].contiguous(), seg, mask, restart


@pytest.mark.parametrize("n,H,smax", [(1, 224, 1), (2, 448, 4096), (37, 224, 4096), (37, 448, 1), (256, 224, 64),
                                      (256, 448, 4096)])
def test_propagate_equals_render_then_pool(n, H, smax):
    from wild_visual_navigation_b200 import ops

    cap, slots, K, poses, fp, seg, mask, restart = _slots_case(n, H, smax, seed=n + H)
    dev = "cuda"
    trav = torch.tensor([11 / 16], device=dev)
    y = torch.full((cap, smax), float("nan"), device=dev)
    yv = torch.full((cap, smax), 0xAB, dtype=torch.uint8, device=dev)
    sv = torch.full((cap,), -7, dtype=torch.int32, device=dev)
    m = mask.to(dev)
    y0, yv0, sv0, m0 = y.clone(), yv.clone(), sv.clone(), m.clone()
    st = torch.tensor(slots, dtype=torch.int32, device=dev)
    ws = ops.mission_propagate_workspace(n, smax, dev)
    ops.mission_propagate(st, restart.to(dev), K.to(dev), poses.to(dev), fp.to(dev), trav, seg.to(dev), m, y, yv, sv, ws)

    # the composition on the same slots: restarted slots from zeros, three identical channels
    sl = torch.tensor(slots)
    sup = mask[sl].clone()
    sup[restart.bool()] = 0.0
    sup = sup[:, None].expand(n, 3, H, H).contiguous().to(dev)
    ops.project_and_render(K[sl].to(dev), poses[sl].to(dev), fp[None].expand(n, -1, -1).contiguous().to(dev),
                           torch.ones(3, device=dev), H, H, render=False, supervision=sup, traversability=trav)
    want_y, want_v = ops.pool_supervision(seg[sl].long().to(dev), sup, smax)
    torch.cuda.synchronize()
    assert torch.equal(m[st.long()].view(torch.int32), sup[:, 0].view(torch.int32))
    assert torch.equal(yv[st.long()].bool(), want_v)
    assert torch.allclose(y[st.long()], want_y, rtol=1e-6, atol=0)
    assert torch.equal(sv[st.long()], want_v.any(1).int())
    assert smax == 1 or ((~want_v).any() and (want_y[~want_v] == 0).all())
    other = torch.tensor([s for s in range(cap) if s not in slots], dtype=torch.long, device=dev)
    for a, b in ((m, m0), (y, y0), (yv, yv0), (sv, sv0)):
        assert torch.equal(a[other].view(torch.uint8), b[other].view(torch.uint8))
    assert int(ws.count_nonzero()) == 0                  # the workspace is left zero for the next call
    # a second event on the same workspace is the composition again
    ops.mission_propagate(st, None, K.to(dev), poses.to(dev), fp.to(dev), trav * 0.5, seg.to(dev), m, y, yv, sv, ws)
    ops.project_and_render(K[sl].to(dev), poses[sl].to(dev), fp[None].expand(n, -1, -1).contiguous().to(dev),
                           torch.ones(3, device=dev), H, H, render=False, supervision=sup, traversability=trav * 0.5)
    want_y, want_v = ops.pool_supervision(seg[sl].long().to(dev), sup, smax)
    assert torch.equal(m[st.long()].view(torch.int32), sup[:, 0].view(torch.int32))
    assert torch.equal(yv[st.long()].bool(), want_v) and torch.allclose(y[st.long()], want_y, rtol=1e-6, atol=0)


def _params(learner, D):
    from wild_visual_navigation_b200.traversability_estimator import default_params

    p = default_params(learner == "LinearRnvp")
    p["model"]["name"] = learner
    for k in ("simple_mlp_cfg", "double_mlp_cfg", "linear_rnvp_cfg"):
        p["model"][k]["input_size"] = D
    return p


def _estimator(learner, g, D):
    from wild_visual_navigation_b200 import TraversabilityEstimator

    p = g["params"]
    return TraversabilityEstimator(_params(learner, D), device="cuda", max_distance=p["max_distance"],
                                   image_distance_thr=p["image_distance_thr"],
                                   supervision_distance_thr=p["supervision_distance_thr"],
                                   min_samples_for_training=p["min_samples"], anomaly_detection=learner == "LinearRnvp",
                                   mission_graph_capacity=64, mission_graph_smax=64)


def _flat(te):
    return torch.cat([q.detach().flatten() for q in te._model.parameters()])


@pytest.mark.parametrize("learner", ["SimpleMLP", "DoubleMLP", "LinearRnvp"])
def test_trajectory_matches_reference_golden(golden_dir, learner):
    from oracle import mission_graph as omg
    from wild_visual_navigation_b200.traversability_estimator.mission_graph import SupervisionNode

    g = torch.load(os.path.join(golden_dir, "mission_graph.pt"), weights_only=False)
    D, H = 32, g["H"]
    te, twin = _estimator(learner, g, D), _estimator(learner, g, D)
    feats = {}
    added, events, samples = [], [], []
    n_mission = n_lab = n_far = 0
    trains = 0
    for ev in omg.scenario(H=H, D=D):
        if ev[0] == "mission":
            n = ev[1]
            if n_mission % 2:   # half the frames as extract_batch results, half as node objects
                feat = torch.zeros(1, 64, D)
                feat[0, : n["features"].shape[0]] = n["features"]
                r = {"seg": n["seg"][None].cuda(), "feat": feat.cuda(),
                     "n_segments": torch.tensor([n["features"].shape[0]], dtype=torch.int32).cuda()}
                ok = te.add_mission_frames(r, n["pose_base_in_world"][None], n["K"], [n["timestamp"]],
                                           pose_cam_in_base=omg.camera_in_base()) == 1
            else:
                node = SimpleNamespace(features=n["features"].cuda(), feature_segments=n["seg"].cuda(),
                                       pose_cam_in_world=n["pose_cam_in_world"], pose_base_in_world=n["pose_base_in_world"],
                                       K=n["K"], timestamp=n["timestamp"])
                ok = te.add_mission_node(node)
            n_mission += 1
            added.append((n["timestamp"], bool(ok)))
            feats[n["timestamp"]] = n["features"]
        elif ev[0] == "supervision":
            p = ev[1]
            gr = te._mission_graph
            in_range = [nd.timestamp for nd in gr.get_nodes_within_radius_range()] if gr is not None else []
            pn = SupervisionNode(timestamp=p["timestamp"], pose_base_in_world=p["pose_base_in_world"],
                                 pose_footprint_in_world=p["pose_footprint_in_world"], width=p["width"],
                                 supervision=torch.ones(1), traversability=p["traversability"].clone())
            ok = te.add_supervision_node(pn)
            want = g["events"][len(events)]
            assert ok == want["propagated"], p["timestamp"]
            if ok:
                assert in_range == want["in_range"], p["timestamp"]
                by_t = {nd.timestamp: nd for nd in gr.get_nodes()}
                for t, (wy, wyv) in omg.golden_labels(g, want).items():
                    S = wy.shape[0]
                    gy = gr.y[by_t[t].slot, :S].cpu()
                    gyv = gr.y_valid[by_t[t].slot, :S].cpu().bool()
                    assert torch.equal(gyv, wyv), (p["timestamp"], t)
                    d = (gy - wy).abs()
                    n_lab += S
                    n_far += int((d > 1e-6 * wy.abs()).sum())
                    assert d.max() <= 5e-3, (p["timestamp"], t, d.max().item())
            events.append(ok)
        else:
            out = te.train()
            want = g["samples"][len(samples)]
            got = [nd.timestamp for nd in te.last_sampled_nodes] if out.get("loss_total", -1) != -1 else None
            samples.append(got)
            assert got == want
            if got is None:
                continue
            trains += 1
            # the same step on a batch assembled here: the scenario's features, the sampled nodes' labels
            gr = te._mission_graph
            by_t = {nd.timestamp: nd for nd in gr.get_nodes()}
            S = [feats[t].shape[0] for t in got]
            feat = torch.zeros(len(got), gr.smax, D)
            for i, t in enumerate(got):
                feat[i, : S[i]] = feats[t]
            y = torch.cat([gr.y[by_t[t].slot, : S[i]] for i, t in enumerate(got)])
            yv = torch.cat([gr.y_valid[by_t[t].slot, : S[i]] for i, t in enumerate(got)])
            twin.train_on_padded(feat.cuda(), torch.tensor(S, dtype=torch.int32).cuda(), y, yv)
            # the SimpleMLP step sums its weight gradients with split-K atomics, so two runs agree to rounding only
            mt, mw = te._trainer.metrics[:3], twin._trainer.metrics[:3]
            assert torch.allclose(mt, mw, rtol=1e-4, atol=1e-6), (trains, mt.tolist(), mw.tolist())
            assert torch.allclose(_flat(te), _flat(twin), rtol=0, atol=5e-3), f"train() {trains} differs"
            if learner != "SimpleMLP" and trains >= 3:
                break
    assert learner != "SimpleMLP" or (added == g["added"] and samples == g["samples"])
    assert n_far <= 0.01 * max(n_lab, 1), f"{n_far} of {n_lab} labels beyond 1e-6 relative"
    print(f"{learner}: {trains} train steps, {n_far} of {n_lab} labels off by an edge pixel")


def test_add_supervision_node_does_not_synchronise(golden_dir):
    from oracle import mission_graph as omg
    from wild_visual_navigation_b200.traversability_estimator.mission_graph import SupervisionNode

    g = torch.load(os.path.join(golden_dir, "mission_graph.pt"), weights_only=False)
    te = _estimator("SimpleMLP", g, 32)
    n_prop = 0
    for ev in omg.scenario(H=g["H"], D=32)[:80]:
        if ev[0] == "mission":
            n = ev[1]
            te.add_mission_node(SimpleNamespace(features=n["features"].cuda(), feature_segments=n["seg"].cuda(),
                                                pose_cam_in_world=n["pose_cam_in_world"],
                                                pose_base_in_world=n["pose_base_in_world"], K=n["K"],
                                                timestamp=n["timestamp"]))
        elif ev[0] == "supervision":
            p = ev[1]
            pn = SupervisionNode(timestamp=p["timestamp"], pose_base_in_world=p["pose_base_in_world"],
                                 pose_footprint_in_world=p["pose_footprint_in_world"], width=p["width"],
                                 supervision=torch.ones(1), traversability=p["traversability"].clone())
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                n_prop += int(te.add_supervision_node(pn))
            finally:
                torch.cuda.set_sync_debug_mode("default")
    assert n_prop > 5
