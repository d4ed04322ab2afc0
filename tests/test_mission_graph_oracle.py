"""CPU checks of the mission graph's data path: the oracle (oracle/mission_graph.py) against the golden that the
reference's own graphs.py / nodes.py / add_supervision_node wrote (tests/golden/make_golden_mission_graph.py), the
library's host-side graph logic against the oracle, and the new C ABI entry.

The scripted trajectory covers refused mission frames, refused (too close) supervision nodes that lower the last
node's traversability, the 30 s sweep that restarts in-range nodes from zero masks, and train()'s sampling."""
import os
import random

import pytest
import torch

from oracle import mission_graph as omg


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "mission_graph.pt"), weights_only=False)


def _run_oracle(g, capacity=None):
    p = g["params"]
    o = omg.MissionGraphOracle(g["H"], g["H"], p["image_distance_thr"], p["supervision_distance_thr"], p["max_distance"],
                               capacity=capacity)
    random.seed(42)
    out = {"added": [], "events": [], "samples": []}
    for ev in omg.scenario(H=g["H"]):
        if ev[0] == "mission":
            out["added"].append((ev[1]["timestamp"], o.add_mission_node(ev[1])))
        elif ev[0] == "supervision":
            ts = o.add_supervision_node(dict(ev[1], traversability=ev[1]["traversability"].clone()))
            labels = {}
            if ts:
                labels = {nd["timestamp"]: (nd["y"], nd["y_valid"]) for nd in o.nodes if nd["timestamp"] in ts}
            out["events"].append({"timestamp": ev[1]["timestamp"], "propagated": ts is not None, "in_range": ts or [],
                                  "labels": labels})
        else:
            out["samples"].append([nd["timestamp"] for nd in o.sample(p["batch_size"])]
                                  if len(o.valid_nodes()) > p["min_samples"] else None)
    return o, out


def test_oracle_reproduces_reference_golden(golden):
    _, out = _run_oracle(golden)
    assert out["added"] == golden["added"]
    assert len(out["events"]) == len(golden["events"])
    n_wiped = 0
    for got, want in zip(out["events"], golden["events"]):
        assert got["propagated"] == want["propagated"] and got["in_range"] == want["in_range"], want["timestamp"]
        for t, (y, yv) in omg.golden_labels(golden, want).items():
            gy, gyv = got["labels"][t]
            assert torch.equal(gyv, yv)
            assert torch.allclose(gy, y, rtol=1e-6, atol=0), (want["timestamp"], t)
            n_wiped += int(not yv.any())
    assert out["samples"] == golden["samples"]
    assert n_wiped > 0                                          # the 30 s sweep restarted in-range nodes from zeros
    assert sum(not a for _, a in golden["added"]) == 4          # the edge gate refused the repeated frames


def test_ring_wraps_without_changing_labels(golden):
    """A ring of 24 nodes (the in-range window is ~20) gives the same nodes, in-range sets and labels."""
    _, out = _run_oracle(golden, capacity=24)
    assert out["added"] == golden["added"]
    for got, want in zip(out["events"], golden["events"]):
        assert got["in_range"] == want["in_range"]
        for t, (y, yv) in omg.golden_labels(golden, want).items():
            assert torch.equal(got["labels"][t][1], yv) and torch.allclose(got["labels"][t][0], y, rtol=1e-6, atol=0)


def test_library_graph_logic_matches_oracle(golden):
    """The library's float64 host math (SE(3) distance, footprint, range query) against the oracle's float32."""
    from wild_visual_navigation_b200.traversability_estimator import mission_graph as mg

    ev = [e[1] for e in omg.scenario(H=golden["H"]) if e[0] == "mission"]
    for a, b in zip(ev[:-1], ev[1:]):
        assert abs(mg.pose_distance(b["pose_base_in_world"], a["pose_base_in_world"])
                   - float(omg.distance(b["pose_base_in_world"], a["pose_base_in_world"]))) < 1e-5
    sup = [e[1] for e in omg.scenario(H=golden["H"]) if e[0] == "supervision"]
    p, q = sup[5], sup[3]
    want = omg.footprint(p, q)
    got = mg.footprint_between(mg.SupervisionNode(pose_footprint_in_world=p["pose_footprint_in_world"], width=0.6),
                               mg.SupervisionNode(pose_footprint_in_world=q["pose_footprint_in_world"], width=0.6))
    assert torch.equal(got, want)
    ts = [0.0, 1.25, 2.5, 3.75, 4.4]
    # 4.4 is within 1 s of 3.75, so node 3 is the query node: the last node then receives labels
    assert mg.range_query(ts, [1.0, 1.0, 1.0, 0.5], 2.0) == (3, [1, 2, 4])
    assert mg.range_query(ts, [1.0, 1.0, 1.0, 2.5], 2.0) == (3, [1, 2])   # the later side is farther than 2
    assert mg.range_query(ts[:4], [1.0, 1.0, 1.0], 2.0) == (3, [1, 2])


def test_abi_version_and_mission_propagate_exports():
    import __graft_entry__ as g

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.exists(os.path.join(root, "wild_visual_navigation_b200", "libwvn_b200.so")):
        g.build()
    from wild_visual_navigation_b200 import _C

    l = _C.lib()
    assert l.wvn_version() == 108
    assert hasattr(l, "wvn_mission_propagate") and hasattr(l, "wvn_mission_propagate_workspace_bytes")
    assert l.wvn_mission_propagate_workspace_bytes(3, 10) == 3 * (2 * 10 * 4 + 4)
