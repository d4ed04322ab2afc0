"""Writes tests/golden/mission_graph.pt by running the reference's OWN graphs.py / nodes.py and its
``TraversabilityEstimator.add_mission_node`` / ``add_supervision_node`` (traversability_estimator.py:166-300) on the
scripted trajectory of oracle/mission_graph.py.scenario(), plus train()'s sampling (:458-463, graphs.py:137-143) under
``random.seed(42)``.

    WVN_REFERENCE_ROOT=<reference checkout> python tests/golden/make_golden_mission_graph.py

The estimator module itself cannot be imported here (pytorch_lightning, pytictac, ...), so the two methods' source is
read with ``ast`` and compiled against a bare namespace (nothing is copied into this repository).  liegroups and kornia
are absent: ``SE3.from_matrix(...).log()`` comes from oracle/mission_graph.py's restatement and the kornia routines from
oracle/image_projector.py, through stub modules, as make_golden.py does for the image projector; networkx is the real
one.  Recorded: which mission frames were added, the in-range node timestamps of every supervision event, the labels
(y, y_valid) of those nodes after the event, and the sampled node timestamps of every train() that passed its gate.
The labels are packed into one float32 ``y`` and one bool ``y_valid`` tensor; each event's ``labels`` maps a node's
timestamp to its (offset, length) there (oracle/mission_graph.py ``golden_labels`` unpacks them).
"""
import ast
import importlib.util
import os
import random
import sys
import textwrap
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import image_projector as oip  # noqa: E402
from oracle import mission_graph as omg  # noqa: E402
from oracle import ref_import  # noqa: E402

H = 224
# max_distance 2.9 m: 19 edges of 0.15 m lie inside and 20 outside by 0.1 m, so float32 and float64 path sums agree
PARAMS = dict(image_distance_thr=0.1, supervision_distance_thr=0.05, max_distance=2.9, min_samples=3, batch_size=8)


def _mod(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def _load(name, rel, package=None):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ref_import.REF_ROOT, rel))
    mod = importlib.util.module_from_spec(spec)
    if package:
        mod.__package__ = package
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def _method(rel, name, scope):
    path = os.path.join(ref_import.REF_ROOT, rel)
    src = open(path).read()
    fn = next(n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == name)
    exec(compile(textwrap.dedent("\n".join(src.splitlines()[fn.lineno - 1 : fn.end_lineno])), path, "exec"), scope)
    return scope[name]


class _PinholeCamera:
    def __init__(self, intrinsics, extrinsics, height, width):
        self.intrinsics, self.extrinsics, self.height, self.width = intrinsics, extrinsics, height, width

    batch_size = property(lambda self: self.intrinsics.shape[0])
    camera_matrix = property(lambda self: self.intrinsics[..., :3, :3])

    def project(self, point_3d):
        return oip.convert_points_from_homogeneous(oip.transform_points(self.intrinsics @ self.extrinsics, point_3d))


class _SE3:
    def __init__(self, mat):
        self.mat = mat

    @classmethod
    def from_matrix(cls, mat, normalize=False):
        return cls(mat)

    def log(self):
        return omg.se3_log(self.mat)


def load_reference():
    _mod("pytictac", Timer=object, accumulate_time=lambda f: f)
    for n in ("kornia", "kornia.geometry", "kornia.geometry.camera", "kornia.utils", "liegroups"):
        _mod(n)
    _mod("kornia.geometry.camera.pinhole", PinholeCamera=_PinholeCamera)
    _mod("kornia.geometry.linalg", transform_points=oip.transform_points)
    _mod("kornia.utils.draw", draw_convex_polygon=oip.draw_convex_polygon)
    _mod("liegroups.torch", SE3=_SE3, SO3=object)
    root = _mod("wild_visual_navigation")
    root.__path__ = []
    ip = _load("ref_image_projector", "wild_visual_navigation/image_projector/image_projector.py")
    _mod("wild_visual_navigation.image_projector", ImageProjector=ip.ImageProjector)
    meshes = _load("ref_meshes", "wild_visual_navigation/utils/meshes.py")
    data = _load("ref_data", "wild_visual_navigation/utils/data.py")
    _mod("wild_visual_navigation.utils", make_box=meshes.make_box, make_plane=meshes.make_plane,
         make_polygon_from_points=meshes.make_polygon_from_points, make_dense_plane=meshes.make_dense_plane,
         Data=data.Data)
    te = _mod("wild_visual_navigation.traversability_estimator")
    te.__path__ = []
    nodes = _load("wild_visual_navigation.traversability_estimator.nodes",
                  "wild_visual_navigation/traversability_estimator/nodes.py", "wild_visual_navigation.traversability_estimator")
    graphs = _load("wild_visual_navigation.traversability_estimator.graphs",
                   "wild_visual_navigation/traversability_estimator/graphs.py", "wild_visual_navigation.traversability_estimator")
    return ip, nodes, graphs


def main():
    assert ref_import.available(), "set WVN_REFERENCE_ROOT to a checkout of the reference"
    ip, nodes, graphs = load_reference()
    WVNMode = types.SimpleNamespace(EXTRACT_LABELS="extract_labels", ONLINE="online")
    scope = {"torch": torch, "ImageProjector": ip.ImageProjector, "WVNMode": WVNMode, "os": os,
             "MissionNode": nodes.MissionNode, "SupervisionNode": nodes.SupervisionNode}
    te_rel = "wild_visual_navigation/traversability_estimator/traversability_estimator.py"
    add_mission_node = _method(te_rel, "add_mission_node", scope)
    add_supervision_node = _method(te_rel, "add_supervision_node", scope)

    est = types.SimpleNamespace(
        _pause_mission_graph=False, _pause_supervision_graph=False, _device="cpu", _mode=WVNMode.ONLINE,
        _debug_info_node_count=0,
        _supervision_graph=graphs.DistanceWindowGraph(max_distance=PARAMS["max_distance"],
                                                      edge_distance=PARAMS["supervision_distance_thr"]),
        _mission_graph=graphs.BaseGraph(edge_distance=PARAMS["image_distance_thr"]))
    in_range = []
    orig = est._mission_graph.get_nodes_within_radius_range

    def recording(*a, **k):
        out = orig(*a, **k)
        in_range.append(out)
        return out

    est._mission_graph.get_nodes_within_radius_range = recording

    random.seed(42)
    rec = {"params": PARAMS, "H": H, "added": [], "events": [], "samples": []}
    ys, yvs, n_packed = [], [], 0
    for ev in omg.scenario(H=H):
        kind = ev[0]
        if kind == "mission":
            n = ev[1]
            node = nodes.MissionNode(timestamp=n["timestamp"], pose_base_in_world=n["pose_base_in_world"],
                                     pose_cam_in_world=n["pose_cam_in_world"],
                                     image_projector=ip.ImageProjector(n["K"][None], torch.tensor(H), torch.tensor(H)))
            node.features, node.feature_segments = n["features"], n["seg"]
            ok = add_mission_node(est, node)
            rec["added"].append((n["timestamp"], bool(ok)))
        elif kind == "supervision":
            p = ev[1]
            pn = nodes.SupervisionNode(timestamp=p["timestamp"], pose_base_in_world=p["pose_base_in_world"],
                                       pose_footprint_in_world=p["pose_footprint_in_world"], width=p["width"],
                                       supervision=torch.ones(1), traversability=p["traversability"].clone())
            before = len(in_range)
            ok = bool(add_supervision_node(est, pn))
            got = in_range[before] if len(in_range) > before else []
            labels = {}
            for m in got if ok else []:   # packed: one float32 and one bool tensor for all labels, offsets per node
                labels[m.timestamp] = (n_packed, m.supervision_signal.numel())
                ys.append(m.supervision_signal.clone())
                yvs.append(m.supervision_signal_valid.clone())
                n_packed += m.supervision_signal.numel()
            rec["events"].append({"timestamp": p["timestamp"], "propagated": ok,
                                  "in_range": [m.timestamp for m in got] if ok else [], "labels": labels})
        else:
            if est._mission_graph.get_num_valid_nodes() > PARAMS["min_samples"]:
                rec["samples"].append([m.timestamp for m in est._mission_graph.get_n_random_valid_nodes(n=PARAMS["batch_size"])])
            else:
                rec["samples"].append(None)
    rec["y"], rec["y_valid"] = torch.cat(ys).float(), torch.cat(yvs).bool()
    torch.save(rec, os.path.join(HERE, "mission_graph.pt"))
    n_prop = sum(e["propagated"] for e in rec["events"])
    print(f"{sum(a for _, a in rec['added'])} of {len(rec['added'])} frames added, {n_prop} of {len(rec['events'])} "
          f"events propagated, {sum(s is not None for s in rec['samples'])} train() samples")


if __name__ == "__main__":
    main()
