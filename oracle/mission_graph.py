"""TEST INFRASTRUCTURE ONLY (see oracle/__init__.py) — CPU restatement of the mission graph's data path: how a frame
becomes training data in the reference (traversability_estimator.py:166-300 add_mission_node / add_supervision_node,
graphs.py BaseGraph / DistanceWindowGraph, nodes.py MissionNode / SupervisionNode, train()'s sampling :449-463), on top
of oracle/image_projector.py for the footprint rendering and oracle/wvn_path.py for the per-segment pooling.

liegroups is not installed ([EXTERNAL-RECALLED], restated from its published source): ``SE3.from_matrix(T,
normalize=True).log()`` = SVD-normalised rotation, phi = SO3.log (first order below 1e-6 rad), rho = J^-1(phi) t.  It runs
in float32 like the reference's tensors, and the same functions stand in for liegroups when
tests/golden/make_golden_mission_graph.py runs the reference's own graphs.py / nodes.py.

``scenario()`` is the scripted trajectory the golden and the tests share.
"""
from __future__ import annotations

import math
import random

import torch

from oracle import image_projector as oip
from oracle.wvn_path import update_supervision_signal


# ---- liegroups, restated -------------------------------------------------------------------------------------------
def _wedge(v):
    z = torch.zeros((), dtype=v.dtype)
    return torch.stack([torch.stack([z, -v[2], v[1]]), torch.stack([v[2], z, -v[0]]), torch.stack([-v[1], v[0], z])])


def so3_normalize(R):
    U, _, V = torch.svd(R)
    S = torch.eye(3, dtype=R.dtype)
    S[2, 2] = torch.det(U) * torch.det(V)
    return U @ S @ V.T


def so3_log(R):
    cos_angle = (0.5 * torch.trace(R) - 0.5).clamp(-1.0, 1.0)
    angle = cos_angle.acos()
    if (angle - 0.0).abs() < 1e-6:
        P = R - torch.eye(3, dtype=R.dtype)
    else:
        P = (0.5 * angle / angle.sin()) * (R - R.T)
    return torch.stack([P[2, 1], P[0, 2], P[1, 0]])


def so3_inv_left_jacobian(phi):
    angle = phi.norm()
    if (angle - 0.0).abs() < 1e-6:
        return torch.eye(3, dtype=phi.dtype) - 0.5 * _wedge(phi)
    axis = phi / angle
    ha = 0.5 * angle
    hc = ha * (1.0 / ha.tan())
    return hc * torch.eye(3, dtype=phi.dtype) + (1 - hc) * torch.outer(axis, axis) - ha * _wedge(axis)


def se3_log(T):
    """[rho, phi] of SE3.from_matrix(T, normalize=True).log()."""
    R = so3_normalize(T[:3, :3])
    phi = so3_log(R)
    rho = so3_inv_left_jacobian(phi) @ T[:3, 3]
    return torch.cat([rho, phi])


def distance(pose_a, pose_b):
    """BaseNode.distance_to (nodes.py:76-93): a float32 0-dim tensor, as in the reference."""
    return se3_log(pose_a.inverse() @ pose_b)[:3].norm()


# ---- footprint (SupervisionNode.get_side_points / make_footprint_with_node, meshes.make_plane) -----------------------
def side_points(pose_footprint_in_world, width):
    pts = torch.tensor([[0.0, -width / 2, 0.0], [0.0, width / 2, 0.0]], dtype=torch.float32)
    return oip.transform_points(pose_footprint_in_world[None], pts[None])[0]


def footprint(this, other):
    tsp = side_points(this["pose_footprint_in_world"], this["width"])[[1, 0]]
    osp = side_points(other["pose_footprint_in_world"], other["width"])
    return oip.make_polygon_from_points(torch.cat((tsp, osp), dim=0), grid_size=10)


# ---- the estimator's data path ----------------------------------------------------------------------------------------
class MissionGraphOracle:
    """Unbounded (capacity=None) like the reference, or a ring of ``capacity`` nodes like the library's MissionGraph."""

    def __init__(self, H, W, image_distance_thr, supervision_distance_thr, max_distance, capacity=None):
        self.H, self.W = H, W
        self.image_distance_thr, self.sup_thr, self.max_distance = image_distance_thr, supervision_distance_thr, max_distance
        self.capacity = capacity
        self.nodes, self.edges = [], []
        self.sweep_pos = 0          # serial of the first node the 30 s sweep has not dropped
        self.serial = 0
        self.sup_nodes, self.sup_last = [], None

    def add_mission_node(self, n):
        if self.nodes:
            d = distance(n["pose_base_in_world"], self.nodes[-1]["pose_base_in_world"])
            if self.image_distance_thr is not None and d < self.image_distance_thr:
                return False
        if self.capacity is not None and len(self.nodes) == self.capacity:
            old = self.nodes.pop(0)
            self.edges.pop(0)
            self.sweep_pos = max(self.sweep_pos, old["serial"] + 1)
        if self.nodes:
            self.edges.append(d)
        node = dict(n, serial=self.serial, mask=torch.full((3, self.H, self.W), float("nan")), has_mask=True)
        self.serial += 1
        node["y"], node["y_valid"] = update_supervision_signal(node["mask"], node["seg"])
        self.nodes.append(node)
        return True

    def in_range(self):
        t_last = self.nodes[-1]["timestamp"]
        q = next(k for k, nd in enumerate(self.nodes) if abs(nd["timestamp"] - t_last) < 1)
        out = []
        d, k = 0, q - 1
        while k >= 0:
            d = d + self.edges[k]
            if d > self.max_distance:
                break
            out.append(k)
            k -= 1
        d, k = 0, q + 1
        while k < len(self.nodes):
            d = d + self.edges[k - 1]
            if d > self.max_distance:
                break
            out.append(k)
            k += 1
        return sorted(out)

    def add_supervision_node(self, p):
        """-> the timestamps of the in-range nodes that received labels, or None when the event propagated nothing."""
        last_p = self.sup_last
        if last_p is not None and self.sup_thr is not None and distance(p["pose_base_in_world"], last_p["pose_base_in_world"]) < self.sup_thr:
            if (p["traversability"] < last_p["traversability"]).any():
                last_p["traversability"] = p["traversability"]
            return None
        self.sup_last = p
        if last_p is None or not self.nodes:
            return None
        fp = footprint(p, last_p)
        last = self.nodes[-1]
        if not last["has_mask"]:
            return None
        for nd in self.nodes:
            if nd["serial"] < self.sweep_pos:
                continue
            if last["timestamp"] - nd["timestamp"] > 30:
                nd["has_mask"] = False
                self.sweep_pos = nd["serial"] + 1
            else:
                break
        idx = self.in_range()
        if not idx:
            return None
        nodes = [self.nodes[k] for k in idx]
        K = torch.stack([nd["K"] for nd in nodes])
        poses = torch.stack([nd["pose_cam_in_world"] for nd in nodes])
        masks, _, _ = oip.project_and_render(K, self.H, self.W, poses, fp[None].repeat(len(nodes), 1, 1), torch.ones(3))
        for i, nd in enumerate(nodes):
            old = nd["mask"] if nd["has_mask"] else torch.zeros(3, self.H, self.W)
            nd["mask"] = torch.fmin(old, masks[i] * p["traversability"])
            nd["has_mask"] = True
            nd["y"], nd["y_valid"] = update_supervision_signal(nd["mask"], nd["seg"])
        return [nd["timestamp"] for nd in nodes]

    def valid_nodes(self):
        return [nd for nd in self.nodes if bool(nd["y_valid"].any())]

    def sample(self, batch_size):
        nodes = sorted(self.valid_nodes(), key=lambda nd: nd["timestamp"])
        random.shuffle(nodes)
        return nodes[:batch_size]


def golden_labels(golden, event):
    """{node timestamp: (y, y_valid)} of one recorded event of tests/golden/mission_graph.pt (labels stored packed)."""
    return {t: (golden["y"][o : o + n], golden["y_valid"][o : o + n]) for t, (o, n) in event["labels"].items()}


# ---- the scripted trajectory --------------------------------------------------------------------------------------------
def _pose(x, y, yaw, z=0.0):
    T = torch.eye(4)
    c, s = math.cos(yaw), math.sin(yaw)
    T[:2, :2] = torch.tensor([[c, -s], [s, c]])
    T[:3, 3] = torch.tensor([x, y, z])
    return T


def camera_in_base(pitch=0.55, height=1.0):
    """Camera 1 m above the base, looking forward (+x) and pitched down; camera axes z forward, x right, y down."""
    T = torch.eye(4)
    cp, sp = math.cos(pitch), math.sin(pitch)
    z = torch.tensor([cp, 0.0, -sp])
    x = torch.tensor([0.0, -1.0, 0.0])
    y = torch.linalg.cross(z, x)
    T[:3, 0], T[:3, 1], T[:3, 2] = x, y, z
    T[2, 3] = height
    return T


def segmentation(H, W, seed, cell=32):
    """Blocks of cell x cell pixels with seeded ids in [0, (H/cell) (W/cell))."""
    g = torch.Generator().manual_seed(seed)
    nb = (H // cell) * (W // cell)
    ids = torch.randperm(nb, generator=g)
    blocks = ids.reshape(H // cell, W // cell)
    return blocks.repeat_interleave(cell, 0).repeat_interleave(cell, 1).long(), nb


def scenario(n_mission=60, H=224, D=32, seed=0):
    """60 poses along an arc (radius 12 m, 0.15 m apart, one mission frame every 1.25 s, a 224^2 pinhole camera),
    supervision nodes every 0.4 s along the same path with seeded traversabilities (multiples of 1/16, so the per-segment
    sums are exact in float32).  Extras: every 13th mission frame comes twice (the copy is refused by the 0.1 m edge
    gate); supervision nodes 4.8 cm apart alternate with the 0.05 m gate (every other one only lowers the last node's
    traversability), and one lands 1 cm from its predecessor; the robot stands still for 32 s after frame 30, so the
    30 s sweep drops the masks of nodes that are still in range and the next event restarts them from zeros.  -> list of events
    ("mission", node) | ("supervision", node) | ("train",)."""
    g = torch.Generator().manual_seed(seed)
    f = 0.6 * H
    K = torch.tensor([[f, 0, H / 2, 0], [0, f, H / 2, 0], [0, 0, 1, 0], [0, 0, 0, 1.0]])
    cib = camera_in_base()
    R, step, dt = 12.0, 0.15, 1.25

    def base(s):
        th = s / R
        return _pose(R * math.sin(th), R * (1 - math.cos(th)), th)

    stop_i, stop_s = 30, 32.0     # the robot stands still for 32 s after frame 30

    def time_of(i):
        return i * dt + (stop_s if i > stop_i else 0.0)

    def path_at(t):
        if t <= stop_i * dt:
            return t / dt * step
        return max(stop_i * step, (t - stop_s) / dt * step)

    events = []
    sup_t = 0.0
    for i in range(n_mission):
        t = time_of(i)
        s = i * step
        while sup_t <= t:   # the robot's supervision nodes up to this frame's time
            ss = path_at(sup_t)
            trav = torch.tensor([float(torch.randint(1, 16, (1,), generator=g)) / 16])
            events.append(("supervision", {"timestamp": sup_t, "pose_base_in_world": base(ss),
                                           "pose_footprint_in_world": base(ss), "width": 0.6, "traversability": trav}))
            if abs(sup_t - 20.0) < 1e-9:
                events.append(("supervision", {"timestamp": sup_t + 0.01, "pose_base_in_world": base(ss + 0.01),
                                               "pose_footprint_in_world": base(ss + 0.01), "width": 0.6,
                                               "traversability": trav * 0.5}))
            sup_t = round(sup_t + 0.4, 6)
        seg, nb = segmentation(H, H, seed=1000 + i)
        feat = torch.randn(nb, D, generator=g)
        B = base(s)
        node = {"timestamp": t, "pose_base_in_world": B, "pose_cam_in_world": B @ cib, "K": K.clone(), "seg": seg,
                "features": feat}
        events.append(("mission", node))
        if i % 13 == 12:
            B2 = base(s + 0.02)
            events.append(("mission", dict(node, timestamp=t + 0.1, pose_base_in_world=B2, pose_cam_in_world=B2 @ cib)))
        if i >= 8:
            events.append(("train",))
    return events
