"""The mission graph on the GPU (reference: traversability_estimator/graphs.py, nodes.py, and
``TraversabilityEstimator.add_mission_node`` / ``add_supervision_node`` / ``train``, traversability_estimator.py:165-300,
449-497).

``MissionGraph`` is a fixed-capacity ring of slots allocated once: per slot the node's per-segment features, its
segmentation, its supervision mask, its per-segment labels ``y`` / ``y_valid`` and its camera (scaled K and
``pose_cam_in_world``), all on the device.  The bookkeeping — timestamps, base poses, the distances along the chain and
whether a node still has its mask — is a few numbers per node and stays on the host.  A supervision event
(``wvn_mission_propagate``) renders the footprint into every in-range slot, takes ``fmin`` into its mask and re-pools
its labels in one launch, with no host synchronisation.

Differences from the reference, all deliberate:
  * The reference's graph is unbounded.  Here the ring holds ``capacity`` nodes; adding one more overwrites the oldest,
    and that raises ``ValueError`` when the oldest node is still within ``max_distance`` of the newest along the graph
    (it would have received labels), so a ring that is too small cannot silently drop training data.
  * ``edge_distance=None`` means no gating (the reference compares ``d < None`` and raises).
  * The mission graph is a chain (each node has an edge to the one added before it), so Dijkstra's range query is the
    sum of the edge lengths walked outwards from the query node.

Reference behaviour kept, including its quirks:
  * The range query starts at the earliest node whose timestamp is within 1 s of the last node's
    (``get_node_with_timestamp(eps=1)``) and excludes that node (``list(length)[1:]``).  With nodes more than 1 s apart
    that node is the last one, so the newest node never receives the footprint.
  * Every event first drops the mask of each node more than 30 s older than the newest (``clear_debug_data``, a sweep
    that moves forward from the oldest node and stops at the first younger one).  A later event that reaches such a node
    restarts it from a zero mask, which wipes its labels (y becomes 0, so the node stops being valid).
  * A node is valid when at least one of its segments has a positive label (``is_valid``); ``train()`` samples sorted
    valid nodes with ``random.shuffle``.
"""
from __future__ import annotations

import math
import random

import numpy as np
import torch

from .. import ops

SWEEP_SECONDS = 30.0      # traversability_estimator.py:243
QUERY_TIME_EPS = 1.0      # graphs.py:163, get_node_with_timestamp(eps=time_eps=1)


# --------------------------------------------------------------------------------------------
# SE(3) distance (BaseNode.distance_to, nodes.py:76-93: |log(inv(A) B)[:3]|, liegroups restated in float64)
# --------------------------------------------------------------------------------------------
def _wedge(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def se3_log_translation(T: np.ndarray) -> np.ndarray:
    """The translational part rho of the SE(3) logarithm of the 4x4 matrix T, rotation normalised by SVD first
    (SE3.from_matrix(normalize=True).log()[:3])."""
    R, t = T[:3, :3], T[:3, 3]
    U, _, Vh = np.linalg.svd(R)
    S = np.eye(3)
    S[2, 2] = np.linalg.det(U) * np.linalg.det(Vh)
    R = U @ S @ Vh
    cos_angle = min(max(0.5 * np.trace(R) - 0.5, -1.0), 1.0)
    angle = math.acos(cos_angle)
    if abs(angle) < 1e-6:
        phi = np.array([R[2, 1], R[0, 2], R[1, 0]])          # vee(R - I), first order
    else:
        A = (0.5 * angle / math.sin(angle)) * (R - R.T)
        phi = np.array([A[2, 1], A[0, 2], A[1, 0]])
    a = np.linalg.norm(phi)
    if abs(a) < 1e-6:
        J_inv = np.eye(3) - 0.5 * _wedge(phi)
    else:
        axis = phi / a
        ha = 0.5 * a
        hc = ha / math.tan(ha)
        J_inv = hc * np.eye(3) + (1.0 - hc) * np.outer(axis, axis) - ha * _wedge(axis)
    return J_inv @ t


def _as_np(pose) -> np.ndarray:
    if torch.is_tensor(pose):
        pose = pose.detach().cpu()   # a host tensor: no copy, no synchronisation
    return np.asarray(pose, dtype=np.float64).reshape(4, 4)


def pose_distance(pose_a, pose_b) -> float:
    """``BaseNode.distance_to``: node a's distance to node b, from their base poses."""
    return float(np.linalg.norm(se3_log_translation(np.linalg.inv(_as_np(pose_a)) @ _as_np(pose_b))))


# --------------------------------------------------------------------------------------------
# Supervision side (nodes.py:443-617, graphs.py:289-316, utils/meshes.py)
# --------------------------------------------------------------------------------------------
def _transform_points(pose: torch.Tensor, pts: torch.Tensor) -> torch.Tensor:
    """kornia transform_points of (N,3) points by one 4x4 pose, in float32 as the reference runs it."""
    ph = torch.cat([pts, torch.ones_like(pts[:, :1])], dim=1)[None]
    h = torch.bmm(ph, pose.float()[None].transpose(1, 2))[0]
    z = h[:, 3:]
    scale = torch.where(z.abs() > 1e-8, 1.0 / (z + 1e-8), torch.ones_like(z))
    return scale * h[:, :3]


def side_points(pose_footprint_in_world: torch.Tensor, width: float) -> torch.Tensor:
    """``SupervisionNode.get_side_points``: make_plane(x=0, y=width, grid_size=2) — after its torch.unique the two
    points (0, -width/2, 0), (0, width/2, 0) — in the world frame."""
    pts = torch.tensor([[0.0, -width / 2, 0.0], [0.0, width / 2, 0.0]], dtype=torch.float32)
    return _transform_points(pose_footprint_in_world.detach().cpu(), pts)


def polygon_from_points(points: torch.Tensor, grid_size: int = 10) -> torch.Tensor:
    """utils/meshes.py make_polygon_from_points: every edge of the closed point list sampled at grid_size points."""
    n = points.shape[0]
    w = torch.linspace(0, 1, steps=grid_size)
    return torch.cat([torch.lerp(points[i], points[(i + 1) % n], wi)[None] for i in range(n) for wi in w], dim=0)


def footprint_between(this, other, grid_size: int = 10) -> torch.Tensor:
    """``SupervisionNode.make_footprint_with_node`` for traversable footprints: this node's side points swapped, then
    the other's, as one polygon.  Untraversable footprints (``get_untraversable_plane``) raise ``ValueError``; the
    default ``untraversable_thr`` of 0.0 never produces them."""
    if getattr(this, "is_untraversable", False):
        raise ValueError("untraversable footprints (SupervisionNode.get_untraversable_plane) are not supported")
    tsp = side_points(this.pose_footprint_in_world, _width(this))
    osp = side_points(other.pose_footprint_in_world, _width(other))
    tsp = tsp[[1, 0]]
    return polygon_from_points(torch.cat((tsp, osp), dim=0), grid_size=grid_size)


def _width(node):
    return float(getattr(node, "_width", getattr(node, "width", 0.1)))


class SupervisionNode:
    """The reference's ``SupervisionNode`` (nodes.py:443-617) for what the mission graph reads: poses, footprint width,
    traversability (kept pessimistically by ``update_traversability``) and the supervision state that makes it valid."""

    def __init__(self, timestamp: float = 0.0, pose_base_in_world: torch.Tensor = torch.eye(4),
                 pose_footprint_in_base: torch.Tensor = torch.eye(4), pose_footprint_in_world: torch.Tensor = None,
                 twist_in_base: torch.Tensor = None, desired_twist_in_base: torch.Tensor = None, length: float = 0.1,
                 width: float = 0.1, height: float = 0.1, supervision: torch.Tensor = None,
                 traversability: torch.Tensor = torch.FloatTensor([0.0]),
                 traversability_var: torch.Tensor = torch.FloatTensor([1.0]), is_untraversable: bool = False):
        self.timestamp = timestamp
        self.pose_base_in_world = pose_base_in_world
        self.pose_footprint_in_base = pose_footprint_in_base
        self.pose_footprint_in_world = (pose_base_in_world @ pose_footprint_in_base if pose_footprint_in_world is None
                                        else pose_footprint_in_world)
        self.twist_in_base, self.desired_twist_in_base = twist_in_base, desired_twist_in_base
        self._length, self._width, self._height = length, width, height
        self.supervision_state = supervision
        self.traversability, self.traversability_var = traversability, traversability_var
        self.is_untraversable = is_untraversable

    def is_valid(self):
        return isinstance(self.supervision_state, torch.Tensor)

    def distance_to(self, other):
        return pose_distance(self.pose_base_in_world, other.pose_base_in_world)

    def update_traversability(self, traversability, traversability_var):
        if (traversability < self.traversability).any():   # pessimistic: keep the less traversable value
            self.traversability, self.traversability_var = traversability, traversability_var

    def make_footprint_with_node(self, other, grid_size: int = 10):
        return footprint_between(self, other, grid_size)


class DistanceWindowGraph:
    """graphs.py:289-316 on the host: a node closer than ``edge_distance`` to the last added one is refused; adding one
    drops the oldest nodes whose position is farther than ``max_distance`` from it, up to the first that is not."""

    def __init__(self, edge_distance: float = None, max_distance: float = float("inf")):
        self._edge_distance, self._max_distance = edge_distance, max_distance
        self._nodes, self._last = [], None

    @property
    def max_distance(self):
        return self._max_distance

    def add_node(self, node) -> bool:
        if self._last is not None and self._edge_distance is not None:
            if pose_distance(node.pose_base_in_world, self._last.pose_base_in_world) < self._edge_distance:
                return False
        self._nodes.append(node)
        self._last = node
        p = _as_np(node.pose_base_in_world)[:3, 3]
        while self._nodes and np.linalg.norm(_as_np(self._nodes[0].pose_base_in_world)[:3, 3] - p) > self._max_distance:
            self._nodes.pop(0)
        return True

    def get_last_node(self):
        return self._last

    def get_nodes(self):
        return sorted(self._nodes, key=lambda n: n.timestamp)

    def get_num_nodes(self):
        return len(self._nodes)


# --------------------------------------------------------------------------------------------
# the mission graph
# --------------------------------------------------------------------------------------------
def range_query(timestamps, edges, max_distance):
    """Chain form of get_nodes_within_radius_range(last, 0, max_distance): (query index, in-range indices in order).
    ``edges[k]`` is the length of the edge between node k and node k + 1."""
    n = len(timestamps)
    if n == 0:
        return None, []
    t_last = timestamps[-1]
    q = next(k for k in range(n) if abs(timestamps[k] - t_last) < QUERY_TIME_EPS)
    out = []
    d, k = 0.0, q - 1
    while k >= 0:
        d += edges[k]
        if d > max_distance:
            break
        out.append(k)
        k -= 1
    d, k = 0.0, q + 1
    while k < n:
        d += edges[k - 1]
        if d > max_distance:
            break
        out.append(k)
        k += 1
    return q, sorted(out, key=lambda i: (timestamps[i], i))


class MissionGraphNode:
    """A view of one node of a ``MissionGraph``: host bookkeeping plus its slot in the device buffers."""

    __slots__ = ("graph", "slot", "serial", "timestamp", "pose_base_in_world", "has_mask")

    def __init__(self, graph, slot, serial, timestamp, pose_base_in_world, has_mask):
        self.graph, self.slot, self.serial = graph, slot, serial
        self.timestamp, self.pose_base_in_world, self.has_mask = timestamp, pose_base_in_world, has_mask

    def __lt__(self, other):
        return self.timestamp < other.timestamp

    def __repr__(self):
        return f"mission_node_{self.timestamp}"

    def distance_to(self, other):
        return pose_distance(self.pose_base_in_world, other.pose_base_in_world)

    @property
    def features(self):
        return self.graph.features[self.slot]

    @property
    def feature_segments(self):
        return self.graph.seg[self.slot]

    @property
    def supervision_mask(self):
        return self.graph.mask[self.slot] if self.has_mask else None

    @property
    def supervision_signal(self):
        return self.graph.y[self.slot]

    @property
    def supervision_signal_valid(self):
        return self.graph.y_valid[self.slot].bool()

    def is_valid(self):
        return bool(self.graph.valid_flags()[self.slot])


def _pinned(nbytes):
    return torch.empty(max(int(nbytes), 4), dtype=torch.uint8, pin_memory=True)


class MissionGraph:
    """Fixed-capacity ring of mission nodes with their training data and labels on the device (see the module doc).

    Device buffers (``capacity`` slots): ``features`` [cap, smax, D] fp32, ``meta`` [2, cap] int32 (row 0 = n_rows,
    row 1 = valid flag written by each propagation), ``seg`` [cap, H, W] int32, ``mask`` [cap, H, W] fp32 (NaN =
    unlabelled), ``y`` [cap, smax] fp32, ``y_valid`` [cap, smax] uint8, ``K`` / ``pose_cam_in_world`` [cap, 4, 4] fp32."""

    def __init__(self, capacity: int, height: int, width: int, smax: int, dim: int, device="cuda",
                 edge_distance: float = None, max_distance: float = float("inf")):
        if capacity < 1 or smax < 1 or smax > 4096 or height < 1 or width < 1:
            raise ValueError(f"MissionGraph: bad geometry (capacity {capacity}, {height}x{width}, smax {smax})")
        dev = torch.device(device)
        self.capacity, self.height, self.width, self.smax, self.dim = capacity, height, width, smax, dim
        self.device, self.edge_distance, self.max_distance = dev, edge_distance, max_distance
        self.features = torch.zeros(capacity, smax, dim, device=dev)
        self.meta = torch.zeros(2, capacity, device=dev, dtype=torch.int32)
        self.n_rows, self.slot_valid = self.meta[0], self.meta[1]
        self.seg = torch.zeros(capacity, height, width, device=dev, dtype=torch.int32)
        self.mask = torch.full((capacity, height, width), float("nan"), device=dev)
        self.y = torch.zeros(capacity, smax, device=dev)
        self.y_valid = torch.zeros(capacity, smax, device=dev, dtype=torch.uint8)
        self.K = torch.eye(4, device=dev).repeat(capacity, 1, 1)
        self.pose_cam_in_world = torch.eye(4, device=dev).repeat(capacity, 1, 1)
        self._ws = ops.mission_propagate_workspace(capacity, smax, dev)
        self._nodes = []          # live nodes, oldest first
        self._edges = []          # _edges[k]: distance between _nodes[k] and _nodes[k + 1]
        self._serial = 0
        self._sweep_serial = 0    # first node the 30 s sweep has not dropped yet
        self._head = 0            # slot of the oldest node
        self._meta_host = None    # last host copy of meta, None when stale

    # ---- queries (graphs.py:97-143) ------------------------------------------------------------
    def get_nodes(self):
        return sorted(self._nodes)

    def get_first_node(self):
        return self._nodes[0] if self._nodes else None

    def get_last_node(self):
        return self._nodes[-1] if self._nodes else None

    def get_num_nodes(self):
        return len(self._nodes)

    def valid_flags(self):
        """Per slot: at least one positive label.  One device-to-host copy of ``meta`` (n_rows and the flags) when the
        device has changed them since the last call."""
        if self._meta_host is None:
            self._meta_host = self.meta.cpu().numpy()
        return self._meta_host[1]

    def host_n_rows(self):
        self.valid_flags()
        return self._meta_host[0]

    def get_valid_nodes(self):
        v = self.valid_flags()
        return sorted(n for n in self._nodes if v[n.slot])

    def get_num_valid_nodes(self):
        return len(self.get_valid_nodes())

    def get_n_random_valid_nodes(self, n=None):
        nodes = self.get_valid_nodes()
        random.shuffle(nodes)
        return nodes if n is None else nodes[:n]

    def get_nodes_within_radius_range(self, max_distance=None):
        """The in-range nodes of the next supervision event, measured along the graph from the last node."""
        _, idx = range_query([n.timestamp for n in self._nodes], self._edges,
                             self.max_distance if max_distance is None else max_distance)
        return [self._nodes[k] for k in idx]

    # ---- insertion (BaseGraph.add_node, graphs.py:57-86) ---------------------------------------------
    def _reserve(self, timestamp, pose_base_in_world):
        """Gate a new node on its distance to the last one; returns its slot, or None when it is refused."""
        d = None
        if self._nodes:
            d = pose_distance(pose_base_in_world, self._nodes[-1].pose_base_in_world)
            if self.edge_distance is not None and d < self.edge_distance:
                return None
        if len(self._nodes) == self.capacity:
            _, idx = range_query([n.timestamp for n in self._nodes] + [timestamp], self._edges + [d], self.max_distance)
            if idx and idx[0] == 0:
                raise ValueError(f"MissionGraph: the ring of {self.capacity} nodes is full and its oldest node is still "
                                 f"within {self.max_distance} of the newest; raise the capacity")
            old = self._nodes.pop(0)
            if self._edges:
                self._edges.pop(0)
            self._head = (self._head + 1) % self.capacity
            self._sweep_serial = max(self._sweep_serial, old.serial + 1)
        slot = (self._head + len(self._nodes)) % self.capacity
        if self._nodes:
            self._edges.append(d)
        return slot

    def _commit(self, slot, timestamp, pose_base_in_world, has_mask):
        node = MissionGraphNode(self, slot, self._serial, timestamp, _as_np(pose_base_in_world).copy(), has_mask)
        self._serial += 1
        self._nodes.append(node)
        return node

    def _h2d(self, arr: np.ndarray) -> torch.Tensor:
        """Host array -> device through pinned memory, enqueued without waiting."""
        buf = _pinned(arr.nbytes)
        buf.numpy()[: arr.nbytes] = np.frombuffer(np.ascontiguousarray(arr).tobytes(), dtype=np.uint8)
        return buf.to(self.device, non_blocking=True)

    def _reset_slots(self, slots_t):
        self.mask.index_fill_(0, slots_t, float("nan"))
        self.y.index_fill_(0, slots_t, 0.0)
        self.y_valid.index_fill_(0, slots_t, 0)
        self.slot_valid.index_fill_(0, slots_t, 0)
        self._meta_host = None

    def add(self, features, seg, K, pose_cam_in_world, timestamp, pose_base_in_world, has_mask=True):
        """One node: features [S, D] (S <= smax), seg [H, W] (any integer dtype), K the scaled 4x4 camera matrix of the
        H x W image, poses 4x4.  Returns the node, or None when the edge gate refuses it.  A node without a mask
        (``has_mask=False``, the reference's ``use_for_training=False``) starts from a zero mask at its first event."""
        S = features.shape[0]
        if S > self.smax or features.shape[1] != self.dim or tuple(seg.shape) != (self.height, self.width):
            raise ValueError(f"MissionGraph.add: features {tuple(features.shape)} / segmentation {tuple(seg.shape)} do "
                             f"not fit slots of ({self.smax}, {self.dim}) / ({self.height}, {self.width})")
        slot = self._reserve(timestamp, pose_base_in_world)
        if slot is None:
            return None
        cam = np.concatenate([_as_np(K).astype(np.float32).ravel(), _as_np(pose_cam_in_world).astype(np.float32).ravel(),
                              np.array([S], np.int32).view(np.float32), np.array([slot], np.int32).view(np.float32)])
        dev = self._h2d(cam)
        f = dev.view(torch.float32)
        self.K[slot].copy_(f[:16].view(4, 4))
        self.pose_cam_in_world[slot].copy_(f[16:32].view(4, 4))
        self.n_rows[slot : slot + 1].copy_(dev[128:132].view(torch.int32))
        self.features[slot, :S].copy_(features.to(self.device, torch.float32))
        self.seg[slot].copy_(seg.to(self.device))
        self._reset_slots(dev[132:136].view(torch.int32).long())
        return self._commit(slot, timestamp, pose_base_in_world, has_mask)

    def add_frames(self, feat, n_rows, seg, K, poses_cam_in_world, timestamps, poses_base_in_world):
        """A batch of frames as ``FeatureExtractor.extract_batch`` leaves them (feat [B, S, D], n_rows [B] int32 and
        seg [B, H, W] on the device), copied device to device.  K / poses: [B, 4, 4] host tensors (K may be one 4x4).
        Returns the nodes that passed the edge gate."""
        B, S, D = feat.shape
        if S > self.smax or D != self.dim or tuple(seg.shape[1:]) != (self.height, self.width):
            raise ValueError(f"MissionGraph.add_frames: feat {tuple(feat.shape)} / seg {tuple(seg.shape)} do not fit "
                             f"slots of ({self.smax}, {self.dim}) / ({self.height}, {self.width})")
        K = torch.as_tensor(K, dtype=torch.float32).cpu()
        K = K.expand(B, 4, 4) if K.dim() == 2 else K
        taken, slots = [], []
        for b in range(B):
            slot = self._reserve(float(timestamps[b]), poses_base_in_world[b])
            if slot is None:
                continue
            taken.append(b)
            slots.append(slot)
            self._commit(slot, float(timestamps[b]), poses_base_in_world[b], True)
        if not taken:
            return []
        n = len(taken)
        cam = np.concatenate([K[taken].numpy().astype(np.float32).ravel(),
                              np.asarray(torch.as_tensor(poses_cam_in_world, dtype=torch.float32).cpu()[taken]).ravel(),
                              np.asarray(taken, np.int32).view(np.float32), np.asarray(slots, np.int32).view(np.float32)])
        dev = self._h2d(cam)
        f = dev.view(torch.float32)
        frames_t = f[32 * n : 33 * n].view(torch.int32).long()
        slots_t = f[33 * n : 34 * n].view(torch.int32).long()
        self.K.index_copy_(0, slots_t, f[: 16 * n].view(n, 4, 4))
        self.pose_cam_in_world.index_copy_(0, slots_t, f[16 * n : 32 * n].view(n, 4, 4))
        self.features[:, :S].index_copy_(0, slots_t, feat.index_select(0, frames_t))
        self.n_rows.index_copy_(0, slots_t, n_rows.to(torch.int32).index_select(0, frames_t))
        self.seg.index_copy_(0, slots_t, seg.index_select(0, frames_t).to(torch.int32))
        self._reset_slots(slots_t)
        return self._nodes[-n:]

    # ---- one supervision event (add_supervision_node, traversability_estimator.py:233-289) ------------------------
    def sweep(self, t_last):
        """The 30 s ``clear_debug_data`` sweep: drops the masks of the nodes more than 30 s older than ``t_last``."""
        for node in self._nodes:
            if node.serial < self._sweep_serial:
                continue
            if t_last - node.timestamp > SWEEP_SECONDS:
                node.has_mask = False
                self._sweep_serial = node.serial + 1
            else:
                break

    def propagate(self, nodes, footprint: torch.Tensor, traversability):
        """Render ``footprint`` (N, 3) world points with ``traversability`` into ``nodes``' masks and re-pool their
        labels: one H2D copy from pinned memory and one ``wvn_mission_propagate`` launch, nothing waits."""
        n, N = len(nodes), footprint.shape[0]
        trav_dev = torch.is_tensor(traversability) and traversability.is_cuda
        tv = 0.0 if trav_dev else float(torch.as_tensor(traversability).reshape(-1)[0])
        host = np.concatenate([footprint.detach().cpu().float().numpy().ravel(), np.array([tv], np.float32),
                               np.array([nd.slot for nd in nodes], np.int32).view(np.float32),
                               np.array([0 if nd.has_mask else 1 for nd in nodes], np.int32).view(np.float32)])
        dev = self._h2d(host).view(torch.float32)
        points, trav = dev[: 3 * N].view(N, 3), dev[3 * N : 3 * N + 1]
        if trav_dev:
            trav.copy_(traversability.reshape(-1)[:1].float())
        slots = dev[3 * N + 1 : 3 * N + 1 + n].view(torch.int32)
        restart = dev[3 * N + 1 + n : 3 * N + 1 + 2 * n].view(torch.int32).to(torch.uint8)
        ops.mission_propagate(slots, restart, self.K, self.pose_cam_in_world, points, trav, self.seg, self.mask, self.y,
                              self.y_valid, self.slot_valid, self._ws)
        for nd in nodes:
            nd.has_mask = True
        self._meta_host = None

    # ---- training batch (make_batch, traversability_estimator.py:431-446) -------------------------------------------
    def gather(self, nodes):
        """The sampled nodes in the padded layout ``train_on_padded`` takes: feat [B, smax, D], n_rows [B] int32, and
        y / y_valid compacted (node by node, the first n_rows of each).  Uses the host copy of n_rows."""
        nr = self.host_n_rows()
        feat = torch.stack([self.features[nd.slot] for nd in nodes])
        n_rows = torch.stack([self.n_rows[nd.slot] for nd in nodes])
        y = torch.cat([self.y[nd.slot, : int(nr[nd.slot])] for nd in nodes])
        y_valid = torch.cat([self.y_valid[nd.slot, : int(nr[nd.slot])] for nd in nodes])
        return feat, n_rows, y, y_valid
