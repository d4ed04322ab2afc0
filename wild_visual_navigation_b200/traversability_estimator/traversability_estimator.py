"""TraversabilityEstimator — the online learner
(reference: wild_visual_navigation/traversability_estimator/traversability_estimator.py:33-505).

On the hot path and implemented: ``__init__`` (seed 42, SimpleMLP + TraversabilityLoss, or with
``anomaly_detection=True`` LinearRnvp + AnomalyLoss, Adam — :78-105), ``make_batch`` (:431-446), ``train`` (:448-497, same return dict), ``save_checkpoint`` /
``load_checkpoint`` (:377-429, same file format incl. a torch.optim.Adam-compatible
``optimizer_state_dict``), ``pause_learning`` / ``step`` / ``loss``.
Mission nodes that carry camera data (the reference's own ``MissionNode`` objects, or whole
``FeatureExtractor.extract_batch`` results through ``add_mission_frames``) go into a device-resident
mission graph (mission_graph.py), and ``add_supervision_node`` propagates each footprint into every
in-range node's labels on the GPU; ``train()`` then samples labelled nodes from that graph as the
reference does.  Nodes without camera data are kept in a plain list and must already carry their
per-segment features and supervision (``MissionNode`` below), as before.  Visualisation is out of scope.

``train()`` runs forward + loss + backward + Adam as one fixed sequence of fp32 CUDA kernels
(csrc/mlp_train_fused.cu) with all scalars on the device.
In anomaly-detection mode the step is the LinearRnvp flow's (csrc/flow_train.cu: forward, NLL, confidence update,
backward, Adam) on the labelled rows only.  With ``model.name == "DoubleMLP"`` the step is the DoubleMLP's
(csrc/double_mlp_train.cu: the same TraversabilityLoss on two separate networks).
Every learner is data-parallel: with a ``process_group`` the confidence statistics (sums, row counts, extrema) and the
flat gradient are all-reduced inside the step (NCCL over NVLink) for a global-batch step, and every learner takes rows
still padded per frame (``train_on_padded``).
"""
from __future__ import annotations

import os
import random
from threading import Lock

import torch

from .. import ops
from ..model import get_model
from ..utils import AnomalyLoss, Batch, Data, TraversabilityLoss
from .mission_graph import DistanceWindowGraph, MissionGraph, footprint_between


def default_params(anomaly_detection: bool = False):
    """The defaults of ``ExperimentParams`` that define the hot path (cfg/experiment_params.py:44-65,91,104-140); with
    ``anomaly_detection`` the model is ``LinearRnvp`` (what the nodes select with ``model.name = "LinearRnvp"``)."""
    return {
        "model": {"name": "LinearRnvp" if anomaly_detection else "SimpleMLP",
                  "simple_mlp_cfg": {"input_size": 384, "hidden_sizes": [256, 32, 1], "reconstruction": True},
                  "double_mlp_cfg": {"input_size": 384, "hidden_sizes": [64, 32, 1]},
                  "linear_rnvp_cfg": {"input_size": 384, "coupling_topology": [200], "mask_type": "odds",
                                      "conditioning_size": 0, "use_permutation": True, "single_function": False}},
        "loss": {"anomaly_balanced": True, "w_trav": 0.03, "w_temp": 0.0, "w_reco": 0.5, "method": "latest_measurement",
                 "confidence_std_factor": 0.5, "trav_cross_entropy": False},
        "loss_anomaly": {"method": "latest_measurement", "confidence_std_factor": 0.5},
        "optimizer": {"name": "ADAM", "lr": 0.001},
        "ablation_data_module": {"batch_size": 8},
        "general": {"log_confidence": False, "model_path": "/tmp"},
    }


class MissionNode:
    """What ``MissionNode.as_pyg_data`` hands to the learner (nodes.py:199-241): per-segment
    features ``x (S,D)``, supervision ``y (S,)`` in [0,1] and ``y_valid (S,)`` bool."""

    def __init__(self, features: torch.Tensor, supervision_signal: torch.Tensor, supervision_signal_valid: torch.Tensor,
                 timestamp: float = 0.0):
        self.features = features
        self.supervision_signal = supervision_signal
        self.supervision_signal_valid = supervision_signal_valid
        self.timestamp = timestamp

    def is_valid(self):
        return self.features is not None and self.supervision_signal is not None

    def update_supervision_signal(self, supervision_mask: torch.Tensor, feature_segments: torch.Tensor):
        """Per-segment labels from a rendered supervision mask (nodes.py:400-440): ``supervision_mask`` (C,H,W) or
        (H,W) with NaN = unlabelled, ``feature_segments`` (H,W) long.  One CUDA reduction instead of the reference's
        (H, W, S) expansion; S = number of feature rows."""
        from .. import ops

        mask = supervision_mask if supervision_mask.dim() == 3 else supervision_mask[None]
        y, valid = ops.pool_supervision(feature_segments[None].contiguous(), mask[None].float().contiguous(),
                                        int(self.features.shape[0]))
        self.supervision_signal, self.supervision_signal_valid = y[0], valid[0]

    def as_pyg_data(self, anomaly_detection: bool = False):
        if anomaly_detection:   # the flow learns from the labelled rows only (nodes.py:207-214)
            v = self.supervision_signal_valid
            return Data(x=self.features[v], y=self.supervision_signal[v], y_valid=v[v])
        return Data(x=self.features, y=self.supervision_signal, y_valid=self.supervision_signal_valid)


def _get(p, key):
    return p[key] if isinstance(p, dict) else getattr(p, key)


def _check_padded_args(feat, n_rows, y, y_valid, dim, y_optional):
    def bad(what):
        raise ValueError(f"train_on_padded: {what}")

    if not torch.is_tensor(feat) or feat.dim() != 3 or feat.dtype != torch.float32 or feat.shape[2] != dim:
        bad(f"feat must be a (B, smax, {dim}) float32 tensor")
    if not torch.is_tensor(n_rows) or n_rows.dtype != torch.int32 or tuple(n_rows.shape) != (feat.shape[0],):
        bad(f"n_rows must be a ({feat.shape[0]},) int32 tensor")
    if not (y is None and y_optional) and (not torch.is_tensor(y) or y.dim() != 1 or not y.is_floating_point()):
        bad("y must be a 1-D floating-point tensor")
    if not torch.is_tensor(y_valid) or y_valid.dim() != 1 or y_valid.dtype not in (torch.bool, torch.uint8):
        bad("y_valid must be a 1-D bool or uint8 tensor")
    for t in (n_rows, y, y_valid):
        if t is not None and t.device != feat.device:
            bad("feat, n_rows, y and y_valid must be on one device")


class TraversabilityEstimator:
    def __init__(self, params=None, device: str = "cuda", max_distance: float = 3, image_distance_thr: float = None,
                 supervision_distance_thr: float = None, min_samples_for_training: int = 10, vis_node_index: int = 10,
                 mode=None, extraction_store_folder=None, anomaly_detection: bool = False, process_group=None,
                 max_rows: int = 4096, mission_graph_capacity: int = 256, mission_graph_smax: int = None):
        if process_group is not None and not isinstance(process_group, torch.distributed.ProcessGroup):
            raise ValueError(f"process_group must be a torch.distributed.ProcessGroup, got {type(process_group).__name__}")
        self._device = device
        self._mode = mode
        self._extraction_store_folder = extraction_store_folder
        self._min_samples_for_training = min_samples_for_training
        self._vis_node_index = vis_node_index
        self._params = params if params is not None else default_params(anomaly_detection)
        self._anomaly_detection = anomaly_detection
        self._mission_nodes = []
        # the device mission graph is made by the first node that carries camera data (its image size fixes the slots)
        self._mission_graph = None
        self._mission_graph_capacity, self._mission_graph_smax = mission_graph_capacity, mission_graph_smax
        self._image_distance_thr, self._max_distance = image_distance_thr, max_distance
        self._supervision_graph = DistanceWindowGraph(edge_distance=supervision_distance_thr, max_distance=max_distance)
        self._learning_lock = Lock()
        self._pause_training = False

        torch.manual_seed(42)  # seed_everything(42) (:78) — same init as the reference's get_model
        random.seed(42)
        model_cfg = _get(self._params, "model")
        if anomaly_detection != (_get(model_cfg, "name") == "LinearRnvp"):
            raise ValueError("anomaly_detection=True goes with model.name 'LinearRnvp' (and only with it), got "
                             f"{_get(model_cfg, 'name')!r}")
        self._double = _get(model_cfg, "name") == "DoubleMLP"
        self._model = get_model(model_cfg).to(self._device)
        self._model.train()
        gp = _get(self._params, "general")
        self._lr = float(_get(_get(self._params, "optimizer"), "lr"))
        self._loss = torch.tensor([torch.inf])
        self._step = 0
        self._last_confidence = None
        if anomaly_detection:
            la = dict(_get(self._params, "loss_anomaly"))
            self._traversability_loss = AnomalyLoss(**la, log_enabled=_get(gp, "log_confidence"),
                                                    log_folder=_get(gp, "model_path"))
            self._traversability_loss.to(self._device)
            cg = self._traversability_loss._confidence_generator
            self._trainer = ops.FlowTrainer(self._model, max_rows=max_rows, std_factor=cg.std_factor, lr=self._lr,
                                            process_group=process_group)
            self._bind_confidence_state()
            return
        lp = dict(_get(self._params, "loss"))
        self._traversability_loss = TraversabilityLoss(
            **lp, model=self._model, log_enabled=_get(gp, "log_confidence"), log_folder=_get(gp, "model_path"))
        self._traversability_loss.to(self._device)
        m = self._model
        cg = self._traversability_loss._confidence_generator
        if self._double:
            self._trainer = ops.DoubleMlpTrainer(m, max_rows=max_rows, w_trav=lp["w_trav"], w_reco=lp["w_reco"],
                                                 std_factor=cg.std_factor, anomaly_balanced=lp["anomaly_balanced"],
                                                 lr=self._lr, process_group=process_group)
            self._bind_confidence_state()
            return
        self._trainer = ops.MlpTrainer(m.flat_params, m.input_size, m.hidden[0], m.hidden[1], max_rows=max_rows,
                                       w_trav=lp["w_trav"], w_reco=lp["w_reco"], std_factor=cg.std_factor,
                                       anomaly_balanced=lp["anomaly_balanced"], lr=self._lr, process_group=process_group)
        self._bind_confidence_state()

    def _bind_confidence_state(self):
        """Points the fused step at the ConfidenceGenerator's own parameters (mean / std / var / running sums), so the
        module's ``state_dict`` is always current without a copy or a host round trip."""
        cg = self._traversability_loss._confidence_generator
        kf = getattr(cg, "_kalman_filter", None)
        self._trainer.cg_mean, self._trainer.cg_std = cg.mean.data, cg.std.data
        self._trainer.set_confidence(
            cg.method_id, cg.var.data, getattr(cg, "running_n", None), getattr(cg, "running_sum", None),
            getattr(cg, "running_sum_of_squares", None),
            kf_proc_cov=float(kf.proc_cov.item()) if kf is not None else 0.2,
            kf_meas_cov=float(kf.meas_cov.item()) if kf is not None else 1.0)

    # ---- properties ------------------------------------------------------------------------
    @property
    def loss(self):
        return float(self._loss) if not torch.is_tensor(self._loss) else self._loss.detach().item()

    @property
    def step(self):
        return self._step

    @property
    def pause_learning(self):
        return self._pause_training

    @pause_learning.setter
    def pause_learning(self, pause: bool):
        self._pause_training = pause

    def change_device(self, device):
        if torch.device(device) != torch.device(self._device):
            raise RuntimeError("device changes after construction are not supported (buffers are device-bound)")

    # ---- nodes -----------------------------------------------------------------------------
    def add_mission_node(self, node, verbose: bool = False):
        """A node with camera data (``features``, ``feature_segments``, ``pose_cam_in_world``, ``image_projector`` or
        ``K``, ``timestamp``; the reference's ``MissionNode`` has them) goes into the device mission graph, gated by
        ``image_distance_thr`` (traversability_estimator.py:166-196): returns True when it was added for training.
        Any other node (``MissionNode`` above, labels already pooled) is appended to the plain list, as before."""
        if getattr(node, "feature_segments", None) is None or getattr(node, "pose_cam_in_world", None) is None:
            self._mission_nodes.append(node)
            return True
        seg, feat = node.feature_segments, node.features
        K = getattr(node, "K", None)
        if K is None:
            K = node.image_projector.camera.intrinsics
        K = K.reshape(-1, 4, 4)[0]
        g = self._graph_for(seg.shape[-2], seg.shape[-1], feat.shape[0])
        train = bool(getattr(node, "use_for_training", True))
        added = g.add(feat, seg, K, node.pose_cam_in_world, float(node.timestamp),
                      getattr(node, "pose_base_in_world", node.pose_cam_in_world), has_mask=train)
        if added is not None and train and verbose:
            print(f"adding node [{added}], total nodes [{g.get_num_nodes()}]")
        return added is not None and train

    def add_mission_frames(self, r, poses, K, timestamps, pose_cam_in_base=None):
        """Adds a batch of frames straight from ``FeatureExtractor.extract_batch`` (``r``: seg [B,H,W], feat [B,S,D],
        n_segments [B] on the device) to the device mission graph, device to device, each gated by
        ``image_distance_thr`` like ``add_mission_node``.  ``poses``: [B,4,4] base poses in the world (host);
        ``pose_cam_in_base``: [4,4] or [B,4,4] (default identity); ``K``: the scaled [4,4] or [B,4,4] camera matrices
        of the H x W segmentation; ``timestamps``: B floats.  Returns the number of frames added."""
        if r.get("n_segments") is None:
            raise ValueError("add_mission_frames needs per-segment features (extract_batch with a segmentation)")
        poses = torch.as_tensor(poses, dtype=torch.float32).cpu()
        cam = poses if pose_cam_in_base is None else poses @ torch.as_tensor(pose_cam_in_base, dtype=torch.float32).cpu()
        seg, feat = r["seg"], r["feat"]
        g = self._graph_for(seg.shape[-2], seg.shape[-1], feat.shape[1])
        return len(g.add_frames(feat, r["n_segments"], seg, K, cam, [float(t) for t in timestamps], poses))

    def _graph_for(self, h, w, rows):
        g = self._mission_graph
        if g is None:
            smax = self._mission_graph_smax or max(256, (int(rows) + 63) // 64 * 64)
            g = MissionGraph(self._mission_graph_capacity, int(h), int(w), smax, self._model.input_size,
                             device=self._device, edge_distance=self._image_distance_thr, max_distance=self._max_distance)
            self._mission_graph = g
        return g

    def add_supervision_node(self, pnode):
        """One footprint event (traversability_estimator.py:199-300): the supervision graph's edge gate (a node that is
        too close only lowers the last node's traversability, pessimistically), the footprint between this node and the
        last one, the 30 s mask sweep, the range query along the mission graph, then one ``wvn_mission_propagate`` launch
        that renders, fmin-s and re-pools every in-range node's labels.  Host math on a few points, no device-to-host
        copy.  Returns True when labels were propagated."""
        if not pnode.is_valid():
            return False
        last_pnode = self._supervision_graph.get_last_node()
        if not self._supervision_graph.add_node(pnode):
            if last_pnode is not None:
                last_pnode.update_traversability(pnode.traversability, pnode.traversability_var)
            return False
        if last_pnode is None or not last_pnode.is_valid():
            return False
        footprint = footprint_between(pnode, last_pnode)
        g = self._mission_graph
        last = g.get_last_node() if g is not None else None
        if last is None or not last.has_mask:
            return False
        g.sweep(last.timestamp)
        nodes = g.get_nodes_within_radius_range(self._supervision_graph.max_distance)
        if len(nodes) < 1:
            return False
        g.propagate(nodes, footprint, pnode.traversability)
        return True

    def get_mission_nodes(self):
        return self._mission_graph.get_nodes() if self._mission_graph is not None else self._mission_nodes

    def get_supervision_nodes(self):
        return self._supervision_graph.get_nodes()

    def get_num_valid_nodes(self):
        if self._mission_graph is not None:
            return self._mission_graph.get_num_valid_nodes()
        return sum(1 for n in self._mission_nodes if n.is_valid())

    def make_batch(self, batch_size: int = 8):
        """Samples ``batch_size`` random valid nodes (graphs.py:137-143) and concatenates them (utils/data.py:22-58)."""
        nodes = [n for n in self._mission_nodes if n.is_valid()]
        random.shuffle(nodes)
        return Batch.from_data_list([n.as_pyg_data(self._anomaly_detection) for n in nodes[:batch_size]])

    # ---- the train step ----------------------------------------------------------------------
    def train_on_batch(self, graph, n_total=None):
        """forward + TraversabilityLoss + backward + Adam on ``graph`` (x, y, y_valid).  Metrics stay
        on the device in ``self._trainer.metrics``; returns the per-row confidence."""
        with self._learning_lock:
            if self._anomaly_detection:   # AnomalyLoss: the flow's step on the labelled rows of the batch
                conf = self._trainer.step(graph.x, graph.y_valid)
            else:
                conf = self._trainer.step(graph.x, graph.y, graph.y_valid, n_total=n_total)
            self._last_confidence = conf
        self._step += 1
        return conf

    def train_on_padded(self, feat, n_rows, y, y_valid):
        """The same step on rows that are still padded per frame, as ``FeatureExtractor.extract_batch`` returns them:
        ``feat`` (B, smax, D) float32, ``n_rows`` (B,) int32 on the device; ``y`` (float) / ``y_valid`` (bool or uint8)
        are 1-D and indexed by the compacted row number (what ``feat[mask]`` would give).  No host synchronisation (the
        gather happens inside the kernels).  In anomaly-detection mode the flow learns from the rows ``y_valid`` sets
        and ignores ``y`` (it may be None); the returned confidences are those rows', in order."""
        _check_padded_args(feat, n_rows, y, y_valid, self._model.input_size, y_optional=self._anomaly_detection)
        with self._learning_lock:
            conf = self._trainer.step_padded(feat, n_rows, y, y_valid)
            self._last_confidence = conf
        self._step += 1
        return conf

    def train(self):
        """One step of the training loop; same gating and return dict as the reference (:448-497).  With a device
        mission graph the batch is sampled from it (sorted valid nodes, ``random.shuffle``, the first ``batch_size``)
        and trained in the padded layout; reading the valid flags and row counts is one small device-to-host copy."""
        if self._pause_training:
            return {}
        num_valid_nodes = self.get_num_valid_nodes()
        return_dict = {"mission_graph_num_valid_node": num_valid_nodes}
        if num_valid_nodes > self._min_samples_for_training:
            bs = _get(_get(self._params, "ablation_data_module"), "batch_size")
            if self._mission_graph is not None:
                g = self._mission_graph
                self.last_sampled_nodes = g.get_n_random_valid_nodes(n=bs)
                self.train_on_padded(*g.gather(self.last_sampled_nodes))
                graph = True
            else:
                graph = self.make_batch(bs)
                if graph is not None:
                    self.train_on_batch(graph)
            if graph is not None:
                log_step = ((self._step - 1) % 20) == 0
                m = self._trainer.metrics.tolist()  # the reference's three .item() calls, as one D2H copy
                self._loss = torch.tensor(m[0])
                if log_step:
                    print(f"step: {self._step - 1} | loss: {m[0]:5f} | loss_trav: {m[1]:5f} | loss_reco: {m[2]:5f}")
                return_dict["loss_total"] = m[0]
                return_dict["loss_trav"] = m[1]
                return_dict["loss_reco"] = m[2]
                return return_dict
        return_dict["loss_total"] = -1
        return return_dict

    # ---- checkpoints (same on-disk format as the reference, :377-429) --------------------------
    def _optimizer_params(self):
        """The tensors torch.optim.Adam(model.parameters()) would hold, in its order."""
        return list(self._model.parameters())

    def _optimizer_state_dict(self):
        tr, off, state = self._trainer, 0, {}
        for i, p in enumerate(self._optimizer_params()):
            n = p.numel()
            state[i] = {"step": tr.step_counter.float().cpu().reshape(()).clone(),
                        "exp_avg": tr.exp_avg[off : off + n].view_as(p).clone(),
                        "exp_avg_sq": tr.exp_avg_sq[off : off + n].view_as(p).clone()}
            off += n
        group = {"lr": self._lr, "betas": (0.9, 0.999), "eps": 1e-08, "weight_decay": 0, "amsgrad": False,
                 "maximize": False, "foreach": None, "capturable": False, "differentiable": False, "fused": None,
                 "params": list(range(len(state)))}
        return {"state": state, "param_groups": [group]}

    def _load_optimizer_state_dict(self, sd):
        tr, off = self._trainer, 0
        for i, p in enumerate(self._optimizer_params()):
            n = p.numel()
            st = sd["state"].get(i)
            if st is not None:
                tr.exp_avg[off : off + n] = st["exp_avg"].reshape(-1).to(tr.exp_avg.device)
                tr.exp_avg_sq[off : off + n] = st["exp_avg_sq"].reshape(-1).to(tr.exp_avg.device)
                tr.step_counter.fill_(int(st["step"]))
            off += n

    def write_model_handoff(self, path: str) -> str:
        """The learner's side of the weight hand-off (wvn_learning_node.py:381-394): ``.tmp_state_dict.pt``."""
        from ..utils.handoff import write_tmp_state_dict

        with self._learning_lock:
            return write_tmp_state_dict(self._model, self._traversability_loss._confidence_generator, path)

    def save_checkpoint(self, mission_path: str, checkpoint_name: str = "last_checkpoint.pt"):
        with self._learning_lock:
            self._pause_training = True
            os.makedirs(mission_path, exist_ok=True)
            checkpoint_file = os.path.join(mission_path, checkpoint_name)
            torch.save({"step": self._step, "model_state_dict": self._model.state_dict(),
                        "optimizer_state_dict": self._optimizer_state_dict(),
                        "traversability_loss_state_dict": self._traversability_loss.state_dict(),
                        "loss": self.loss}, checkpoint_file)
            print(f"Saved checkpoint to file {checkpoint_file}")
            self._pause_training = False

    def load_checkpoint(self, checkpoint_path: str):
        with self._learning_lock:
            self._pause_training = True
            checkpoint = torch.load(checkpoint_path, map_location=self._device, weights_only=False)  # trusted mission file
            self._model.load_state_dict(checkpoint["model_state_dict"])
            self._load_optimizer_state_dict(checkpoint["optimizer_state_dict"])
            self._traversability_loss.load_state_dict(checkpoint["traversability_loss_state_dict"])
            self._step = checkpoint["step"]
            self._loss = torch.tensor(checkpoint["loss"])
            self._model.train()
            print(f"Loaded checkpoint from file {checkpoint_path}")
            self._pause_training = False
