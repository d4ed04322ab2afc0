"""TraversabilityEstimator — the online learner
(reference: wild_visual_navigation/traversability_estimator/traversability_estimator.py:33-505).

On the hot path and implemented: ``__init__`` (seed 42, SimpleMLP, TraversabilityLoss, Adam —
:78-105), ``make_batch`` (:431-446), ``train`` (:448-497, same return dict), ``save_checkpoint`` /
``load_checkpoint`` (:377-429, same file format incl. a torch.optim.Adam-compatible
``optimizer_state_dict``), ``pause_learning`` / ``step`` / ``loss``.
The mission / supervision graphs (networkx + liegroups, nodes.py / graphs.py), footprint
projection and visualisation are OUT OF SCOPE (SURVEY.md §2): mission nodes are kept in a plain
list and must already carry their per-segment features and supervision (``MissionNode``).

``train()`` runs forward + loss + backward + Adam as one fixed sequence of fp32 CUDA kernels
(csrc/mlp_train.cu) with all scalars on the device; with a ``process_group`` the three confidence
statistics and the flat gradient are all-reduced (NCCL over NVLink) for a global-batch step.
"""
from __future__ import annotations

import os
import random
from threading import Lock

import torch

from .. import ops
from ..model import get_model
from ..utils import Batch, Data, TraversabilityLoss


def default_params():
    """The defaults of ``ExperimentParams`` that define the hot path (cfg/experiment_params.py:44-56,91,104-112)."""
    return {
        "model": {"name": "SimpleMLP",
                  "simple_mlp_cfg": {"input_size": 384, "hidden_sizes": [256, 32, 1], "reconstruction": True}},
        "loss": {"anomaly_balanced": True, "w_trav": 0.03, "w_temp": 0.0, "w_reco": 0.5, "method": "latest_measurement",
                 "confidence_std_factor": 0.5, "trav_cross_entropy": False},
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
        return Data(x=self.features, y=self.supervision_signal, y_valid=self.supervision_signal_valid)


def _get(p, key):
    return p[key] if isinstance(p, dict) else getattr(p, key)


class TraversabilityEstimator:
    def __init__(self, params=None, device: str = "cuda", max_distance: float = 3, image_distance_thr: float = None,
                 supervision_distance_thr: float = None, min_samples_for_training: int = 10, vis_node_index: int = 10,
                 mode=None, extraction_store_folder=None, anomaly_detection: bool = False, process_group=None,
                 max_rows: int = 4096):
        if anomaly_detection:
            raise ValueError("anomaly_detection (LinearRnvp) is outside the H100 hot path")
        self._device = device
        self._mode = mode
        self._extraction_store_folder = extraction_store_folder
        self._min_samples_for_training = min_samples_for_training
        self._vis_node_index = vis_node_index
        self._params = params if params is not None else default_params()
        self._anomaly_detection = anomaly_detection
        self._mission_nodes = []
        self._learning_lock = Lock()
        self._pause_training = False

        torch.manual_seed(42)  # seed_everything(42) (:78) — same init as the reference's get_model
        random.seed(42)
        self._model = get_model(_get(self._params, "model")).to(self._device)
        self._model.train()
        lp = dict(_get(self._params, "loss"))
        gp = _get(self._params, "general")
        self._traversability_loss = TraversabilityLoss(
            **lp, model=self._model, log_enabled=_get(gp, "log_confidence"), log_folder=_get(gp, "model_path"))
        self._traversability_loss.to(self._device)
        self._lr = float(_get(_get(self._params, "optimizer"), "lr"))
        m = self._model
        cg = self._traversability_loss._confidence_generator
        self._trainer = ops.MlpTrainer(m.flat_params, m.input_size, m.hidden[0], m.hidden[1], max_rows=max_rows,
                                       w_trav=lp["w_trav"], w_reco=lp["w_reco"], std_factor=cg.std_factor,
                                       anomaly_balanced=lp["anomaly_balanced"], lr=self._lr, process_group=process_group)
        # the train step writes the ConfidenceGenerator's mean / std straight into the module's parameters
        self._trainer.cg_mean, self._trainer.cg_std = cg.mean.data, cg.std.data
        self._bind_confidence_state()
        self._loss = torch.tensor([torch.inf])
        self._step = 0
        self._last_confidence = None

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
    def add_mission_node(self, node: MissionNode, verbose: bool = False):
        self._mission_nodes.append(node)
        return True

    def get_mission_nodes(self):
        return self._mission_nodes

    def get_num_valid_nodes(self):
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
            conf = self._trainer.step(graph.x, graph.y, graph.y_valid, n_total=n_total)
            self._last_confidence = conf
        self._step += 1
        return conf

    def train_on_padded(self, feat, n_rows, y, y_valid):
        """The same step on rows that are still padded per frame, as ``FeatureExtractor.extract_batch`` returns them:
        ``feat`` (B, smax, D), ``n_rows`` (B,) int32 on the device; ``y`` / ``y_valid`` are indexed by the compacted row
        number (what ``feat[mask]`` would give).  No host synchronisation (the gather happens inside the kernels)."""
        with self._learning_lock:
            conf = self._trainer.step_padded(feat, n_rows, y, y_valid)
            self._last_confidence = conf
        self._step += 1
        return conf

    def train(self):
        """One step of the training loop; same gating and return dict as the reference (:448-497)."""
        if self._pause_training:
            return {}
        num_valid_nodes = self.get_num_valid_nodes()
        return_dict = {"mission_graph_num_valid_node": num_valid_nodes}
        if num_valid_nodes > self._min_samples_for_training:
            graph = self.make_batch(_get(_get(self._params, "ablation_data_module"), "batch_size"))
            if graph is not None:
                log_step = (self._step % 20) == 0
                self.train_on_batch(graph)
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
    def _optimizer_state_dict(self):
        tr, off, state = self._trainer, 0, {}
        for i, p in enumerate(self._model.layers.parameters()):
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
        for i, p in enumerate(self._model.layers.parameters()):
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
