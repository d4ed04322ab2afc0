"""One pass of the whole hot path over a batch of frames — what the two ROS nodes do for every camera frame.

feature node  (wild_visual_navigation_ros/scripts/wvn_feature_extractor_node.py:306-393):
    ``FeatureExtractor.extract`` (ViT -> STEGO segmentation -> per-segment pooling, centroids, adjacency) and the
    per-pixel traversability / confidence maps from the current MLP;
learning node (wvn_learning_node.py:651-656 + traversability_estimator.py:448-497):
    one ``TraversabilityEstimator.train`` step on the pooled rows of those frames, after which the inference side picks up
    the new weights (``load_model``, wvn_feature_extractor_node.py:407-450).

``bench.py`` times exactly ``HotPathStep.step`` and ``tests/test_bench_path_gpu.py`` holds it to the oracle, so the
benchmarked configuration and the tested one are the same object.  The step has no host synchronisation: the pooled
rows go to the trainer padded per frame with their device-side counts (csrc/mlp_train_fused.cu).

``model`` / ``anomaly_detection`` pick the learner as the nodes' ``model.name`` does: SimpleMLP (the default),
DoubleMLP, SimpleGCN, or with ``anomaly_detection=True`` the LinearRnvp flow; each is built with ``input_size`` = the
backbone's feature dimension and trains on the same padded rows, data-parallel with ``process_group``.  The SimpleGCN
also reads each frame's segment adjacency (``edges`` / ``n_edges``), and its maps are segment-wise: the per-segment
traversability and confidence on the frame's graph, scattered through ``seg`` on the device.
"""
from __future__ import annotations

import torch

from .feature_extractor import FeatureExtractor
from .inference import TraversabilityInference
from .traversability_estimator import TraversabilityEstimator


class HotPathStep:
    def __init__(self, device: str, state_dict, head_state_dict, batch: int = 32, input_size: int = 448,
                 backbone_type: str = "vit_small", patch_size: int = 8, chunk: int = 32, flip_tta: bool = False,
                 run_clustering: bool = True, n_image_clusters: int = 20, process_group=None, feature_type: str = "dino",
                 model: str = "SimpleMLP", anomaly_detection: bool = False):
        self.device, self.batch, self.input_size = device, batch, input_size
        self.fe = FeatureExtractor(device, segmentation_type="stego", feature_type=feature_type, input_size=input_size,
                                   state_dict=state_dict, head_state_dict=head_state_dict, flip_tta=flip_tta,
                                   run_clustering=run_clustering, n_image_clusters=n_image_clusters, max_batch=batch,
                                   chunk=chunk, backbone_type=backbone_type, patch_size=patch_size)
        self.smax = self.fe.max_segments
        if model not in ("SimpleMLP", "DoubleMLP", "SimpleGCN"):
            raise ValueError(f"HotPathStep: model must be 'SimpleMLP', 'DoubleMLP' or 'SimpleGCN', got {model!r}")
        self.gcn = model == "SimpleGCN"
        if anomaly_detection and model != "SimpleMLP":
            raise ValueError("HotPathStep: anomaly_detection=True selects the LinearRnvp learner; leave model at its default")
        params = None
        if self.fe.feature_dim != 384 or model != "SimpleMLP" or anomaly_detection:
            from .traversability_estimator.traversability_estimator import default_params

            params = default_params(anomaly_detection)
            if model != "SimpleMLP":
                params["model"]["name"] = model
            cfg = {"SimpleMLP": "simple_mlp_cfg", "DoubleMLP": "double_mlp_cfg", "SimpleGCN": "simple_gcn_cfg"}[model]
            params["model"]["linear_rnvp_cfg" if anomaly_detection else cfg]["input_size"] = self.fe.feature_dim
        self.te = TraversabilityEstimator(params=params, device=device, process_group=process_group,
                                          max_rows=batch * self.smax, anomaly_detection=anomaly_detection)
        self.cg = self.te._traversability_loss._confidence_generator
        self.ti = TraversabilityInference(self.fe._dino, self.te._model, self.cg)

    @torch.no_grad()
    def step(self, img: torch.Tensor, y: torch.Tensor, y_valid: torch.Tensor) -> dict:
        """img: (B,3,H,W) float in [0,1] or (B,H0,W0,3) uint8 camera frames; y / y_valid: supervision of the pooled
        rows in compacted order (frame 0's segments, then frame 1's, ...), at least B*smax entries.
        Returns the extract_batch dict plus ``trav`` / ``conf`` (B,H,H) and ``confidence_rows``.  ``confidence_rows``
        holds one confidence per live row in compacted order; for the LinearRnvp flow it holds the labelled rows'
        (those ``y_valid`` sets), in order, and ``conf`` is None (the node publishes no confidence map there)."""
        r = self.fe.extract_batch(img)                                        # ViT + STEGO seg + pooling + graph
        if self.gcn:   # segment-wise maps on each frame's graph; the step trains on the same rows and edges
            trav, conf = self.ti.predict_frames(r["feat"], r["n_segments"], r["edges"], r["n_edges"], r["seg"])
            crow = self.te.train_on_padded(r["feat"], r["n_segments"], y, y_valid, edges=r["edges"],
                                           n_edges=r["n_edges"])
            r["trav"], r["conf"], r["confidence_rows"] = trav, conf, crow
            return r
        trav, conf = self.ti.predict_from_tokens(r["tokens"], self.input_size)   # per-pixel MLP -> maps
        crow = self.te.train_on_padded(r["feat"], r["n_segments"], y, y_valid)  # fwd + loss + bwd + (all-reduce) + Adam
        self.ti.refresh_weights()                                              # inference sees the updated MLP
        r["trav"], r["conf"], r["confidence_rows"] = trav, conf, crow
        return r

    # ---- CUDA-graph replay of the whole step (the deployment case: one camera frame at a time, where ~120 launches per
    # frame are launch-latency bound).  Everything the step enqueues — the library's kernels, its memsets and the few
    # torch glue ops — is capturable: no host synchronisation, no allocation inside the library after create.
    def capture(self, img: torch.Tensor, y: torch.Tensor, y_valid: torch.Tensor, warmup: int = 2):
        """Captures ``step`` for inputs of this shape; afterwards ``replay(img)`` re-runs it on new frames."""
        self._g_img, self._g_y, self._g_yv = img.clone(), y.clone(), y_valid.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self.step(self._g_img, self._g_y, self._g_yv)
        torch.cuda.current_stream().wait_stream(side)
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph):
            self._g_out = self.step(self._g_img, self._g_y, self._g_yv)
        return self._g_out

    def replay(self, img: torch.Tensor, y: torch.Tensor = None, y_valid: torch.Tensor = None) -> dict:
        """New frames (and optionally labels) through the captured step; returns the same (static) output tensors."""
        self._g_img.copy_(img, non_blocking=True)
        if y is not None:
            self._g_y.copy_(y, non_blocking=True)
            self._g_yv.copy_(y_valid, non_blocking=True)
        self._graph.replay()
        self.te._step += 1
        return self._g_out

