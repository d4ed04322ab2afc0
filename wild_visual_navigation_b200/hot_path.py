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
traversability and confidence on the frame's graph, painted through ``seg`` on the device.

Front ends.  ``segmentation_type`` is "stego" (the default), "slic" or "grid" (``slic_num_components`` / ``cell_size``
go to ``FeatureExtractor``); "random" and "none" are refused, because the node's ``feat[seg]`` reads row -1 for
unpicked pixels and a pixel-wise graph has one row per pixel.  ``feature_type="torchvision"`` with ``model_type``
(resnet18, resnet50, resnet50_dino, efficientnet_b0) runs a feature pyramid.  Its weights come from
``backbone_state_dict`` or ``pretrained_weights``; ``state_dict`` / ``head_state_dict`` stay STEGO's DINO backbone and
head, which segment the frames when ``segmentation_type="stego"`` (``FeatureExtractor``'s ``stego_state_dict``).

``prediction_per_pixel`` is the node's parameter of that name.  With False, or with a SimpleGCN, the maps are
segment-wise (wvn_feature_extractor_node.py:323-338): each pooled row is evaluated once (padded-row inference with the
device-side counts) and its values are painted through ``seg``.  The node evaluates the same row at every pixel of the
segment, so the maps are the same.  A feature pyramid has no per-pixel head, so there ``prediction_per_pixel`` must be
False.  Every configuration runs without host synchronisation and captures in a CUDA graph.
"""
from __future__ import annotations

import torch

from .feature_extractor import FeatureExtractor
from .inference import TraversabilityInference
from .traversability_estimator import TraversabilityEstimator


SEGMENTATION_TYPES = ("stego", "slic", "grid")


class HotPathStep:
    def __init__(self, device: str, state_dict, head_state_dict, batch: int = 32, input_size: int = 448,
                 backbone_type: str = "vit_small", patch_size: int = 8, chunk: int = 32, flip_tta: bool = False,
                 run_clustering: bool = True, n_image_clusters: int = 20, process_group=None, feature_type: str = "dino",
                 model: str = "SimpleMLP", anomaly_detection: bool = False, segmentation_type: str = "stego",
                 prediction_per_pixel: bool = True, model_type: str = None, backbone_state_dict=None,
                 pretrained_weights: str = None, slic_num_components: int = 100, cell_size: int = 32):
        if segmentation_type not in SEGMENTATION_TYPES:
            raise ValueError(f"HotPathStep: segmentation_type must be one of {SEGMENTATION_TYPES}, got "
                             f"{segmentation_type!r}")
        pyramid = feature_type == "torchvision"
        if pyramid:
            if model_type is None:
                raise ValueError("HotPathStep: feature_type='torchvision' needs model_type ('resnet18', 'resnet50', "
                                 "'resnet50_dino' or 'efficientnet_b0')")
            if prediction_per_pixel:
                raise ValueError("HotPathStep: a feature-pyramid backbone has no per-pixel head (the reference defines "
                                 "none); pass prediction_per_pixel=False for segment-wise maps")
        elif model_type is not None or backbone_state_dict is not None or pretrained_weights is not None:
            raise ValueError("HotPathStep: model_type, backbone_state_dict and pretrained_weights select the "
                             "feature_type='torchvision' trunk")
        self.device, self.batch, self.input_size = device, batch, input_size
        self.per_pixel = prediction_per_pixel
        fe_args = dict(head_state_dict=head_state_dict, flip_tta=flip_tta, run_clustering=run_clustering,
                       n_image_clusters=n_image_clusters, max_batch=batch, chunk=chunk, backbone_type=backbone_type,
                       patch_size=patch_size, slic_num_components=slic_num_components, cell_size=cell_size)
        if pyramid:   # the trunk's own weights; STEGO (when it segments) keeps state_dict
            fe_args.update(model_type=model_type, state_dict=backbone_state_dict, pretrained_weights=pretrained_weights,
                           stego_state_dict=state_dict)
        else:
            fe_args.update(state_dict=state_dict)
        self.fe = FeatureExtractor(device, segmentation_type=segmentation_type, feature_type=feature_type,
                                   input_size=input_size, **fe_args)
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
        self.ti = TraversabilityInference(self.fe._tv if pyramid else self.fe._dino, self.te._model, self.cg,
                                          max_rows=batch * self.smax)

    @torch.no_grad()
    def step(self, img: torch.Tensor, y: torch.Tensor, y_valid: torch.Tensor) -> dict:
        """img: (B,3,H,W) float in [0,1] or (B,H0,W0,3) uint8 camera frames; y / y_valid: supervision of the pooled
        rows in compacted order (frame 0's segments, then frame 1's, ...), at least B*smax entries.
        Returns the extract_batch dict plus ``trav`` / ``conf`` (B,H,H) and ``confidence_rows``.  ``confidence_rows``
        holds one confidence per live row in compacted order; for the LinearRnvp flow it holds the labelled rows'
        (those ``y_valid`` sets), in order, and ``conf`` is None (the node publishes no confidence map there)."""
        r = self.fe.extract_batch(img)                                        # backbone + segmentation + pooling + graph
        if self.gcn or not self.per_pixel:
            # segment-wise maps: each pooled row once (the SimpleGCN on its frame's graph), painted through seg
            trav, conf = self.ti.predict_frames(r["feat"], r["n_segments"], r["edges"], r["n_edges"], r["seg"])
            crow = self.te.train_on_padded(r["feat"], r["n_segments"], y, y_valid, edges=r["edges"],
                                           n_edges=r["n_edges"])               # the edges: read by the SimpleGCN only
            self.ti.refresh_weights()                                          # a no-op for the SimpleGCN
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

