"""Per-frame traversability inference — the arithmetic of ``WvnFeatureExtractor.image_callback``
(reference: wild_visual_navigation_ros/scripts/wvn_feature_extractor_node.py:306-370) and of
``quick_start.py:174-214`` without ROS:

    dense_feat = feature_extractor.extract(img, return_dense_features=True)
    x = dense_feat[0].permute(1,2,0).reshape(-1, D);  prediction = model.forward(Data(x=x))
    out_trav = prediction.reshape(H,W,-1)[:,:,0]
    loss_reco = mse(prediction[:,1:], x).mean(1);  confidence = cg.inference_without_update(loss_reco)

fused as: ViT tokens -> (bilinear sample -> 3 wgmma GEMMs -> sigmoid / reco-loss / confidence
epilogue) per pixel; neither ``dense_feat`` (308 MB/frame) nor the (P, 385) prediction is stored.

In anomaly-detection mode (a ``LinearRnvp`` model, wvn_feature_extractor_node.py:332-338) traversability is the
generator's ``inference_without_update`` of the per-row NLL and there is no confidence map (the node forces
``publish_confidence = False``): per pixel, the tokens are upsampled in a sampling kernel and every layer of the four
nets runs as a wgmma GEMM (bf16 operands, fp32 accumulation) over chunks of pixels, with the coupling arithmetic, NLL and
confidence in fp32 kernels (csrc/flow_train.cu); ``predict_segments`` runs the fp32 flow on the pooled rows.

A ``DoubleMLP`` runs through the same MLP handle.  Per pixel, for h1 in {64, 128} and h2 = 32, the fused head's
DoubleMLP instantiation (csrc/pixel_head.cu: G of both networks interpolated, layer 2 as one wgmma chain per network);
other shapes, and ``predict_segments``, run the two networks packed as one block-structured MLP (layer 1 both nets'
rows, layer 2 block-diagonal, layer 3 the traversability row on net 0's half and the reconstruction rows on net 1's)
through the unfused GEMM chain.

A ``SimpleGCN`` predicts segment-wise only (``predict_segments`` with the frame's segment adjacency, csrc/gcn_train.cu):
there is no graph over pixels, so ``predict`` / ``predict_from_tokens`` raise ``ValueError`` (the reference's node
builds ``Data(x=...)`` without ``edge_index`` and cannot run a GCN either).

Segment-wise mode (``prediction_per_pixel: False``, wvn_feature_extractor_node.py:323-338): the node runs the model on
``feat[seg.reshape(-1)]``, every pixel carrying its segment's pooled row, so it evaluates each row once per pixel of
the segment.  ``predict_frames`` evaluates each pooled row once, for a whole batch as ``extract_batch`` leaves it
(rows padded per frame, device-side counts), and paints the values through ``seg`` (csrc/segment_kernels.cu); it works
for every learner and never synchronises with the host.  The front end passed in may be a ``DinoInterface``, a
``StegoInterface`` (its DINO backbone gives the token grid), a ``TorchVisionInterface`` or ``None``.  A feature pyramid
has no token grid and the reference defines no per-pixel head on it (its per-pixel branch indexes ``dense_feat[0]`` of
the pyramid dict and crashes), so there ``predict`` / ``predict_from_tokens`` raise ``ValueError``.
"""
from __future__ import annotations

import torch

from . import ops
from .feature_extractor.stego_interface import StegoInterface
from .feature_extractor.torchvision_interface import TorchVisionInterface
from .model.linear_rnvp import LinearRnvp
from .model.simple_gcn import SimpleGCN
from .model.simple_mlp import DoubleMLP, SimpleMLP
from .utils.confidence_generator import ConfidenceGenerator


class TraversabilityInference:
    """``frontend``: the feature front end whose tokens the per-pixel calls read — a ``DinoInterface``, a
    ``StegoInterface`` (its DINO backbone), a ``TorchVisionInterface`` (segment-wise only) or ``None`` (segment-wise
    only).  ``max_rows``: padded rows per ``predict_frames`` call (max_batch * smax) the handles are sized for at
    construction, so that call allocates nothing in the library."""

    def __init__(self, frontend, model: SimpleMLP, confidence_generator: ConfidenceGenerator, chunk_rows: int = 0,
                 max_rows: int = 1024):
        self._pyramid = isinstance(frontend, TorchVisionInterface)
        if isinstance(frontend, StegoInterface):
            frontend = frontend._dino
        dino = None if self._pyramid else frontend   # the token grid of the per-pixel calls, if there is one
        self._gcn = isinstance(model, SimpleGCN)
        if self._gcn:
            model.check_supported()
            self._dino, self._model, self._cg = dino, model, confidence_generator
            self._gcn_infer = ops.GcnInference(model, max_rows=max(1024, max_rows))
            self._flow = self._double = False
            return
        self._flow = isinstance(model, LinearRnvp)
        if self._flow:
            if model.flat_params is None or not model.flat_params.is_cuda:
                raise ValueError("TraversabilityInference: the LinearRnvp must be on a CUDA device")
            self._dino, self._model, self._cg = dino, model, confidence_generator
            self._flow_infer = ops.FlowInference(model.input_size, model.hidden, max_rows=max(1024, max_rows),
                                                 chunk_pixels=chunk_rows)
            self.refresh_weights()
            return
        self._double = isinstance(model, DoubleMLP)
        if self._double:
            model.check_supported()
        else:
            assert model.fused_ok(), "model must be the hot-path SimpleMLP(D,[256,32,1],reconstruction=True) on CUDA"
        self._dino = dino
        self._model = model
        self._cg = confidence_generator
        # a feature-pyramid backbone (TorchVisionInterface) has no token grid: only the segment-wise mode applies
        grid = getattr(dino, "grid", 0)
        self._mlp = ops.MlpInference(model.input_size, model.hidden[0], model.hidden[1], chunk_rows,
                                       tokens_per_frame=max(grid * grid, getattr(getattr(dino, "_model", None), "npad", 0)),
                                       double=self._double)
        self.refresh_weights()

    def refresh_weights(self):
        """Re-pack the bf16 GEMM operands after the MLP parameters changed (the node's ``load_model``,
        wvn_feature_extractor_node.py:407-450, runs at <= 1 Hz).  For a LinearRnvp the bf16 operands of the per-pixel
        path are re-packed; masks and permutations are read from the module's buffers on every call.  A SimpleGCN's
        kernels read its fp32 parameters on every call: nothing to re-pack."""
        if self._gcn:
            return
        if self._flow:
            self._flow_infer.set_params(self._model.flat_params)
            return
        self._mlp.set_params(self._model.flat_params)

    def load_model(self, path: str) -> bool:
        """The node's ``load_model`` (wvn_feature_extractor_node.py:407-446): pick up ``.tmp_state_dict.pt`` if the
        learner wrote new weights; returns True when the MLP / confidence generator were updated."""
        from .utils.handoff import read_tmp_state_dict

        changed = read_tmp_state_dict(self._model, self._cg, path)
        if changed:
            self.refresh_weights()
        return changed

    @torch.no_grad()
    def predict(self, img: torch.Tensor):
        """img (B,3,H,W) in [0,1] -> (trav (B,H,H), conf (B,H,H)) fp32 on the device."""
        self._check_per_pixel()
        tokens = self._dino.inference_tokens(img)
        return self.predict_from_tokens(tokens, img.shape[2])

    @torch.no_grad()
    def predict_from_tokens(self, tokens: torch.Tensor, out_size: int):
        self._check_per_pixel()
        g = self._dino.grid
        if self._flow:   # anomaly mode: (trav, None) — the node publishes no confidence map here
            return self._flow_infer.pixels(self._model, tokens, (g, g), (out_size, out_size), self._cg.mean.data,
                                           self._cg.std.data, self._cg.std_factor), None
        vit = self._dino._model
        last = getattr(vit, "last_tokens", None)
        if ((not self._double or self._mlp.fused_shape) and last is not None and tokens.data_ptr() == last.data_ptr() and tokens.shape[1:] == last.shape[1:]
                and tokens.shape[0] <= last.shape[0] and self._model.input_size == vit.dim and out_size % 64 == 0):
            # these ARE the backbone's last tokens: its bf16 copy goes to the head as it is (no re-cast of 4.8 MB/frame)
            return self._mlp.pixels_from_vit(vit, tokens.shape[0], (out_size, out_size), self._cg.mean.data,
                                             self._cg.std.data, self._cg.std_factor)
        return self._mlp.pixels(tokens, (g, g), (out_size, out_size), self._cg.mean.data, self._cg.std.data,
                                self._cg.std_factor)

    def _check_per_pixel(self):
        if self._gcn:
            raise ValueError("SimpleGCN predicts per segment only (there is no graph over pixels): use predict_segments "
                             "with the frame's edges")
        if self._pyramid:
            raise ValueError("a feature-pyramid backbone has no per-pixel head (the reference defines none): use "
                             "predict_frames, or predict_segments for one frame")
        if self._dino is None:
            raise ValueError("no token front end was given: per-pixel maps need one; use predict_frames or "
                             "predict_segments")

    @torch.no_grad()
    def predict_rows(self, feat, n_rows, edges=None, n_edges=None):
        """Padded-row inference on a batch as ``extract_batch`` leaves it: feat [B, smax, D] and n_rows [B] int32 on
        the device -> (trav, conf) [B, smax], NaN on padding rows; conf is None for the LinearRnvp.  A SimpleGCN also
        needs the frames' edges [B, E, 2] / n_edges [B].  Device ops only (no host synchronisation)."""
        m, s, f = self._cg.mean.data, self._cg.std.data, self._cg.std_factor
        if self._gcn:
            if edges is None or n_edges is None:
                raise ValueError("predict_frames: a SimpleGCN needs the frames' edges and n_edges")
            return self._gcn_infer.rows_padded(feat, n_rows, edges, n_edges, m, s, f)
        if self._flow:
            return self._flow_infer.trav_padded(self._model, feat, n_rows, m, s, f), None
        return self._mlp.rows_padded(feat, n_rows, m, s, f)

    @torch.no_grad()
    def predict_frames(self, feat, n_rows, edges, n_edges, seg):
        """Segment-wise maps of a batch as ``extract_batch`` leaves it: feat [B, smax, D], n_rows [B] int32, edges
        [B, E, 2] / n_edges [B] (read by the SimpleGCN only; may be None otherwise), seg [B, H, W] int64 or int32 ->
        (trav, conf) [B, H, W], each pixel its segment's value (NaN for an id outside [0, n_rows)); conf is None for the
        LinearRnvp.  Device ops only (no host synchronisation)."""
        trav, conf = self.predict_rows(feat, n_rows, edges, n_edges)
        return ops.segment_maps(seg, n_rows, trav, conf)

    @torch.no_grad()
    def predict_segments(self, feat: torch.Tensor, seg: torch.Tensor, edges: torch.Tensor = None):
        """Segment-wise mode (``prediction_per_pixel=False``, node :324-327): MLP on the S pooled rows,
        scattered back through ``seg``.  For a LinearRnvp: (trav[seg], None), trav the confidence of each row's NLL.
        A SimpleGCN runs on the frame's graph ``edges`` (2, E) (source, target segment ids, as ``extract`` returns
        them), which it requires; the other learners ignore it."""
        if self._gcn:
            if edges is None:
                raise ValueError("predict_segments: a SimpleGCN needs the frame's edges (2, E)")
            trav, conf = self._gcn_infer.rows(feat, edges, self._cg.mean.data, self._cg.std.data, self._cg.std_factor)
            return trav[seg], conf[seg]
        if self._flow:
            return self._flow_infer.trav(self._model, feat, self._cg.mean.data, self._cg.std.data,
                                         self._cg.std_factor)[seg], None
        trav, conf = self._mlp.rows(feat, self._cg.mean.data, self._cg.std.data, self._cg.std_factor)
        return trav[seg], conf[seg]
