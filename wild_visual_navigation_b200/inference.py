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
"""
from __future__ import annotations

import torch

from . import ops
from .model.linear_rnvp import LinearRnvp
from .model.simple_gcn import SimpleGCN
from .model.simple_mlp import DoubleMLP, SimpleMLP
from .utils.confidence_generator import ConfidenceGenerator


class TraversabilityInference:
    def __init__(self, dino, model: SimpleMLP, confidence_generator: ConfidenceGenerator, chunk_rows: int = 0):
        self._gcn = isinstance(model, SimpleGCN)
        if self._gcn:
            model.check_supported()
            self._dino, self._model, self._cg = dino, model, confidence_generator
            self._gcn_infer = ops.GcnInference(model)
            self._flow = self._double = False
            return
        self._flow = isinstance(model, LinearRnvp)
        if self._flow:
            if model.flat_params is None or not model.flat_params.is_cuda:
                raise ValueError("TraversabilityInference: the LinearRnvp must be on a CUDA device")
            self._dino, self._model, self._cg = dino, model, confidence_generator
            self._flow_infer = ops.FlowInference(model.input_size, model.hidden, max_rows=1024, chunk_pixels=chunk_rows)
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
                                       tokens_per_frame=max(grid * grid, getattr(dino._model, "npad", 0)),
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
        self._no_pixels_for_gcn()
        tokens = self._dino.inference_tokens(img)
        return self.predict_from_tokens(tokens, img.shape[2])

    @torch.no_grad()
    def predict_from_tokens(self, tokens: torch.Tensor, out_size: int):
        self._no_pixels_for_gcn()
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

    def _no_pixels_for_gcn(self):
        if self._gcn:
            raise ValueError("SimpleGCN predicts per segment only (there is no graph over pixels): use predict_segments "
                             "with the frame's edges")

    @torch.no_grad()
    def predict_frames(self, feat, n_rows, edges, n_edges, seg):
        """SimpleGCN, segment-wise on a batch as ``extract_batch`` leaves it: feat [B, smax, D], n_rows [B], edges
        [B, E, 2] / n_edges [B] on the device, seg [B, H, W] -> (trav, conf) [B, H, W], each pixel its segment's value.
        Device ops only (no host synchronisation)."""
        if not self._gcn:
            raise ValueError("predict_frames is the SimpleGCN's segment-wise path")
        trav, conf = self._gcn_infer.rows_padded(feat, n_rows, edges, n_edges, self._cg.mean.data, self._cg.std.data,
                                                 self._cg.std_factor)
        B = seg.shape[0]
        idx = seg.reshape(B, -1).long()
        return trav.gather(1, idx).view_as(seg), conf.gather(1, idx).view_as(seg)

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
