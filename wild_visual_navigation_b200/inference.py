"""Per-frame traversability inference — the arithmetic of ``WvnFeatureExtractor.image_callback``
(reference: wild_visual_navigation_ros/scripts/wvn_feature_extractor_node.py:306-370) and of
``quick_start.py:174-214`` without ROS:

    dense_feat = feature_extractor.extract(img, return_dense_features=True)
    x = dense_feat[0].permute(1,2,0).reshape(-1, D);  prediction = model.forward(Data(x=x))
    out_trav = prediction.reshape(H,W,-1)[:,:,0]
    loss_reco = mse(prediction[:,1:], x).mean(1);  confidence = cg.inference_without_update(loss_reco)

fused as: ViT tokens -> (bilinear sample -> 3 wgmma GEMMs -> sigmoid / reco-loss / confidence
epilogue) per pixel; neither ``dense_feat`` (308 MB/frame) nor the (P, 385) prediction is stored.
"""
from __future__ import annotations

import torch

from . import ops
from .model.simple_mlp import SimpleMLP
from .utils.confidence_generator import ConfidenceGenerator


class TraversabilityInference:
    def __init__(self, dino, model: SimpleMLP, confidence_generator: ConfidenceGenerator, chunk_rows: int = 0):
        assert model.fused_ok(), "model must be the hot-path SimpleMLP(D,[256,32,1],reconstruction=True) on CUDA"
        self._dino = dino
        self._model = model
        self._cg = confidence_generator
        # a feature-pyramid backbone (TorchVisionInterface) has no token grid: only the segment-wise mode applies
        grid = getattr(dino, "grid", 0)
        self._mlp = ops.MlpInference(model.input_size, model.hidden[0], model.hidden[1], chunk_rows,
                                       tokens_per_frame=max(grid * grid, getattr(dino._model, "npad", 0)))
        self.refresh_weights()

    def refresh_weights(self):
        """Re-pack the bf16 GEMM operands after the MLP parameters changed (the node's ``load_model``,
        wvn_feature_extractor_node.py:407-450, runs at <= 1 Hz)."""
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
        tokens = self._dino.inference_tokens(img)
        return self.predict_from_tokens(tokens, img.shape[2])

    @torch.no_grad()
    def predict_from_tokens(self, tokens: torch.Tensor, out_size: int):
        g = self._dino.grid
        vit = self._dino._model
        last = getattr(vit, "last_tokens", None)
        if (last is not None and tokens.data_ptr() == last.data_ptr() and tokens.shape[1:] == last.shape[1:]
                and tokens.shape[0] <= last.shape[0] and self._model.input_size == vit.dim and out_size % 64 == 0):
            # these ARE the backbone's last tokens: its bf16 copy goes to the head as it is (no re-cast of 4.8 MB/frame)
            return self._mlp.pixels_from_vit(vit, tokens.shape[0], (out_size, out_size), self._cg.mean.data,
                                             self._cg.std.data, self._cg.std_factor)
        return self._mlp.pixels(tokens, (g, g), (out_size, out_size), self._cg.mean.data, self._cg.std.data,
                                self._cg.std_factor)

    @torch.no_grad()
    def predict_segments(self, feat: torch.Tensor, seg: torch.Tensor):
        """Segment-wise mode (``prediction_per_pixel=False``, node :324-327): MLP on the S pooled rows,
        scattered back through ``seg``."""
        trav, conf = self._mlp.rows(feat, self._cg.mean.data, self._cg.std.data, self._cg.std_factor)
        return trav[seg], conf[seg]
