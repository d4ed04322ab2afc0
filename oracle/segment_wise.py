"""ORACLE — the node's segment-wise inference (``prediction_per_pixel: False``, wvn_feature_extractor_node.py:319-365),
restated in plain torch in the dtype of its inputs (float64 in the tests):

    input_feat = feat[seg.reshape(-1)];  prediction = model.forward(Data(x=input_feat))
    SimpleMLP:  out_trav = prediction[:, 0];  loss_reco = mse(prediction[:, 1:], x, reduction="none").mean(1);
                confidence = confidence_generator.inference_without_update(loss_reco)
    LinearRnvp: losses = logprob.sum(1) + log_det;  out_trav = inference_without_update(-losses)  (no confidence map)

``node_maps`` is that per-pixel evaluation; ``segment_maps`` evaluates each of the S rows once and paints the values
through ``seg`` (what ``TraversabilityInference.predict_frames`` computes).  Every pixel of a segment carries the same
row, and each output is a function of its row alone, so the two are equal.
"""
from __future__ import annotations

import torch

from . import linear_rnvp
from .wvn_path import mlp_forward


def _confidence(x, mean, std, std_factor: float):
    """ConfidenceGenerator.inference_without_update (utils/confidence_generator.py:182-193) in the dtype of x."""
    mean, std = mean.to(x.dtype), std.to(x.dtype)
    shifted = mean + std * std_factor
    lo = torch.maximum(shifted - std, torch.zeros_like(std))
    hi = shifted + std
    return 1 - (torch.clip(x, lo, hi) - lo) / (hi - lo)


def mlp_head(sd: dict, cg_mean, cg_std, std_factor: float):
    """rows x [N, D] -> (trav [N], confidence [N]) of a SimpleMLP(D, [h1, h2, 1], reconstruction=True)."""
    def run(x):
        pred = mlp_forward(x, sd)
        loss_reco = ((pred[:, 1:] - x) ** 2).mean(1)
        return pred[:, 0], _confidence(loss_reco, cg_mean, cg_std, std_factor)
    return run


def flow_head(sd: dict, cg_mean, cg_std, std_factor: float):
    """rows x [N, D] -> (trav [N], None) of a LinearRnvp: the generator's confidence of each row's NLL."""
    def run(x):
        r = linear_rnvp.forward(sd, x)
        losses = r["logprob"].sum(1) + r["log_det"]
        return _confidence(-losses, cg_mean, cg_std, std_factor), None
    return run


def node_maps(feat: torch.Tensor, seg: torch.Tensor, head):
    """The node: the model on feat[seg.reshape(-1)], one row per pixel -> (trav, conf) shaped like seg."""
    trav, conf = head(feat[seg.reshape(-1)])
    return trav.reshape(seg.shape), (conf.reshape(seg.shape) if conf is not None else None)


def segment_maps(feat: torch.Tensor, seg: torch.Tensor, head):
    """Each segment's row once, painted through seg -> (trav, conf) shaped like seg."""
    trav, conf = head(feat)
    return trav[seg], (conf[seg] if conf is not None else None)
