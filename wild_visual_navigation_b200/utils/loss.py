"""TraversabilityLoss (reference: wild_visual_navigation/utils/loss.py:57-164) and AnomalyLoss (:16-54).

Holds the loss weights and the ConfidenceGenerator.  In the reference ``forward`` builds an
autograd graph; here the whole fwd + loss + bwd + Adam step is one fused kernel sequence driven
by ``TraversabilityEstimator.train`` (csrc/mlp_train.cu).  ``forward`` keeps the reference's
signature and return triple for monitoring use: it evaluates the same loss terms (no grad).
"""
from __future__ import annotations

import torch
from torch import nn

from .confidence_generator import ConfidenceGenerator


class TraversabilityLoss(nn.Module):
    def __init__(self, w_trav: float, w_reco: float, w_temp: float, anomaly_balanced: bool, model: nn.Module,
                 method: str, confidence_std_factor: float, log_enabled: bool = False, log_folder: str = "/tmp",
                 trav_cross_entropy=False):
        super().__init__()
        if trav_cross_entropy:
            raise ValueError("trav_cross_entropy is not supported on the H100 hot path (reference default: False)")
        self._w_trav, self._w_reco, self._w_temp = w_trav, w_reco, w_temp
        # registered as a sub-module exactly as the reference does (loss.py:74: ``self._model = model``), so that
        # ``traversability_loss_state_dict`` carries ``_model.layers.{0,2,4}.{weight,bias}`` next to
        # ``_confidence_generator.*`` and checkpoints interoperate with the reference in both directions
        self._model = model
        self._anomaly_balanced = anomaly_balanced
        self._confidence_generator = ConfidenceGenerator(
            std_factor=confidence_std_factor, method=method, log_enabled=log_enabled, log_folder=log_folder)

    def reset(self):
        if self._anomaly_balanced:
            self._confidence_generator.reset()

    @torch.no_grad()
    def forward(self, graph, res: torch.Tensor, update_generator: bool = True, step: int = 0, log_step: bool = False):
        d = graph.x.shape[1]
        loss_reco = ((res[:, -d:] - graph.x) ** 2).mean(dim=1)
        if update_generator:
            confidence = self._confidence_generator.update(x=loss_reco, x_positive=loss_reco[graph.y_valid], step=step)
        else:
            confidence = self._confidence_generator.inference_without_update(x=loss_reco)
        raw = (res[:, 0] - graph.y) ** 2
        if self._anomaly_balanced:
            w = torch.where(graph.y_valid, torch.ones_like(confidence), 1 - confidence)
            loss_trav_confidence = (raw * w).sum() / graph.y.shape[0]
        else:
            loss_trav_confidence = raw.mean()
        loss_reco_mean = loss_reco[graph.y_valid].mean()
        loss = self._w_trav * loss_trav_confidence + self._w_reco * loss_reco_mean
        aux = {"loss_reco": loss_reco_mean, "loss_trav": raw.mean(), "loss_temp": torch.zeros_like(loss),
               "loss_trav_confidence": loss_trav_confidence, "confidence": confidence}
        return loss, aux, res

    @torch.no_grad()
    def update_node_confidence(self, node):
        reco_loss = ((node.prediction[:, 1:] - node.features) ** 2).mean(dim=1)
        node.confidence = self._confidence_generator.inference_without_update(reco_loss)


class AnomalyLoss(nn.Module):
    """The LinearRnvp learner's loss (reference: utils/loss.py:16-54): ``-mean(logprob.sum(1) + log_det)``, with the
    ConfidenceGenerator updated on the per-row NLL (``x = x_positive``: the batch holds only labelled rows).  The
    training step itself runs fused in csrc/flow_train.cu (``ops.FlowTrainer``); ``forward`` keeps the reference's
    signature and return triple for direct use (no grad)."""

    def __init__(self, confidence_std_factor: float, method: str, log_enabled: bool = False, log_folder: str = "/tmp"):
        super().__init__()
        self._confidence_generator = ConfidenceGenerator(
            std_factor=confidence_std_factor, method=method, log_enabled=log_enabled, log_folder=log_folder)

    @torch.no_grad()
    def forward(self, graph, res: dict, update_generator: bool = True, step: int = 0, log_step: bool = False):
        loss_aux = {"loss_trav": torch.tensor([0.0]), "loss_reco": torch.tensor([0.0])}
        losses = res["logprob"].sum(1) + res["log_det"]
        confidence = None
        if update_generator:
            confidence = self._confidence_generator.update(x=-losses.clone(), x_positive=-losses.clone(), step=step)
        loss_aux["confidence"] = confidence
        return -torch.mean(losses), loss_aux, confidence

    def update_node_confidence(self, node):
        node.confidence = 0
