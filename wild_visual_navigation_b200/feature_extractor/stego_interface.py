"""StegoInterface (reference: wild_visual_navigation/feature_extractor/stego_interface.py:19-135).

``inference(img) -> (linear_pred, cluster_pred)`` with the ``features`` / ``cluster_segments`` /
``linear_segments`` properties.  The STEGO head runs as three wgmma GEMMs on the ViT tokens
(csrc/vit_backbone.cu: vit_stego_head); the cluster / linear probes are folded into the head's output
columns (weights.fold_stego_head) and evaluated at patch resolution, then one kernel does the
bilinear(align_corners=False) upsampling + argmax per pixel — algebraically the upstream
``postprocess`` (upsample the 90-d code, then probe every pixel) without the 448x448x90 tensor.
``run_clustering=True`` (WVN's default through ``FeatureExtractor``): the cluster prediction comes from a per-image
k-means of the code with ``n_image_clusters`` clusters (csrc/stego_kmeans.cu — one launch per batch of frames; the
nearest-centroid scores replace the cluster-probe logits before the same upsample+argmax kernel).
``run_crf=True`` (the reference StegoInterface's default, off in WVN's FeatureExtractor): the cluster and linear
predictions are the argmax of STEGO's dense CRF (csrc/dense_crf.cu, definition oracle/dense_crf.py) over the upsampled
probe log-probabilities and the transformed image, instead of the plain argmax.  It cannot be combined with
``run_clustering=True``.
"""
from __future__ import annotations

import torch

from .. import ops
from .dino_interface import DinoInterface, _Cfg
from .weights import (HEAD_CLUSTER_COL, HEAD_CODE_COL, HEAD_LINEAR_COL, fold_stego_head, synthetic_stego_head)


class StegoInterface:
    def __init__(self, device: str, input_size: int = 448, model_path: str = None, n_image_clusters: int = 40,
                 run_crf: bool = False, run_clustering: bool = False, cfg=None, backbone_type: str = "vit_small",
                 patch_size: int = 8, head_state_dict=None, backbone_state_dict=None, flip_tta: bool = True,
                 max_batch: int = 32, chunk: int = 0, code_dim: int = 90, kmeans_iters: int = 10):
        self._cfg = _Cfg(cfg) if cfg else _Cfg(model_path=model_path, input_size=input_size, run_crf=run_crf,
                                               run_clustering=run_clustering, n_image_clusters=n_image_clusters)
        if self._cfg.run_crf and self._cfg.run_clustering:
            raise ValueError("run_crf=True with run_clustering=True is not supported: what upstream feeds the CRF after "
                             "its per-image k-means cannot be pinned; pass run_clustering=False")
        self._kmeans_iters = kmeans_iters
        self._device = device
        self._flip_tta = flip_tta
        if head_state_dict is None:
            if model_path:
                # a STEGO Lightning checkpoint pickles OmegaConf hyper-parameters: needs the full unpickler (trusted file)
                ck = torch.load(model_path, map_location="cpu", weights_only=False)
                sd = ck.get("state_dict", ck)
                head_state_dict = {k.replace("segmentation_head.", ""): v.squeeze(-1).squeeze(-1) if v.dim() == 4 else v
                                   for k, v in sd.items() if k.startswith(("segmentation_head.", "cluster_probe.",
                                                                           "linear_probe."))}
                if backbone_state_dict is None:
                    backbone_state_dict = {k.split("backbone.model.", 1)[1]: v for k, v in sd.items()
                                           if "backbone.model." in k} or None
            else:
                from .weights import VIT_SHAPES
                head_state_dict = synthetic_stego_head(VIT_SHAPES[backbone_type]["dim"], code_dim)
        self._head = head_state_dict
        self._code_dim = int(head_state_dict["cluster1.0.weight"].shape[0])
        self._n_clusters = int(head_state_dict["cluster_probe.clusters"].shape[0])
        if self._cfg.run_clustering and not (1 <= self._cfg.n_image_clusters <= 64):
            raise ValueError("n_image_clusters must be in [1, 64]")
        self._n_classes = int(head_state_dict["linear_probe.weight"].shape[0])
        self._dino = DinoInterface(device, input_size=input_size, backbone_type=backbone_type, patch_size=patch_size,
                                   max_batch=max_batch * (2 if flip_tta else 1), chunk=chunk,
                                   state_dict=backbone_state_dict, head_weights=fold_stego_head(head_state_dict))
        self._code = self._cluster_pred = self._linear_pred = self._head_out = self._cl64 = self._li64 = self._code_tok = None
        self._tokens = self._img = None
        # the CRF's workspaces are sized once, for max_batch frames of input_size x input_size
        self._crf = (ops.DenseCrf(input_size, max(self._n_clusters, self._n_classes), chunk=min(2, max_batch))
                     if self._cfg.run_crf else None)

    def change_device(self, device):
        self._dino.change_device(device)

    @torch.no_grad()
    def inference(self, img: torch.Tensor):
        """img (B,3,H,W) -> (linear_pred, cluster_pred), each (1,B,H,H) int32 like the reference.
        Camera frames (B,H0,W0,3) uint8 are accepted too: they are resized (NEAREST) / center-cropped to
        ``input_size`` inside the patch loader, i.e. H = W = input_size as after ``ImageProjector.resize_image``."""
        self._forward(img, want_linear=True)
        return self.linear_segments, self.cluster_segments

    @torch.no_grad()
    def _forward(self, img: torch.Tensor, want_linear: bool):
        """Backbone + head (+ per-image k-means) + per-pixel cluster argmax.  ``FeatureExtractor`` calls this with
        ``want_linear=False``: WVN only consumes ``cluster_segments`` (feature_extractor.py:237-249), so the linear-probe
        argmax, the int32 copies and the contiguous code tensor are produced lazily by the properties below."""
        if img.dtype == torch.uint8:
            img = img.to(self._device)
            B, H, W = img.shape[0], self._cfg.input_size, self._cfg.input_size
            assert not self._flip_tta, "flip TTA needs the float image (flip is applied to the transformed image)"
        else:
            img = img.to(self._device, dtype=torch.float32)
            B, _, H, W = img.shape
        vit = self._dino._model
        g, npad = vit.grid, vit.npad
        if self._flip_tta:
            # Stego.get_code: average with the pass over the horizontally flipped TRANSFORMED image (the flip happens
            # inside the patch loader, after resize + crop); flip back at patch level
            tokens = vit.forward(img, flip_tta=True)
            out = vit.stego_head(2 * B)                                  # [2B * npad, C]: straight pass, then flipped pass
            ops.flip_average(out, B, npad, g)                            # in place on the straight half (one kernel)
            head = out[: B * npad]
            self._tokens = tokens[:B]
        else:
            self._tokens = vit.forward(img)
            head = vit.stego_head(B)
        S = self._cfg.input_size
        n_cluster_logits = self._n_clusters
        if self._cfg.run_clustering:
            # per-image k-means of the code: the nearest-centroid scores overwrite the cluster-probe logit columns
            n_cluster_logits = self._cfg.n_image_clusters
            ops.stego_kmeans(head, B, npad, g * g, HEAD_CODE_COL, self._code_dim, HEAD_CLUSTER_COL, n_cluster_logits,
                             self._kmeans_iters)
        self._head_out, self._geom = head, (B, H, npad, g, S)
        self._code_tok = self._code = self._cluster_pred = self._linear_pred = self._li64 = None
        if self._crf is not None:
            self._img = img
            self._cl64 = self._to_image_size(self._crf_labels(HEAD_CLUSTER_COL, self._n_clusters, cluster=True))
            if want_linear:
                self._li64 = self._to_image_size(self._crf_labels(HEAD_LINEAR_COL, self._n_classes, cluster=False))
            self._img_hw = (H, W)
            return
        if want_linear:
            cl, li = ops.logits_argmax(head, HEAD_CLUSTER_COL, n_cluster_logits, B, npad, g, g, S, S,
                                       col0_b=HEAD_LINEAR_COL, classes_b=self._n_classes)
            self._li64 = self._to_image_size(li)
        else:
            cl = ops.logits_argmax(head, HEAD_CLUSTER_COL, n_cluster_logits, B, npad, g, g, S, S)
        self._cl64 = self._to_image_size(cl)   # (B, H, H) int64 cluster ids
        self._img_hw = (H, W)

    def _crf_labels(self, col0, classes, cluster):
        """Dense-CRF labels (B, S, S) of the cluster probe (2 <normalize(code), normalize(c_k)>) or the linear probe."""
        B, H, npad, g, S = self._geom
        if cluster:
            return self._crf.run(self._img, self._head_out, npad, g, col0, classes, HEAD_CODE_COL, self._code_dim, 2.0)
        return self._crf.run(self._img, self._head_out, npad, g, col0, classes)

    def _to_image_size(self, pred):
        B, H, npad, g, S = self._geom
        if (S, S) != (H, H):  # stego_interface.py:108-109: predictions go to (H, H) with 'nearest'
            pred = torch.nn.functional.interpolate(pred[None].float(), (H, H), mode="nearest")[0].long()
        return pred

    @property
    def model(self):
        return self._dino._model

    @property
    def max_segments(self):
        """Upper bound of the cluster ids ``cluster_segments`` can hold (+1)."""
        return self._cfg.n_image_clusters if self._cfg.run_clustering else self._n_clusters

    @property
    def input_size(self):
        return self._cfg.input_size

    @property
    def linear_segments(self):
        if self._linear_pred is None and self._head_out is not None:
            if self._li64 is None and self._crf is not None:
                self._li64 = self._to_image_size(self._crf_labels(HEAD_LINEAR_COL, self._n_classes, cluster=False))
            if self._li64 is None:
                B, H, npad, g, S = self._geom
                self._li64 = self._to_image_size(ops.logits_argmax(self._head_out, HEAD_LINEAR_COL, self._n_classes, B, npad,
                                                                   g, g, S, S))
            self._linear_pred = self._li64[None].int()
        return self._linear_pred

    @property
    def cluster_segments(self):
        if self._cluster_pred is None and self._head_out is not None:
            self._cluster_pred = self._cl64[None].int()
        return self._cluster_pred

    @property
    def cluster_ids(self):
        """(B, H, H) int64 cluster ids — the form the segment kernels consume (no int32 round trip)."""
        return self._cl64

    @property
    def code_tokens(self):
        """(B, P, 90) fp32 code at patch resolution — what the fused consumers use."""
        if self._code_tok is None and self._head_out is not None:
            B, H, npad, g, S = self._geom
            self._code_tok = self._head_out.view(B, npad, -1)[:, 1 : 1 + g * g, HEAD_CODE_COL : HEAD_CODE_COL + self._code_dim].contiguous()
        return self._code_tok

    @property
    def backbone_tokens(self):
        return self._tokens

    @property
    def features(self):
        """Dense (B, 90, H, H) code, bilinear align_corners=True (stego_interface.py:107) — materialised lazily."""
        if self._code is None:
            g = self._dino.grid
            H = self._img_hw[0]
            self._code = ops.upsample_dense(self.code_tokens, g, g, H, H)
        return self._code
