"""FeatureExtractor (reference: wild_visual_navigation/feature_extractor/feature_extractor.py:20-398).

``extract(img, **kwargs) -> (edges, feat, seg, center, dense_feat)`` with the reference's kwargs
(``return_dense_features``, ``n_random_pixels``, ``cell_size``).  Differences in HOW, not WHAT:
  * the per-segment mean of the bilinearly upsampled features is computed from the ViT tokens by a
    segmented reduction (csrc/segment_kernels.cu) — the 308 MB/frame dense tensor is formed only
    when ``return_dense_features=True`` asks for it;
  * adjacency + centroids come from the same pass (no per-segment Python loops / host syncs);
  * when segmentation and features are both "stego"/"dino" on the same backbone, one ViT forward
    serves both (the reference runs two backbones); with "dinov2" / "dinov2_reg" features, STEGO's DINO backbone
    segments and a second, DINOv2 handle gives the features;
  * "torchvision" features (``model_type`` resnet18 / resnet50 / resnet50_dino / efficientnet_b0) are a feature
    pyramid (four levels, five for EfficientNet-B0) pooled per segment level by level (csrc/resnet_kernels.cu), as
    sparsify_features' dict branch does.  Where a segment has no
    cell at a coarse level the reference raises AttributeError; here it takes the cell under its centroid.  "random" and
    "none" segmentation crash in the reference with a pyramid and raise ValueError here.
Supported: segmentation_type in {"slic" (the constructor default), "stego", "grid", "random", "none"/None},
feature_type in {"dino", "dinov2", "dinov2_reg", "stego", "torchvision"}.  "slic" is an all-integer SLIC kernel (csrc/slic_kernels.cu; fast_slic itself is an
un-vendored C++ package, see oracle/slic.py for what is and is not restated).  "sift", "histogram"
features are out of scope (SURVEY.md §2) and raise.
"""
from __future__ import annotations

import torch

from .. import ops
from .dino_interface import DinoInterface
from .segment_extractor import SegmentExtractor
from .stego_interface import StegoInterface
from .torchvision_interface import MODEL_TYPES, TorchVisionInterface


class FeatureExtractor:
    def __init__(self, device: str, segmentation_type: str = "slic", feature_type: str = "dino",
                 input_size: int = 448, **kwargs):
        self._device = device
        self._segmentation_type = segmentation_type
        self._feature_type = feature_type
        self._input_size = input_size
        self.segment_extractor = SegmentExtractor()
        if segmentation_type not in ("slic", "stego", "grid", "random", "none", None):
            raise ValueError(f"segmentation_type [{segmentation_type}] not supported")
        # fast_slic.Slic(num_components, compactness) of the reference (feature_extractor.py:88-95)
        self._slic_num_components = kwargs.get("slic_num_components", 100)
        self._slic_compactness = kwargs.get("slic_compactness", 10)
        self._slic_iters = kwargs.get("slic_iters", 10)
        # grid segmentation's cell size when extract / extract_batch are not given one (segment_grid's default, 32)
        self._cell_size = kwargs.get("cell_size", 32)
        common = dict(backbone_type=kwargs.get("backbone_type", "vit_small"), patch_size=kwargs.get("patch_size", 8),
                      max_batch=kwargs.get("max_batch", 1), chunk=kwargs.get("chunk", 0))
        need_stego = feature_type == "stego" or segmentation_type == "stego"
        if feature_type == "stego":
            self._feature_dim = 90
        elif feature_type == "torchvision":
            if segmentation_type in ("random", "none", None):
                # the reference indexes / returns the pyramid dict as a tensor there and crashes
                raise ValueError(f"segmentation_type [{segmentation_type}] does not work with torchvision features")
            if "model_type" not in kwargs:
                raise ValueError(f"feature_type 'torchvision' needs model_type ({', '.join(MODEL_TYPES)})")
        elif "dino" in feature_type:
            # the reference hard-codes 384 for every dino variant (feature_extractor.py:56)
            self._feature_dim = 384 if common["backbone_type"] == "vit_small" else 768
        else:
            raise ValueError(f"Extractor[{feature_type}] is outside the H100 hot path")
        # the feature backbone, as the reference picks it (feature_extractor.py:61): "dino", "dinov2" or "dinov2_reg"
        backbone = kwargs.get("backbone", feature_type)
        # STEGO's own backbone is DINO; it serves the features too unless they come from another backbone
        share = feature_type == "stego" or backbone == "dino"
        if need_stego:
            self._stego = StegoInterface(device=device, input_size=input_size, run_crf=kwargs.get("run_crf", False),
                                         run_clustering=kwargs.get("run_clustering", True),  # the reference's default (:51)
                                         n_image_clusters=kwargs.get("n_image_clusters", 20),
                                         head_state_dict=kwargs.get("head_state_dict"),
                                         backbone_state_dict=kwargs.get("state_dict" if share else "stego_state_dict"),
                                         flip_tta=kwargs.get("flip_tta", True),
                                         kmeans_iters=kwargs.get("kmeans_iters", 10), **common)
        else:
            self._stego = None
        self._tv = None
        if feature_type == "torchvision":
            # with segmentation_type="stego", STEGO segments on its own DINO backbone (`stego_state_dict`)
            self._dino = None
            self._tv = TorchVisionInterface(device, kwargs["model_type"], input_size, max_batch=common["max_batch"],
                                            pretrained=kwargs.get("pretrained", True), state_dict=kwargs.get("state_dict"),
                                            pretrained_weights=kwargs.get("pretrained_weights"))
            self._extractor = self._tv
            # the reference never sets it for torchvision (reading it raises); the pooled row width
            self._feature_dim = self._tv.feature_dim
        elif need_stego and share:
            self._dino = self._stego._dino
            self._extractor = self._stego if feature_type == "stego" else self._dino
        else:
            # with segmentation_type="stego" and DINOv2 features: a second handle; `state_dict` is this backbone's
            # and `stego_state_dict` STEGO's
            self._dino = DinoInterface(device=device, input_size=input_size, backbone=backbone,
                                       state_dict=kwargs.get("state_dict"),
                                       pretrained_weights=kwargs.get("pretrained_weights"), **common)
            self._extractor = self._dino

    # ---- reference properties ---------------------------------------------------------------
    @property
    def feature_type(self):
        return self._feature_type

    @property
    def feature_dim(self):
        return self._feature_dim

    @property
    def segmentation_type(self):
        return self._segmentation_type

    @property
    def max_segments(self):
        """Upper bound of segments per frame (rows of the padded ``feat`` per frame) of the stego, slic and grid
        segmentations at ``input_size`` (grid: at the constructor's ``cell_size``); None for the others."""
        if self._segmentation_type == "stego":
            return self._stego.max_segments
        if self._segmentation_type == "slic":
            _, nx, ny = ops.slic_geometry(self._input_size, self._input_size, self._slic_num_components)
            return nx * ny
        if self._segmentation_type == "grid":
            return ((self._input_size + self._cell_size - 1) // self._cell_size) ** 2
        return self._stego.max_segments if self._stego is not None else None

    def change_device(self, device):
        self._device = device
        self._extractor.change_device(device)

    # ---- the hot call -----------------------------------------------------------------------
    @torch.no_grad()
    def extract(self, img, **kwargs):
        img = img.to(self._device, dtype=torch.float32)
        B, _, H, W = img.shape
        assert B == 1, "extract() keeps the reference's single-frame contract; use extract_batch() for B > 1"
        r = self.extract_batch(img, **kwargs)
        seg = r["seg"][0]
        if self._segmentation_type in ("none", None):
            n, feat = seg.numel(), None
        else:
            n = int(r["n_segments"][0].item())
            feat = r["feat"][0, :n]
        dense = r["dense"] if kwargs.get("return_dense_features", False) else None
        if self._segmentation_type == "random":
            return None, feat, seg, None, dense
        if self._segmentation_type in ("none", None):   # segment_pixelwise: dense features are the features (:389-396)
            return r["edges"].T, r["feat"], seg, r["centers"], dense
        ne = int(r["n_edges"][0].item())
        if ne < 0:  # the kernel flags an edge-buffer overflow with -(true count) instead of dropping edges silently
            raise RuntimeError(f"adjacency list has {-ne} edges, more than the buffer of {r['edges'].shape[1]}")
        edges = r["edges"][0, :ne].T.contiguous()
        center = r["centers"][0, :n]
        return edges, feat, seg, center, dense

    @torch.no_grad()
    def extract_batch(self, img, **kwargs):
        """Batched form of ``extract`` (no per-frame host sync): returns padded device tensors
        seg [B,H,W] i64, feat [B,smax,D], centers [B,smax,2], edges [B,E,2], n_edges [B], n_segments [B]."""
        if img.dtype == torch.uint8:  # camera frames (B,H0,W0,3): ingest fused into the patch loader (§8f rank 1)
            img = img.to(self._device)
            B, H, W = img.shape[0], self._input_size, self._input_size
        else:
            img = img.to(self._device, dtype=torch.float32)
            B, _, H, W = img.shape
        g = self._dino.grid if self._dino is not None else None
        # 1. segmentation (+ the one backbone pass)
        tokens = None
        if self._segmentation_type == "stego":
            self._stego._forward(img, want_linear=False)
            # relabelled in place, as in the reference (segment_stego's loop mutates the interface's tensor too: `.to` on
            # the same device returns it, feature_extractor.py:240-246)
            seg = self._stego.cluster_ids.contiguous()
            smax = self._stego.max_segments
            counts = ops.relabel(seg, smax)
            if self._feature_type == "stego":
                tokens = self._stego.code_tokens
            elif self._dino is self._stego._dino:
                tokens = self._stego.backbone_tokens
            # otherwise the features come from their own backbone (DINOv2), run in step 2
        elif self._segmentation_type == "grid":
            cell = kwargs.get("cell_size", self._cell_size)
            ys = torch.arange(H, device=img.device) // cell
            xs = torch.arange(W, device=img.device) // cell
            ncol = (W + cell - 1) // cell
            seg = (ys[:, None] * ncol + xs[None, :]).expand(B, H, W).contiguous()
            smax = int(((H + cell - 1) // cell) * ncol)
            counts = torch.full((B,), smax, device=img.device, dtype=torch.int32)
        elif self._segmentation_type == "random":
            nr = kwargs.get("n_random_pixels", 100)
            seg = torch.full((B, H * W), -1, dtype=torch.long, device=img.device)
            for b in range(B):
                idx = torch.randperm(H * W, device=img.device)[:nr]
                seg[b, idx] = torch.arange(0, nr, device=img.device)
            seg = seg.reshape(B, H, W)
            smax = nr
            counts = torch.full((B,), nr, device=img.device, dtype=torch.int32)
        elif self._segmentation_type == "slic":
            if img.dtype == torch.uint8:
                raise ValueError("slic segmentation takes the resized float image (B,3,H,W), as the reference passes it")
            K = self._slic_num_components
            seg = ops.slic(img, K, self._slic_compactness, self._slic_iters)
            _, nx, ny = ops.slic_geometry(H, W, K)
            smax = nx * ny
            counts = ops.relabel(seg, smax)   # clusters that lost all their pixels leave no gap (no NaN feature rows)
        else:  # pixel-wise ("none" / None, segment_pixelwise :179-196): every pixel is its own segment
            assert B == 1, "pixel-wise segmentation is single-frame (200 704 nodes per 448x448 frame)"
            dev = img.device
            seg = torch.arange(0, H * W, device=dev).reshape(1, H, W)
            ys, xs = torch.arange(H, device=dev, dtype=torch.int32), torch.arange(W, device=dev, dtype=torch.int32)
            centers = torch.stack((ys[:, None].expand(H, W).reshape(-1), xs[None, :].expand(H, W).reshape(-1)), 1)  # (y, x)
            s0 = seg[0]
            hor = torch.stack((s0[:, :-1].reshape(-1), s0[:, 1:].reshape(-1)), 1)
            ver = torch.stack((s0[:-1, :].reshape(-1), s0[1:, :].reshape(-1)), 1)
            edges = torch.cat((hor, ver), 0)
            if self._feature_type == "stego":
                self._stego._forward(img, want_linear=False)
                tokens = self._stego.code_tokens
            else:
                tokens = self._dino.inference_tokens(img)
            dense = ops.upsample_dense(tokens, g, g, H, H)
            return {"seg": seg, "feat": dense, "centers": centers, "edges": edges, "n_edges": None, "n_segments": None,
                    "tokens": tokens, "dense": dense}
        # 2. features
        if self._tv is not None:
            # feature pyramid: per segment and level, the mean over the level's nearest-downsampled segmentation
            taps = self._tv.inference_taps(img)
            want_graph = self._segmentation_type != "random"
            r = ops.segment_reduce(seg, smax, want_centers=True, want_edges=want_graph)
            feat = ops.segment_pool_pyramid(seg, smax, taps, r["centers"])
            out = {"seg": seg, "feat": feat, "centers": r["centers"], "edges": r["edges"], "n_edges": r["n_edges"],
                   "n_segments": counts, "tokens": None, "dense": None}
            if kwargs.get("return_dense_features", False):
                out["dense"] = self._tv.dense(taps)
            return out
        if tokens is None:
            if self._feature_type == "stego":
                self._stego._forward(img, want_linear=False)
                tokens = self._stego.code_tokens
            else:
                tokens = self._dino.inference_tokens(img)
        # 3. per-segment pooling + graph structure in one pass
        want_graph = self._segmentation_type != "random"
        r = ops.segment_reduce(seg, smax, tokens=tokens, grid=(g, g), want_centers=want_graph, want_edges=want_graph)
        out = {"seg": seg, "feat": r["feat"], "centers": r["centers"], "edges": r["edges"], "n_edges": r["n_edges"],
               "n_segments": counts, "tokens": tokens, "dense": None}
        if kwargs.get("return_dense_features", False):
            out["dense"] = ops.upsample_dense(tokens, g, g, H, H)
        return out
