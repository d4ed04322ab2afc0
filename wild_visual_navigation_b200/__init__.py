"""wild_visual_navigation_b200 — H100-native (sm_90a) hot path of Wild Visual Navigation.

Keeps the reference's class surface for the per-frame path (SURVEY.md §8b):
``FeatureExtractor`` / ``DinoInterface`` / ``TorchVisionInterface`` / ``StegoInterface`` / ``SegmentExtractor`` /
``SimpleMLP`` / ``DoubleMLP`` / ``SimpleGCN`` / ``LinearRnvp`` / ``get_model`` / ``Data`` / ``Batch`` / ``ConfidenceGenerator`` /
``TraversabilityLoss`` / ``AnomalyLoss`` / ``TraversabilityEstimator`` — implemented on hand-written CUDA
kernels behind the C ABI in ``include/wvn_b200.h``.  No CPU fallback.
"""
import os

WVN_ROOT_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

from .utils import Data, Batch, ConfidenceGenerator, TraversabilityLoss, AnomalyLoss  # noqa: E402,F401
from .model import SimpleMLP, DoubleMLP, SimpleGCN, LinearRnvp, get_model  # noqa: E402,F401
from .feature_extractor import (  # noqa: E402,F401
    DinoInterface,
    StegoInterface,
    SegmentExtractor,
    FeatureExtractor,
    TorchVisionInterface,
)
from .traversability_estimator import TraversabilityEstimator  # noqa: E402,F401
from .image_projector import ImageProjector  # noqa: E402,F401
from .inference import TraversabilityInference  # noqa: E402,F401
from .hot_path import HotPathStep  # noqa: E402,F401
