from .segment_extractor import SegmentExtractor
from .dino_interface import DinoInterface
from .stego_interface import StegoInterface
from .torchvision_interface import TorchVisionInterface
from .feature_extractor import FeatureExtractor
