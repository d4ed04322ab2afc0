from .data import Data, Batch
from .confidence_generator import ConfidenceGenerator
from .loss import AnomalyLoss, TraversabilityLoss
from .handoff import write_tmp_state_dict, read_tmp_state_dict, TMP_STATE_DICT_NAME
from .wire import encode_image_features, decode_image_features
