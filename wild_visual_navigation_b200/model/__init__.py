from .simple_mlp import DoubleMLP, SimpleMLP
from .linear_rnvp import LinearRnvp
from .network_register import get_model
