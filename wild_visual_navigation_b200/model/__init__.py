from .simple_mlp import DoubleMLP, SimpleMLP
from .simple_gcn import SimpleGCN
from .linear_rnvp import LinearRnvp
from .network_register import get_model
