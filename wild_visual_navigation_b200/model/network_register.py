"""Name -> model registry (reference: wild_visual_navigation/model/network_register.py:44-55)."""
from .linear_rnvp import LinearRnvp
from .simple_gcn import SimpleGCN
from .simple_mlp import DoubleMLP, SimpleMLP


def get_model(model_cfg):
    """model_cfg: mapping / attribute bag with ``name`` and ``simple_mlp_cfg`` / ``double_mlp_cfg`` / ``simple_gcn_cfg`` /
    ``linear_rnvp_cfg`` like ``ExperimentParams.model`` (cfg/experiment_params.py:104-140)."""
    get = (lambda k: model_cfg[k]) if isinstance(model_cfg, dict) else (lambda k: getattr(model_cfg, k))
    name = get("name")
    if name == "SimpleMLP":
        cfg = get("simple_mlp_cfg")
        cfg = dict(cfg) if isinstance(cfg, dict) else dict(vars(cfg))
        return SimpleMLP(**cfg)
    if name == "DoubleMLP":
        cfg = get("double_mlp_cfg")
        cfg = dict(cfg) if isinstance(cfg, dict) else dict(vars(cfg))
        return DoubleMLP(**cfg)
    if name == "SimpleGCN":
        cfg = get("simple_gcn_cfg")
        cfg = dict(cfg) if isinstance(cfg, dict) else dict(vars(cfg))
        return SimpleGCN(**cfg)
    if name == "LinearRnvp":
        cfg = get("linear_rnvp_cfg")
        cfg = dict(cfg) if isinstance(cfg, dict) else dict(vars(cfg))
        return LinearRnvp(**cfg)
    raise ValueError(f"model '{name}' is outside the H100 hot path (SimpleMLP, DoubleMLP, LinearRnvp; SURVEY.md §2)")
