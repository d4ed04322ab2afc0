"""Name -> model registry (reference: wild_visual_navigation/model/network_register.py:44-55)."""
from .simple_mlp import SimpleMLP


def get_model(model_cfg):
    """model_cfg: mapping / attribute bag with ``name`` and ``simple_mlp_cfg`` like
    ``ExperimentParams.model`` (cfg/experiment_params.py:104-112)."""
    get = (lambda k: model_cfg[k]) if isinstance(model_cfg, dict) else (lambda k: getattr(model_cfg, k))
    name = get("name")
    if name == "SimpleMLP":
        cfg = get("simple_mlp_cfg")
        cfg = dict(cfg) if isinstance(cfg, dict) else dict(vars(cfg))
        return SimpleMLP(**cfg)
    raise ValueError(f"model '{name}' is outside the H100 hot path (only SimpleMLP; SURVEY.md §2)")
