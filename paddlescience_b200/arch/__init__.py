from .base import Arch
from .mlp import MLP, ModifiedMLP, PirateNet
from .deeponet import DeepONet
from .he_deeponets import HEDeepONets
from .chip_deeponets import ChipDeepONets
from .activation import get_activation

__all__ = ["Arch", "MLP", "ModifiedMLP", "PirateNet", "DeepONet", "HEDeepONets", "ChipDeepONets", "get_activation", "build_model"]


def build_model(cfg):
    """ppsci/arch/__init__.py:116-141 — build a model from a plain dict config."""
    cfg = dict(cfg)
    name = cfg.pop("name")
    return globals()[name](**cfg)
