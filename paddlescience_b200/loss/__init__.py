from . import mtl
from .base import Loss
from .l2 import L2RelLoss
from .mse import CausalMSELoss, MSELoss, MSELossWithL2Decay

__all__ = ["Loss", "MSELoss", "CausalMSELoss", "MSELossWithL2Decay", "L2RelLoss", "mtl", "build_loss"]


def build_loss(cfg):
    cfg = dict(cfg)
    name = cfg.pop("name")
    return globals()[name](**cfg)
