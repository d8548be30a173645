"""``L2RelLoss`` (reference: ppsci/loss/l2.py:218-311), for validators.

It is evaluated in torch on the evaluation path.  It has no fused head kernel, so a training constraint given it
raises (``utils/expression.py``) rather than train another loss."""
from __future__ import annotations

from typing import Dict, Optional, Union

import torch

from . import base


class L2RelLoss(base.Loss):
    r"""Per sample (row) ``||x - y||_2 / ||y||_2`` over the sample's trailing dimensions, times ``weight_dict[key]``,
    reduced by ``mean`` or ``sum`` and scaled by ``weight``.  For ``[N, 1]`` columns a sample is one point.

    >>> import torch
    >>> out = {"u": torch.tensor([[0.5, 0.9], [1.1, -1.3]]), "v": torch.tensor([[0.5, 0.9], [1.1, -1.3]])}
    >>> lab = {"u": torch.tensor([[-1.8, 1.0], [-0.2, 2.5]]), "v": torch.tensor([[0.1, 0.1], [0.1, 0.1]])}
    >>> {k: round(float(v), 6) for k, v in L2RelLoss(weight={"u": 0.8, "v": 0.2})(out, lab).items()}
    {'u': 1.087762, 'v': 1.849008}
    """

    def __init__(self, reduction: str = "mean", weight: Optional[Union[float, Dict[str, float]]] = None):
        if reduction not in ["mean", "sum"]:
            raise ValueError(f"reduction should be 'mean' or 'sum', but got {reduction}")
        super().__init__(reduction, weight)

    @staticmethod
    def rel_loss(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        x_, y_ = x.reshape(x.shape[0], -1), y.reshape(y.shape[0], -1)
        return torch.linalg.vector_norm(x_ - y_, dim=1) / torch.linalg.vector_norm(y_, dim=1)

    def forward(self, output_dict, label_dict, weight_dict=None) -> Dict[str, torch.Tensor]:
        losses = {}
        for key in label_dict:
            loss = self.rel_loss(output_dict[key], label_dict[key])
            if weight_dict and key in weight_dict:
                w = torch.as_tensor(weight_dict[key], dtype=loss.dtype, device=loss.device)
                loss = loss * (w.reshape(loss.shape) if w.numel() == loss.numel() else w)
            loss = loss.sum() if self.reduction == "sum" else loss.mean()
            if isinstance(self.weight, (float, int)):
                loss = loss * self.weight
            elif isinstance(self.weight, dict) and key in self.weight:
                loss = loss * self.weight[key]
            losses[key] = loss
        return losses
