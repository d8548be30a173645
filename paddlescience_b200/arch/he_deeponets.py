"""``HEDeepONets`` (reference: ppsci/arch/he_deeponets.py:28-193): the heat exchanger's operator network.

Two branch nets read the hot and the cold side's mass flow rates, one trunk net the coordinates (x, t):

    G_k = sum_{i in block k} heat(qm_h)_i * act(trunk(x, t))_i * cold(qm_c)_i + b_k,   k = 0, 1, 2 (T_h, T_c, T_w),

block k being features kF .. (k+1)F - 1 of the 3F outputs of every sub-network.  The branch outputs get no activation
(the reference builds ``heat_act`` / ``cold_act`` and never applies them).  Every constraint, with or without
derivatives, trains through the operator jet head shared with physics-informed DeepONet (``BranchTrunkArch``)."""
from __future__ import annotations

from typing import Dict, Tuple, Union

import torch

from .deeponet import BranchTrunkArch, SubNet


class HEDeepONets(BranchTrunkArch):
    """Same arguments and defaults as the reference (he_deeponets.py:73-93), plus ``dtype``.  Parameters save and load
    under the reference's keys (``heat_net.*``, ``cold_net.*``, ``trunk_net.*``, ``b`` of shape (3,)).

    Constraint expressions see T_h(x, t, qm_h), T_c(x, t, qm_c) and T_w(x, t): they may differentiate the outputs with
    respect to the trunk inputs and read a branch input as a column when its ``*_num_loc`` is 1 (the heat exchanger's
    coefficients divide by qm_h and qm_c)."""

    def __init__(
        self,
        heat_input_keys: Tuple[str, ...],
        cold_input_keys: Tuple[str, ...],
        trunk_input_keys: Tuple[str, ...],
        output_keys: Tuple[str, ...],
        heat_num_loc: int,
        cold_num_loc: int,
        num_features: int,
        branch_num_layers: int,
        trunk_num_layers: int,
        branch_hidden_size: Union[int, Tuple[int, ...]],
        trunk_hidden_size: Union[int, Tuple[int, ...]],
        branch_skip_connection: bool = False,
        trunk_skip_connection: bool = False,
        branch_activation: str = "tanh",
        trunk_activation: str = "tanh",
        branch_weight_norm: bool = False,
        trunk_weight_norm: bool = False,
        use_bias: bool = True,
        dtype: torch.dtype = torch.float32,
    ):
        super().__init__()
        if len(output_keys) != 3:  # he_deeponets.py:172-189 forms exactly three outputs
            raise ValueError(f"HEDeepONets has exactly three outputs (T_h, T_c, T_w), got output_keys={tuple(output_keys)}")
        self.heat_input_keys, self.cold_input_keys = tuple(heat_input_keys), tuple(cold_input_keys)
        self.trunk_input_keys = tuple(trunk_input_keys)
        self.input_keys = self.trunk_input_keys + self.heat_input_keys + self.cold_input_keys
        branch = SubNet("branch", branch_num_layers, branch_hidden_size, branch_skip_connection, branch_activation,
                        branch_weight_norm)
        trunk = SubNet("trunk", trunk_num_layers, trunk_hidden_size, trunk_skip_connection, trunk_activation, trunk_weight_norm)
        self._setup([("heat_net", self.heat_input_keys, heat_num_loc, branch), ("cold_net", self.cold_input_keys, cold_num_loc, branch)],
                    ("trunk_net", self.trunk_input_keys, trunk), output_keys, num_features, use_bias, dtype)

    def fused_train_forward(self, loss_fn, input_dict, label_dict, weight_dict, output_expr=None,
                            extra_keys=()) -> Dict[str, torch.Tensor]:
        """Losses of one constraint (label keys in order; a key without an expression is that output) and their
        gradient accumulated into ``self.flat.grad``, through the operator jet head.  A constraint without derivatives
        compiles to a values-only head (no trunk jets)."""
        self._check_fused(loss_fn)
        return self._jet_train_forward(loss_fn, input_dict, label_dict, weight_dict, output_expr, extra_keys)
