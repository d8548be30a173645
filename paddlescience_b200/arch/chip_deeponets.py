"""``ChipDeepONets`` (reference: ppsci/arch/chip_deeponets.py:28-199): the chip-heat operator network.

Three branch nets read the heat source's sensor values (``num_loc`` columns), the boundary data (``BC_num_loc``) and
the boundary type (``bctype_loc``), one trunk net the coordinates:

    G = sum_i u(u_sensors)_i * act(trunk(x, y))_i * bc(bc_data)_i * bctype(bc)_i + b.

The branch outputs get no activation (the reference builds ``branch_act`` / ``bc_act`` and never applies them).  Every
constraint, with or without derivatives, trains through the operator jet head with three branch factors
(``BranchTrunkArch``); its expressions may select their residual by boundary type with ``torch.where(bc == k, ...)``."""
from __future__ import annotations

from typing import Dict, Tuple, Union

import torch

from .deeponet import BranchTrunkArch, SubNet


class ChipDeepONets(BranchTrunkArch):
    """Same arguments, defaults and ``input_keys`` order (trunk, branch, BC, BCtype) as the reference
    (chip_deeponets.py:82-110), plus ``dtype``.  ``branch_net`` takes the ``branch_*`` settings, ``BC_net`` and
    ``BCtype_net`` the ``BC_*`` ones.  Parameters save and load under the reference's keys (``branch_net.*``,
    ``BCtype_net.*``, ``BC_net.*``, ``trunk_net.*``, ``b`` of shape (1,))."""

    def __init__(
        self,
        branch_input_keys: Tuple[str, ...],
        BCtype_input_keys: Tuple[str, ...],
        BC_input_keys: Tuple[str, ...],
        trunk_input_keys: Tuple[str, ...],
        output_keys: Tuple[str, ...],
        num_loc: int,
        bctype_loc: int,
        BC_num_loc: int,
        num_features: int,
        branch_num_layers: int,
        BC_num_layers: int,
        trunk_num_layers: int,
        branch_hidden_size: Union[int, Tuple[int, ...]],
        BC_hidden_size: Union[int, Tuple[int, ...]],
        trunk_hidden_size: Union[int, Tuple[int, ...]],
        branch_skip_connection: bool = False,
        BC_skip_connection: bool = False,
        trunk_skip_connection: bool = False,
        branch_activation: str = "tanh",
        BC_activation: str = "tanh",
        trunk_activation: str = "tanh",
        branch_weight_norm: bool = False,
        BC_weight_norm: bool = False,
        trunk_weight_norm: bool = False,
        use_bias: bool = True,
        dtype: torch.dtype = torch.float32,
    ):
        super().__init__()
        if len(output_keys) != 1:  # chip_deeponets.py:195-197 forms one output
            raise ValueError(f"ChipDeepONets has exactly one output, got output_keys={tuple(output_keys)}")
        self.branch_input_keys, self.BCtype_input_keys = tuple(branch_input_keys), tuple(BCtype_input_keys)
        self.BC_input_keys, self.trunk_input_keys = tuple(BC_input_keys), tuple(trunk_input_keys)
        self.input_keys = self.trunk_input_keys + self.branch_input_keys + self.BC_input_keys + self.BCtype_input_keys
        branch = SubNet("branch", branch_num_layers, branch_hidden_size, branch_skip_connection, branch_activation,
                        branch_weight_norm)
        bc = SubNet("BC", BC_num_layers, BC_hidden_size, BC_skip_connection, BC_activation, BC_weight_norm)
        trunk = SubNet("trunk", trunk_num_layers, trunk_hidden_size, trunk_skip_connection, trunk_activation, trunk_weight_norm)
        self._setup([("branch_net", self.branch_input_keys, num_loc, branch),
                     ("BCtype_net", self.BCtype_input_keys, bctype_loc, bc),
                     ("BC_net", self.BC_input_keys, BC_num_loc, bc)],
                    ("trunk_net", self.trunk_input_keys, trunk), output_keys, num_features, use_bias, dtype)

    def fused_train_forward(self, loss_fn, input_dict, label_dict, weight_dict, output_expr=None,
                            extra_keys=()) -> Dict[str, torch.Tensor]:
        """Losses of one constraint (label keys in order; a key without an expression is the output) and their gradient
        accumulated into ``self.flat.grad``, through the operator jet head.  A constraint without derivatives compiles
        to a values-only head (no trunk jets)."""
        self._check_fused(loss_fn)
        return self._jet_train_forward(loss_fn, input_dict, label_dict, weight_dict, output_expr, extra_keys)
