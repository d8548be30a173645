"""Oracle for ``ChipDeepONets``: a torch-CPU restatement of the reference's forward (ppsci/arch/chip_deeponets.py), built
from the sub-network and activation restatements of ``oracle/ppsci_oracle.py``, and an evaluator of sympy residuals
with ``Piecewise`` / ``Eq`` nodes (the form ``where(bc == k, a, b)`` traces to) on top of ``eval_expr``."""
from typing import Dict, Sequence

import sympy as sp
import torch

from oracle.ppsci_oracle import OracleDeepONet, eval_expr, get_activation


class OracleChipDeepONets:
    """Functional ChipDeepONets over one flat buffer laid out [branch | BCtype | BC | trunk | b], each sub-network starting
    at a multiple of 4 and laid out like OracleMLP.  branch_net: MLP(input_dim=num_loc, output_dim=F) with the branch
    settings; BCtype_net / BC_net: MLP(input_dim=bctype_loc / BC_num_loc, output_dim=F) with the BC settings
    (chip_deeponets.py:126-159); trunk_net: MLP(input_dim=len(trunk_input_keys), output_dim=F) followed by the trunk
    activation (chip_deeponets.py:161-185); G = sum(u * act(trunk) * bc * bctype) + b (chip_deeponets.py:186-193).  The
    branch activations are built but never applied to the branch outputs (chip_deeponets.py:172-173).  ``effective``
    optionally maps (flat, sub-network index, its parameter slice) to the effective [W | b] of a reparametrised
    sub-network."""

    def __init__(self, branch_input_keys, BCtype_input_keys, BC_input_keys, trunk_input_keys, output_keys, num_loc: int,
                 bctype_loc: int, BC_num_loc: int, num_features: int, branch_hidden: Sequence[int],
                 BC_hidden: Sequence[int], trunk_hidden: Sequence[int], branch_activation: str = "tanh",
                 BC_activation: str = "tanh", trunk_activation: str = "tanh", use_bias: bool = True, effective=None):
        self.keys = [tuple(branch_input_keys), tuple(BCtype_input_keys), tuple(BC_input_keys), tuple(trunk_input_keys)]
        self.input_keys = self.keys[3] + self.keys[0] + self.keys[2] + self.keys[1]  # chip_deeponets.py:118-123
        self.output_keys = tuple(output_keys)
        F = num_features
        self.widths = [[num_loc] + list(branch_hidden) + [F], [bctype_loc] + list(BC_hidden) + [F],
                       [BC_num_loc] + list(BC_hidden) + [F], [len(self.keys[3])] + list(trunk_hidden) + [F]]
        self.acts = [get_activation(branch_activation), get_activation(BC_activation), get_activation(BC_activation),
                     get_activation(trunk_activation)]
        self.use_bias = use_bias
        self.effective = effective
        self.los, lo = [], 0
        for w in self.widths:
            self.los.append(lo)
            n = sum(a * b + b for a, b in zip(w[:-1], w[1:]))
            lo = (lo + n + 3) // 4 * 4
        self.bias_off = lo

    def __call__(self, flat: torch.Tensor, x: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        feats = []
        for j, w in enumerate(self.widths):
            n = sum(a * b + b for a, b in zip(w[:-1], w[1:]))
            p = flat[self.los[j]: self.los[j] + n]
            p = self.effective(flat, j, p) if self.effective is not None else p
            feats.append(OracleDeepONet._mlp(p, w, self.acts[j], torch.cat([x[k] for k in self.keys[j]], dim=1)))
        u, bctype, bc, t = feats
        g = (u * self.acts[3](t) * bc * bctype).sum(dim=1, keepdim=True)
        return {self.output_keys[0]: g + flat[self.bias_off] if self.use_bias else g}


def eval_piecewise(expr: sp.Basic, data: Dict[str, torch.Tensor]) -> torch.Tensor:
    """``eval_expr`` that also evaluates ``Piecewise((a, Eq(l, r)), ..., (z, True))`` as nested ``torch.where`` (what
    paddle.where computes): every Piecewise node is evaluated on its own and handed to ``eval_expr`` as a column."""
    cols = dict(data)

    def ev_pw(pw: sp.Piecewise) -> torch.Tensor:
        (val, cond), rest = pw.args[0], pw.args[1:]
        if cond == sp.true:
            return eval_piecewise(val, cols)
        assert isinstance(cond, sp.Eq), cond
        c = eval_piecewise(cond.lhs, cols) == eval_piecewise(cond.rhs, cols)
        return torch.where(c, eval_piecewise(val, cols), ev_pw(sp.Piecewise(*rest)) if len(rest) > 1 or rest[0][1] != sp.true
                           else eval_piecewise(rest[0][0], cols))

    subs = {}
    for pw in expr.atoms(sp.Piecewise):
        if any(o is not pw and o.has(pw) for o in expr.atoms(sp.Piecewise)):
            continue  # evaluated inside its enclosing Piecewise
        name = f"_pw{len(subs)}"
        cols[name] = ev_pw(pw)
        subs[pw] = sp.Symbol(name)
    return eval_expr(expr.xreplace(subs), cols)
