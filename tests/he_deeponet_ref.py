"""Oracle for ``HEDeepONets``: a torch-CPU restatement of the reference's forward (ppsci/arch/he_deeponets.py), built
from the sub-network and activation restatements of ``oracle/ppsci_oracle.py``.  Autograd over it supplies the x and t
derivatives ``O.train_forward_backward`` needs."""
from typing import Dict, Sequence

import torch

from oracle.ppsci_oracle import OracleDeepONet, get_activation


class OracleHEDeepONets:
    """Functional HEDeepONets over one flat buffer laid out [heat | cold | trunk | b(3)], each sub-network starting at a
    multiple of 4 and laid out like OracleMLP.  heat_net / cold_net: MLP(input_dim=*_num_loc, output_dim=3F) on the
    branch inputs (he_deeponets.py:107-127); trunk_net: MLP(input_dim=len(trunk_input_keys), output_dim=3F) on the
    trunk inputs side by side (he_deeponets.py:129-139), followed by the trunk activation (he_deeponets.py:165);
    G_k = sum over features kF .. (k+1)F - 1 of heat * act(trunk) * cold, plus b[k] (he_deeponets.py:167-186).  The
    branch activations are built but never applied to the branch outputs (he_deeponets.py:141-142).  ``effective``
    optionally maps (flat, sub-network index, its parameter slice) to the effective [W | b] of a reparametrised
    sub-network."""

    def __init__(self, heat_input_keys, cold_input_keys, trunk_input_keys, output_keys, heat_num_loc: int, cold_num_loc: int,
                 num_features: int, branch_hidden: Sequence[int], trunk_hidden: Sequence[int],
                 branch_activation: str = "tanh", trunk_activation: str = "tanh", use_bias: bool = True, effective=None):
        self.heat_keys, self.cold_keys, self.trunk_keys = tuple(heat_input_keys), tuple(cold_input_keys), tuple(trunk_input_keys)
        self.input_keys = self.trunk_keys + self.heat_keys + self.cold_keys  # he_deeponets.py:98-100
        self.output_keys = tuple(output_keys)
        self.F = num_features
        width = 3 * num_features
        self.widths = [[heat_num_loc] + list(branch_hidden) + [width], [cold_num_loc] + list(branch_hidden) + [width],
                       [len(self.trunk_keys)] + list(trunk_hidden) + [width]]
        self.bact, self.tact = get_activation(branch_activation), get_activation(trunk_activation)
        self.use_bias = use_bias
        self.effective = effective
        self.los, lo = [], 0
        for w in self.widths:
            self.los.append(lo)
            n = sum(a * b + b for a, b in zip(w[:-1], w[1:]))
            lo = (lo + n + 3) // 4 * 4
        self.bias_off = lo

    def __call__(self, flat: torch.Tensor, x: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        subs = []
        for j, w in enumerate(self.widths):
            n = sum(a * b + b for a, b in zip(w[:-1], w[1:]))
            p = flat[self.los[j]: self.los[j] + n]
            subs.append(self.effective(flat, j, p) if self.effective is not None else p)
        cat = lambda keys: torch.cat([x[k] for k in keys], dim=1)  # noqa: E731  (MLP.concat_to_tensor)
        heat = OracleDeepONet._mlp(subs[0], self.widths[0], self.bact, cat(self.heat_keys))
        cold = OracleDeepONet._mlp(subs[1], self.widths[1], self.bact, cat(self.cold_keys))
        y = self.tact(OracleDeepONet._mlp(subs[2], self.widths[2], self.tact, cat(self.trunk_keys)))
        F = self.F
        out = {}
        for k, key in enumerate(self.output_keys):
            g = (heat[:, k * F:(k + 1) * F] * y[:, k * F:(k + 1) * F] * cold[:, k * F:(k + 1) * F]).sum(dim=1, keepdim=True)
            out[key] = g + flat[self.bias_off + k] if self.use_bias else g
        return out
