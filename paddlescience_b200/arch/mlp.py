"""``MLP`` with the reference's constructor (ppsci/arch/mlp.py:179-315) whose forward — values and
input derivatives alike — runs in the native jet kernels.

Parameters live in ONE flat fp32/fp64 buffer laid out [W_1 (in,out) | b_1 | W_2 | b_2 | ...]
(the reference's nn.Linear layout is [in,out], mlp.py:246,274).  ``linears[i].weight`` /
``.bias`` / ``last_fc`` are views into it, and ``state_dict()`` uses the reference's key names
(``linears.0.weight`` ...) so checkpoints translate 1:1.

``weight_norm=True`` (reference: ``WeightNormLinear``, mlp.py:31-53, used by the hidden layers): the trainable
vector is ``[V_1 | b_1 | ... | W_last | b_last | g_1 ... g_{L-1}]`` and the buffer the kernels read holds the
effective weights ``W_l = g_l * V_l / ||V_l||_col``; the engine call is unchanged, the reparametrisation and its
chain rule are a handful of column-wise torch operations on the (small) weight matrices before / after it
(``engine_params`` / ``engine_grads`` / ``finish_grads``).
"""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import Dict, List, Optional, Tuple, Union

import numpy as np
import torch
from torch import nn

from ..engine.compiler import NetSpec, compile_residuals
from . import activation as act_mod
from . import base


class _LinearView:
    """View of one layer inside the flat parameter buffer."""

    def __init__(self, owner: "MLP", index: int):
        self._owner = owner
        self._index = index

    @property
    def weight(self) -> torch.Tensor:
        """Effective weight [in, out] (a view for plain layers, g * V / ||V||_col for weight-normalised ones)."""
        a, b = self._owner._shapes[self._index]
        off = self._owner._w_off[self._index]
        v = self._owner.flat.data[off: off + a * b].view(a, b)
        if self._owner._wn_layer(self._index):
            if self._owner.random_weight:
                return v * self.weight_g
            return v * (self.weight_g / v.norm(p=2, dim=0, keepdim=True))
        return v

    @property
    def weight_v(self) -> torch.Tensor:
        if not self._owner._wn_layer(self._index):
            raise AttributeError("weight_v exists only for weight-normalised layers")
        a, b = self._owner._shapes[self._index]
        off = self._owner._w_off[self._index]
        return self._owner.flat.data[off: off + a * b].view(a, b)

    @property
    def weight_g(self) -> torch.Tensor:
        if not self._owner._wn_layer(self._index):
            raise AttributeError("weight_g exists only for weight-normalised layers")
        off = self._owner._g_off[self._index]
        return self._owner.flat.data[off: off + self._owner._shapes[self._index][1]]

    @property
    def bias(self) -> torch.Tensor:
        a, b = self._owner._shapes[self._index]
        off = self._owner._b_off[self._index]
        return self._owner.flat.data[off: off + b]

    @property
    def weight_grad(self) -> Optional[torch.Tensor]:
        g = self._owner.flat.grad
        if g is None:
            return None
        a, b = self._owner._shapes[self._index]
        off = self._owner._w_off[self._index]
        return g[off: off + a * b].view(a, b)

    @property
    def bias_grad(self) -> Optional[torch.Tensor]:
        g = self._owner.flat.grad
        if g is None:
            return None
        a, b = self._owner._shapes[self._index]
        off = self._owner._b_off[self._index]
        return g[off: off + b]


class MLP(base.Arch):
    """Multi layer perceptron network (same arguments as the reference, mlp.py:179-193).

    ``weight_norm``, ``random_weight`` and ``skip_connection`` are host-side reparametrisations around the unchanged
    engine call (effective [W | b] before it, chain rule after it).  ``fourier={"dim": D, "scale": s}``
    (FourierEmbedding, mlp.py:117-136, applied after the period embedding, mlp.py:298-315) is one more linear layer
    for the kernels: ``[cos(x B), sin(x B)] = sin(x [B | B] + [pi/2 | 0])`` — tied effective weights, a constant bias
    and ``sin`` as that layer's activation (``NetSpec.act_first``); the gradient of the trainable kernel ``B`` is the
    sum of the two halves of the effective layer's weight gradient.  Not yet supported (raise ``NotImplementedError``
    at construction): trainable periods.  ``fourier`` composes with weight_norm / random_weight / skip_connection (one
    staging buffer: the tied first layer in front of the reparametrised linear layers).
    """

    # 1: ModifiedMLP (two embedding layers + the gate after every hidden layer); 2: PirateNet (blocks of three layers,
    # gates after the first two, adaptive residual after the third; the embeddings read the Fourier features)
    _gated = 0

    def __init__(
        self,
        input_keys: Tuple[str, ...],
        output_keys: Tuple[str, ...],
        num_layers: Optional[int],
        hidden_size: Union[int, Tuple[int, ...]],
        activation: str = "tanh",
        skip_connection: bool = False,
        weight_norm: bool = False,
        input_dim: Optional[int] = None,
        output_dim: Optional[int] = None,
        periods: Optional[Dict[str, Tuple[float, bool]]] = None,
        fourier: Optional[Dict[str, Union[float, int]]] = None,
        random_weight: Optional[Dict[str, float]] = None,
        dtype: torch.dtype = torch.float32,
    ):
        super().__init__()
        self.input_keys = tuple(input_keys)
        self.output_keys = tuple(output_keys)
        self.periods = dict(periods) if periods else None
        if isinstance(hidden_size, (tuple, list)):
            if num_layers is not None:
                raise ValueError("num_layers should be None when hidden_size is specified")
            hidden = [int(h) for h in hidden_size]
        elif isinstance(hidden_size, int):
            if not isinstance(num_layers, int):
                raise ValueError("num_layers should be an int when hidden_size is an int")
            hidden = [hidden_size] * num_layers
        else:
            raise ValueError(f"hidden_size should be list of int or int, but got {type(hidden_size)}")
        self.weight_norm = bool(weight_norm)
        self.fourier = dict(fourier) if fourier else None
        if self.fourier:
            if int(self.fourier["dim"]) % 2 != 0:  # FourierEmbedding.__init__, mlp.py:120-121
                raise ValueError(f"out_features must be even, but got {self.fourier['dim']}.")
        # random_weight = {"mean": m, "std": s}: RandomWeightFactorization on EVERY layer incl. last_fc (mlp.py:56-92,
        # 248-256, 262-270): W = g * V (column scaling), g = exp(N(m, s)), V = glorot_normal / g
        self.random_weight = dict(random_weight) if random_weight else None
        if (skip_connection or self.random_weight) and weight_norm:
            raise NotImplementedError("weight_norm cannot be combined with skip_connection / random_weight (the reference "
                                      "picks weight_norm first, mlp.py:238-250)")
        if skip_connection and self.random_weight:
            raise NotImplementedError("MLP(skip_connection=True, random_weight=...) is not supported yet")
        if input_dim is not None and input_dim != len(self.input_keys) + (len(self.periods) if self.periods else 0):
            raise NotImplementedError("input_dim different from the (period-embedded) key count is not supported")
        if output_dim is not None and output_dim != len(self.output_keys):
            raise NotImplementedError("output_dim different from len(output_keys) is not supported")
        self.activation = act_mod.get_activation(activation)
        # features: period-embedded keys expand to (cos, sin)  (mlp.py:108-114, base.py:109-112)
        feat_src: List[int] = []
        feat_kind: List[int] = []
        feat_omega: List[float] = []
        for i, k in enumerate(self.input_keys):
            if self.periods and k in self.periods:
                p, trainable = self.periods[k]
                if trainable:
                    raise NotImplementedError("trainable periods are not supported by the jet kernels yet")
                w = 2 * np.pi / float(p)
                feat_src += [i, i]
                feat_kind += [1, 2]
                feat_omega += [w, w]
            else:
                feat_src.append(i)
                feat_kind.append(0)
                feat_omega.append(0.0)
        if self.periods:
            for k in self.periods:
                if k not in self.input_keys:
                    raise KeyError(f"period key {k} is not an input key")
        widths = [len(feat_src)] + hidden + [len(self.output_keys)]
        eng_widths = widths
        if self.fourier:  # the embedding is layer 1 of the network the kernels see; the reference's own layers start at D
            d_f = int(self.fourier["dim"])
            eng_widths = [len(feat_src), d_f] + hidden + [len(self.output_keys)]
            widths = [d_f] + hidden + [len(self.output_keys)]
        # trainable activation parameters: Stan's beta per unit (activation.py:28-46), Swish's beta per layer (:49-58)
        self._beta_len = {"stan": list(hidden), "swish": [1] * len(hidden)}.get(self.activation, [])
        if self._beta_len and self._gated:
            raise NotImplementedError(f"{type(self).__name__}(activation={self.activation!r}): activations with a trainable "
                                      "parameter are supported by the plain MLP plans only")
        self._net = NetSpec(self.input_keys, self.output_keys, feat_src, feat_kind, feat_omega, eng_widths,
                            {"swish": "swish_b"}.get(self.activation, self.activation),
                            act_first="sin" if self.fourier else None, gated=int(self._gated))
        self._shapes = list(zip(widths[:-1], widths[1:]))
        self._n_hidden = len(hidden)
        if self._gated:  # embed_u / embed_v (n_feat -> hidden[0]) stored behind last_fc: [... | Wu | bu | Wv | bv]
            if len(set(hidden)) != 1:
                raise ValueError("ModifiedMLP takes one hidden_size for all layers")
            self._shapes += [(widths[0], hidden[0])] * 2
        self._w_off, self._b_off = [], []
        off = 0
        for a, b in self._shapes:
            self._w_off.append(off)
            off += a * b
            self._b_off.append(off)
            off += b
        self._alpha_off, self._n_blocks = off, 0
        if self._gated == 2:  # PirateNetBlock.alpha, one trainable scalar per block (mlp.py:592-597), behind the embeddings
            self._n_blocks = len(hidden) // 3
            off += self._n_blocks
        self._beta_off = []
        for n_b in self._beta_len:  # acts.i.beta, behind the alphas (the engine's order: hidden layer by hidden layer)
            self._beta_off.append(off)
            off += n_b
        self._n_eff = off  # length of the [W | b] buffer of the reference's own linear layers
        self._n_lin = off
        self._f_n0 = 0     # fourier: length of the effective first layer [W0 | b0] in front of them in the engine buffer
        self._g_off = {}   # weight_norm / random_weight: layer index -> offset of its gain vector g (behind the last bias)
        if self.weight_norm or self.random_weight:
            for i, (a, b) in enumerate(self._shapes):
                if self._wn_layer(i):
                    self._g_off[i] = off
                    off += b
        if self.fourier:  # trainable kernel B [n_feat, D/2] stored behind the linear layers
            nf, dh = len(feat_src), int(self.fourier["dim"]) // 2
            self._f_shape = (nf, dh)
            self._f_off = off
            off += nf * dh
            self._f_n0 = nf * 2 * dh + 2 * dh
        self.flat = nn.Parameter(torch.zeros(off, dtype=dtype))
        self.linears = [_LinearView(self, i) for i in range(len(hidden))]
        self.last_fc = _LinearView(self, len(hidden))
        if self._gated:
            self.embed_u = _LinearView(self, len(hidden) + 1)
            self.embed_v = _LinearView(self, len(hidden) + 2)
        # Reference semantics of skip_connection (mlp.py:281-296), restated exactly: at every even hidden layer i >= 2
        # the code executes ``skip = y; y = y + skip`` — the freshly assigned skip IS y, so the pre-activation is
        # doubled (the first even layer only records skip).  A doubled pre-activation is the same linear layer with
        # W and b scaled by 2: the kernels read effective weights 2 W_i, 2 b_i for those layers and the chain rule
        # returns 2 x their gradients (host-side reparametrisation, like weight_norm).
        # ModifiedMLP (mlp.py:495-504) doubles the GATED output of those layers instead (``y = y + skip`` behind the
        # gate): the next linear layer sees 2 y, i.e. its weight (not its bias) is doubled.
        self.skip_connection = bool(skip_connection)
        self._skip_layers = [i for i in range(len(hidden)) if self.skip_connection and i % 2 == 0 and i >= 2]
        # the engine reads effective weights from a staging buffer [W0 | b0 (fourier) | reparametrised linear layers]
        self._has_eff = bool(self.weight_norm or self.random_weight or self.fourier or self._skip_layers)
        if self._has_eff:
            self.register_buffer("_eff", torch.zeros(self._f_n0 + self._n_eff, dtype=dtype), persistent=False)
            self.register_buffer("_eff_grad", torch.zeros(self._f_n0 + self._n_eff, dtype=dtype), persistent=False)
        self.reset_parameters()
        self._value_plan = None

    # ---- parameters ------------------------------------------------------------------------
    def reset_parameters(self):
        """Xavier-uniform weights, zero bias (Paddle's nn.Linear default initialisers)."""
        with torch.no_grad():
            for i, (a, b) in enumerate(self._shapes):
                lim = math.sqrt(6.0 / (a + b))
                w = (torch.rand(a * b, dtype=torch.float64) * 2 - 1) * lim
                if self.activation == "siren" and i < self._n_hidden:
                    # Siren.init_for_first_layer / init_for_hidden_layer (activation.py:103-136, applied in mlp.py:256-260)
                    lim = 1.0 / a if i == 0 else math.sqrt(6.0 / a) / 30.0
                    w = (torch.rand(a * b, dtype=torch.float64) * 2 - 1) * lim
                self.flat.data[self._w_off[i]: self._w_off[i] + a * b] = w.to(self.flat.dtype)
                self.flat.data[self._b_off[i]: self._b_off[i] + b] = 0
                if self._wn_layer(i) and not self.random_weight:  # WeightNormLinear._init_weights: V xavier-uniform, g = 1, bias = 0
                    self.flat.data[self._g_off[i]: self._g_off[i] + b] = 1
                if self.random_weight:  # RandomWeightFactorization._init_weights (mlp.py:77-88)
                    v = torch.randn(a, b, dtype=torch.float64) * math.sqrt(2.0 / (a + b))  # glorot normal
                    g = torch.exp(self.random_weight["mean"] + self.random_weight["std"] * torch.randn(b, dtype=torch.float64))
                    self.flat.data[self._w_off[i]: self._w_off[i] + a * b] = (v / g).reshape(-1).to(self.flat.dtype)
                    self.flat.data[self._g_off[i]: self._g_off[i] + b] = g.to(self.flat.dtype)

            for o, n_b in zip(self._beta_off, self._beta_len):  # Constant(1) (activation.py:38-41), Swish(beta=1.0)
                self.flat.data[o: o + n_b] = 1
            if self._n_blocks:  # alpha = 0: every block starts as the identity (mlp.py:592-597)
                self.flat.data[self._alpha_off: self._alpha_off + self._n_blocks] = 0
            if self.fourier:  # FourierEmbedding: Normal(std=scale) (mlp.py:123-126)
                nf, dh = self._f_shape
                k = torch.randn(nf * dh, dtype=torch.float64) * float(self.fourier["scale"])
                self.flat.data[self._f_off: self._f_off + nf * dh] = k.to(self.flat.dtype)

    @property
    def fourier_kernel(self) -> torch.Tensor:
        """View of the FourierEmbedding kernel B [n_feat, D/2] (``fourier_emb.kernel`` in the reference)."""
        nf, dh = self._f_shape
        return self.flat.data[self._f_off: self._f_off + nf * dh].view(nf, dh)

    def net_spec(self) -> NetSpec:
        return self._net

    # ---- what the engine reads / accumulates into ---------------------------------------------------
    def _wn_layer(self, i: int) -> bool:
        """Layer i is stored factored as (weight_v, weight_g): weight-normalised hidden layers (mlp.py:234-246; last_fc is
        plain) or every layer under random weight factorization."""
        if self.random_weight:
            return True
        return self.weight_norm and i != self._n_hidden  # hidden layers (and the gated networks' embed_u / embed_v)

    def _skip_slices(self):
        """(start, stop) ranges of the staging buffer that the reference's skip connection doubles."""
        out = []
        for i in self._skip_layers:
            if self._gated:  # the layer BEHIND hidden layer i reads 2 y: its weight
                a, b = self._shapes[i + 1]
                out.append((self._w_off[i + 1], self._w_off[i + 1] + a * b))
            else:  # the pre-activation of hidden layer i is doubled: W_i and b_i (contiguous)
                a, b = self._shapes[i]
                out.append((self._w_off[i], self._b_off[i] + b))
        return out

    def engine_params(self) -> torch.Tensor:
        """The flat [W_1 | b_1 | ...] buffer passed to the native calls (effective weights under weight_norm /
        random_weight / skip_connection, the tied first layer of the Fourier embedding in front)."""
        if not self._has_eff:
            return self.flat.data
        with torch.no_grad():
            lin = self._eff[self._f_n0: self._f_n0 + self._n_eff]
            lin.copy_(self.flat.data[: self._n_eff])
            for i, (a, b) in enumerate(self._shapes):
                if not self._wn_layer(i):
                    continue
                v = self.flat.data[self._w_off[i]: self._w_off[i] + a * b].view(a, b)
                g = self.flat.data[self._g_off[i]: self._g_off[i] + b]
                scale = g if self.random_weight else g / v.norm(p=2, dim=0, keepdim=True)
                lin[self._w_off[i]: self._w_off[i] + a * b].view(a, b).copy_(v * scale)
            for lo, hi in self._skip_slices():
                lin[lo:hi].mul_(2.0)
            if self.fourier:
                nf, dh = self._f_shape
                k = self.fourier_kernel
                w0 = self._eff[: nf * 2 * dh].view(nf, 2 * dh)
                w0[:, :dh].copy_(k)
                w0[:, dh:].copy_(k)
                b0 = self._eff[nf * 2 * dh: self._f_n0]
                b0[:dh] = math.pi / 2  # cos(z) = sin(z + pi/2)
                b0[dh:] = 0
        return self._eff

    def engine_grads(self) -> torch.Tensor:
        """Buffer the native calls accumulate the weight gradient into (same layout as ``engine_params``)."""
        if self.flat.grad is None:
            self.flat.grad = torch.zeros_like(self.flat.data)
        return self._eff_grad if self._has_eff else self.flat.grad

    def finish_grads(self):
        """Chain rule of the reparametrisations: gradients w.r.t. the effective weights -> the stored parameters
        ((V, g), the tied Fourier kernel, the doubled layers); then the staging buffer is cleared.  No-op for plain
        layers (the kernels accumulated into ``flat.grad`` directly)."""
        if not self._has_eff:
            return
        with torch.no_grad():
            gr = self.flat.grad
            lin_g = self._eff_grad[self._f_n0: self._f_n0 + self._n_eff]
            for lo, hi in self._skip_slices():
                lin_g[lo:hi].mul_(2.0)  # d/dW = 2 d/dW_eff
            gr[: self._n_eff] += lin_g  # biases and plain layers pass through; the V parts are fixed below
            for i, (a, b) in enumerate(self._shapes):
                if not self._wn_layer(i):
                    continue
                sl = slice(self._w_off[i], self._w_off[i] + a * b)
                v = self.flat.data[sl].view(a, b)
                g = self.flat.data[self._g_off[i]: self._g_off[i] + b]
                dw = lin_g[sl].view(a, b)
                if self.random_weight:  # W = g * V  ->  dV = g * dW,  dg = sum_in V * dW
                    gr[sl].view(a, b).add_(g * dw - dw)
                    gr[self._g_off[i]: self._g_off[i] + b] += (v * dw).sum(dim=0)
                    continue
                norm = v.norm(p=2, dim=0, keepdim=True)
                dot = (dw * v).sum(dim=0, keepdim=True)  # [1, out]
                dv = (g / norm) * (dw - v * (dot / (norm * norm)))
                gr[sl].view(a, b).add_(dv - dw)  # replace the pass-through dW by dV
                gr[self._g_off[i]: self._g_off[i] + b] += (dot / norm).view(-1)
            if self.fourier:  # the tied kernel takes the sum of both halves; the constant bias [pi/2 | 0] takes none
                nf, dh = self._f_shape
                dw0 = self._eff_grad[: nf * 2 * dh].view(nf, 2 * dh)
                gr[self._f_off: self._f_off + nf * dh].view(nf, dh).add_(dw0[:, :dh] + dw0[:, dh:])
            self._eff_grad.zero_()

    @property
    def dtype(self) -> torch.dtype:
        return self.flat.dtype

    def _layer_names(self):
        names = [f"linears.{i}" for i in range(self._n_hidden)] + ["last_fc"]
        if self._gated:  # nn.Sequential(Linear, act): the linear layer is item 0 (mlp.py:397-438)
            names += ["embed_u.0", "embed_v.0"]
        return names

    def _views(self):
        return self.linears + [self.last_fc] + ([self.embed_u, self.embed_v] if self._gated else [])

    def state_dict(self, *args, **kwargs):  # reference-style keys
        out = OrderedDict()
        views = self._views()
        for i, (name, v) in enumerate(zip(self._layer_names(), views)):
            if self._wn_layer(i):
                out[f"{name}.weight_v"] = v.weight_v.detach().clone()
                out[f"{name}.weight_g"] = v.weight_g.detach().clone()
            else:
                out[f"{name}.weight"] = v.weight.detach().clone()
            out[f"{name}.bias"] = v.bias.detach().clone()
        for i, (o, n_b) in enumerate(zip(self._beta_off, self._beta_len)):  # acts is a LayerList of Stan / Swish layers
            b = self.flat.data[o: o + n_b].detach().clone()
            out[f"acts.{i}.beta"] = b if self.activation == "stan" else b.reshape(())
        if self.fourier:
            out["fourier_emb.kernel"] = self.fourier_kernel.detach().clone()
        return out

    def load_state_dict(self, state_dict, strict: bool = True):
        views = self._views()
        known = self._layer_names() + (["fourier_emb"] if self.fourier else []) + [f"acts.{i}" for i in range(len(self._beta_off))]
        missing, unexpected = [], [k for k in state_dict if k.rsplit(".", 1)[0] not in known]
        with torch.no_grad():
            for i, (o, n_b) in enumerate(zip(self._beta_off, self._beta_len)):
                key = f"acts.{i}.beta"
                if key not in state_dict:
                    missing.append(key)
                    continue
                src = state_dict[key]
                src = torch.as_tensor(np.asarray(src.cpu() if hasattr(src, "cpu") else src)).reshape(-1)
                self.flat.data[o: o + n_b].copy_(src.to(self.flat.dtype).to(self.flat.device))
            if self.fourier:
                if "fourier_emb.kernel" in state_dict:
                    src = state_dict["fourier_emb.kernel"]
                    src = torch.as_tensor(np.asarray(src.cpu() if hasattr(src, "cpu") else src))
                    self.fourier_kernel.copy_(src.to(self.flat.dtype).to(self.flat.device))
                else:
                    missing.append("fourier_emb.kernel")
            for i, (name, v) in enumerate(zip(self._layer_names(), views)):
                for part in (("weight_v", "weight_g", "bias") if self._wn_layer(i) else ("weight", "bias")):
                    key = f"{name}.{part}"
                    if key not in state_dict:
                        missing.append(key)
                        continue
                    src = torch.as_tensor(np.asarray(state_dict[key].cpu() if hasattr(state_dict[key], "cpu") else state_dict[key]))
                    getattr(v, part).copy_(src.to(self.flat.dtype).to(self.flat.device))
        if strict and (missing or unexpected):
            raise KeyError(f"missing keys {missing}, unexpected keys {unexpected}")
        return missing, unexpected

    set_state_dict = load_state_dict

    # ---- forward (values only) -----------------------------------------------------------------
    def _plan_values(self):
        from ..engine.plan import ResidualPlan

        if self._value_plan is None or self._value_plan.dtype != self.flat.dtype:
            cr = compile_residuals(self._net, {}, with_grad=False)
            self._value_plan = ResidualPlan(cr, self.flat.dtype, [], [])
        return self._value_plan

    def forward_tensor(self, x: torch.Tensor) -> torch.Tensor:
        """Values of the network for a concatenated (already embedded) input is not offered: the
        kernels read the raw columns.  Use ``forward`` with the input dict."""
        raise NotImplementedError("use MLP.forward(input_dict); the native kernels read the raw input columns")

    def forward(self, x: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if self._input_transform is not None:
            x = self._input_transform(x)
        first = x[self.input_keys[0]]
        if first.device.type != "cuda" or self.flat.device != first.device:
            raise RuntimeError(
                "paddlescience_b200.arch.MLP.forward runs only on a CUDA (H100) device: the engine has no "
                f"CPU fallback (inputs on {first.device}, parameters on {self.flat.device})")
        plan = self._plan_values()
        cols = {k: x[k].to(self.flat.dtype) for k in self.input_keys}
        jets, _ = plan.forward(cols, self.engine_params(), want_jets=True, want_residuals=False)
        y = jets[0]  # [N, n_out]
        shape = tuple(first.shape[:-1]) + (1,) if first.dim() > 1 else (first.numel(), 1)
        out = {k: y[:, j].reshape(shape) for j, k in enumerate(self.output_keys)}
        if self._output_transform is not None:
            out = self._output_transform(x, out)
        return out


class ModifiedMLP(MLP):
    """Modified multi layer perceptron (https://arxiv.org/pdf/2001.04536.pdf) — same arguments as the reference
    (mlp.py:318-487).  ``forward_tensor`` of the reference (mlp.py:488-506):

        u = act(embed_u(x)); v = act(embed_v(x))
        for linear: y = act(linear(y)); y = y * u + (1 - y) * v
        y = last_fc(y)

    runs inside the engine as a gated plan (``ppsci_plan_spec.gated``): two more first layers from the same seeds and a
    jet-product gate after every hidden layer (csrc/kernels_gate.cuh), values, input derivatives of any supported order
    and the weight gradient included.  The flat parameter vector is ``[W_1 | b_1 | ... | last_fc | Wu | bu | Wv | bv]``;
    checkpoints use the reference's keys (``linears.i.*``, ``last_fc.*``, ``embed_u.0.*``, ``embed_v.0.*``).
    With ``fourier`` the embedding is the engine's first layer and ``embed_u`` / ``embed_v`` read its stored output
    (any ``fourier["dim"]``).  ``periods``, ``fourier``, ``weight_norm`` (hidden layers and both embeddings),
    ``random_weight`` (every layer) and ``skip_connection`` (the reference's ``y = y + skip`` behind the gate, i.e. a
    doubled input of the next layer) are host-side reparametrisations as in ``MLP``; ``skip_connection`` together with
    weight_norm / random_weight raises ``NotImplementedError``."""

    _gated = 1

    def __init__(
        self,
        input_keys: Tuple[str, ...],
        output_keys: Tuple[str, ...],
        num_layers: int,
        hidden_size: int,
        activation: str = "tanh",
        skip_connection: bool = False,
        weight_norm: bool = False,
        input_dim: Optional[int] = None,
        output_dim: Optional[int] = None,
        periods: Optional[Dict[str, Tuple[float, bool]]] = None,
        fourier: Optional[Dict[str, Union[float, int]]] = None,
        random_weight: Optional[Dict[str, float]] = None,
        dtype: torch.dtype = torch.float32,
    ):
        if not isinstance(hidden_size, int):  # mlp.py:381-382
            raise ValueError(f"hidden_size should be int, but got {type(hidden_size)}")
        if not isinstance(num_layers, int):  # mlp.py:378-379
            raise ValueError("num_layers should be an int")
        if num_layers < 1:
            raise ValueError("ModifiedMLP needs at least one hidden layer (embed_u / embed_v map onto hidden_size)")
        if skip_connection and (weight_norm or random_weight):
            raise NotImplementedError("ModifiedMLP(skip_connection=True) together with weight_norm / random_weight is not "
                                      "supported yet")
        super().__init__(input_keys, output_keys, num_layers, hidden_size, activation, skip_connection, weight_norm,
                         input_dim, output_dim, periods, fourier, random_weight, dtype)


class PirateNet(MLP):
    """PirateNet (https://arxiv.org/pdf/2402.00326.pdf) — same arguments as the reference (mlp.py:627-798).
    ``forward_tensor`` (mlp.py:800-809) over ``PirateNetBlock.forward`` (mlp.py:617-624):

        u = act(embed_u(x)); v = act(embed_v(x))                       # x = the Fourier features
        per block:  f = act(linear1(x)); z1 = f u + (1 - f) v
                    g = act(linear2(z1)); z2 = g u + (1 - g) v
                    h = act(linear3(z2)); x = alpha h + (1 - alpha) x   # alpha: trainable scalar, 0 at start
        y = last_fc(x)

    runs inside the engine as a gated plan of kind 2 (``ppsci_plan_spec.gated``, csrc/kernels_gate.cuh): the Fourier
    embedding is the engine's first layer (tied weights, ``sin`` activation, like ``MLP(fourier=...)``), the gates and the
    adaptive residual are jet-level elementwise kernels between the linear layers, dLoss/dalpha is reduced on the device.
    The block input must have the blocks' width: ``fourier["dim"] == hidden_size`` (the reference's own constraint:
    ``PirateNetBlock(cur_size)`` adds its input to a ``cur_size``-wide output and multiplies it with ``hidden_size``-wide
    embeddings).  Flat parameter vector: ``[blocks' linears | last_fc | Wu | bu | Wv | bv | alphas | fourier kernel]``;
    checkpoints use the reference's keys (``blocks.k.linear{1,2,3}.*``, ``blocks.k.alpha``, ``embed_{u,v}.0.*``,
    ``last_fc.*``, ``fourier_emb.kernel``).  ``random_weight`` (every layer: the configuration of the reference's
    examples) and ``weight_norm`` (the two embeddings) are host-side reparametrisations as in ``MLP``; a PirateNet
    without ``fourier`` raises ``NotImplementedError``."""

    _gated = 2

    def __init__(
        self,
        input_keys: Tuple[str, ...],
        output_keys: Tuple[str, ...],
        num_blocks: int,
        hidden_size: int,
        activation: str = "tanh",
        weight_norm: bool = False,
        input_dim: Optional[int] = None,
        output_dim: Optional[int] = None,
        periods: Optional[Dict[str, Tuple[float, bool]]] = None,
        fourier: Optional[Dict[str, Union[float, int]]] = None,
        random_weight: Optional[Dict[str, float]] = None,
        dtype: torch.dtype = torch.float32,
    ):
        if not isinstance(hidden_size, int):  # mlp.py:700-705
            raise ValueError(f"hidden_size should be int, but got {type(hidden_size)}")
        if not isinstance(num_blocks, int):
            raise ValueError("num_blocks should be an int")
        if num_blocks < 1:
            raise ValueError("PirateNet needs at least one block")
        if not fourier:
            raise NotImplementedError("PirateNet without fourier features is not supported (the blocks need an input of "
                                      "their own width)")
        if int(fourier["dim"]) != hidden_size:
            raise ValueError(f"PirateNet blocks keep their input width: fourier['dim'] ({fourier['dim']}) must equal "
                             f"hidden_size ({hidden_size})")
        super().__init__(input_keys, output_keys, None, (hidden_size,) * (3 * num_blocks), activation, False, weight_norm,
                         input_dim, output_dim, periods, fourier, random_weight, dtype)

    def _wn_layer(self, i: int) -> bool:
        """random_weight factorises every layer (blocks, embeddings, last_fc); weight_norm only the two embeddings
        (mlp.py:722-759 — PirateNetBlock takes no weight_norm, last_fc is plain)."""
        if self.random_weight:
            return True
        return self.weight_norm and i > self._n_hidden

    @property
    def alphas(self) -> torch.Tensor:
        """View of the blocks' residual weights ``alpha`` [num_blocks]."""
        return self.flat.data[self._alpha_off: self._alpha_off + self._n_blocks]

    def _layer_names(self):
        return [f"blocks.{i // 3}.linear{i % 3 + 1}" for i in range(self._n_hidden)] + ["last_fc", "embed_u.0", "embed_v.0"]

    def state_dict(self, *args, **kwargs):
        out = super().state_dict(*args, **kwargs)
        for k in range(self._n_blocks):
            out[f"blocks.{k}.alpha"] = self.alphas[k: k + 1].detach().clone()
        return out

    def load_state_dict(self, state_dict, strict: bool = True):
        sd = dict(state_dict)
        missing = []
        with torch.no_grad():
            for k in range(self._n_blocks):
                key = f"blocks.{k}.alpha"
                if key in sd:
                    src = sd.pop(key)
                    src = torch.as_tensor(np.asarray(src.cpu() if hasattr(src, "cpu") else src)).reshape(-1)
                    self.alphas[k: k + 1].copy_(src.to(self.flat.dtype).to(self.flat.device))
                else:
                    missing.append(key)
        if strict and missing:
            raise KeyError(f"missing keys {missing}")
        m2, unexpected = super().load_state_dict(sd, strict)
        return missing + m2, unexpected

    set_state_dict = load_state_dict
