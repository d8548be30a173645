"""``DeepONet`` (reference: ppsci/arch/deeponet.py:28-154):  G(u)(y) = sum_i branch(u)_i * act(trunk(y))_i + b.

Both sub-networks run in the native kernels (values only, C = 1): the branch net reads its ``[N, num_loc]`` sensor
matrix as a dense first-layer operand (``dense_in``), the trunk net its coordinate column as an input seed.  The
combination, the loss and their derivatives are elementwise work on ``[N, num_features]`` done with torch on the
device; the weight gradients of the two MLPs come from ``ppsci_b200_values_fwd_bwd`` fed with dL/d(branch),
dL/d(trunk).  One flat parameter buffer  [branch | trunk | b]  so the flat optimizers apply unchanged."""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import Dict, List, Tuple, Union

import torch
from torch import nn

from ..engine.compiler import NetSpec, compile_residuals
from . import activation as act_mod
from . import base

_TORCH_ACT = {
    "tanh": torch.tanh, "sin": torch.sin, "cos": torch.cos, "sigmoid": torch.sigmoid, "silu": torch.nn.functional.silu,
    "swish": torch.nn.functional.silu, "gelu": torch.nn.functional.gelu, "relu": torch.relu, "identity": lambda t: t,
    "elu": torch.nn.functional.elu, "selu": torch.nn.functional.selu, "leaky_relu": torch.nn.functional.leaky_relu,
    "siren": lambda t: torch.sin(30.0 * t),
}


def _hidden(num_layers, hidden_size) -> List[int]:
    if isinstance(hidden_size, (tuple, list)):
        if num_layers is not None:
            raise ValueError("num_layers should be None when hidden_size is specified")
        return [int(h) for h in hidden_size]
    if not isinstance(num_layers, int):
        raise ValueError("num_layers should be an int when hidden_size is an int")
    return [int(hidden_size)] * num_layers


class _SubnetReparam:
    """Host-side reparametrisation of one sub-network around the unchanged native calls, exactly as ``arch.MLP`` does it:
    ``weight_norm`` (WeightNormLinear on the hidden layers, mlp.py:31-53, 234-246: W = g V / ||V||_col, stored as V in the
    weight slot and g behind the model's other parameters) and ``skip_connection`` (mlp.py:281-296 as executed: the
    pre-activation of every even hidden layer i >= 2 is doubled, i.e. effective 2 W_i, 2 b_i)."""

    def __init__(self, widths, lo: int, weight_norm: bool, skip: bool, g_off: int):
        self.shapes = list(zip(widths[:-1], widths[1:]))
        self.lo = lo
        self.weight_norm, self.skip = bool(weight_norm), bool(skip)
        self.w_off, self.b_off, off = [], [], 0
        for a, b in self.shapes:
            self.w_off.append(off)
            off += a * b
            self.b_off.append(off)
            off += b
        self.n = off
        n_hidden = len(self.shapes) - 1
        self.g_off = []  # absolute offsets of the gain vectors of the weight-normalised hidden layers
        for _, b in (self.shapes[:-1] if self.weight_norm else []):
            self.g_off.append(g_off)
            g_off += b
        self.g_end = g_off
        self.skip_layers = [i for i in range(n_hidden) if self.skip and i % 2 == 0 and i >= 2]
        self.active = self.weight_norm or bool(self.skip_layers)
        self.eff = self.eff_grad = None

    def params(self, flat: torch.Tensor) -> torch.Tensor:
        raw = flat.data[self.lo: self.lo + self.n]
        if not self.active:
            return raw
        if self.eff is None or self.eff.device != raw.device or self.eff.dtype != raw.dtype:
            self.eff, self.eff_grad = torch.empty_like(raw), torch.zeros_like(raw)
        with torch.no_grad():
            self.eff.copy_(raw)
            for i, (a, b) in enumerate(self.shapes[:-1]):
                w = self.eff[self.w_off[i]: self.w_off[i] + a * b].view(a, b)
                if self.weight_norm:
                    g = flat.data[self.g_off[i]: self.g_off[i] + b]
                    w.mul_(g / w.norm(p=2, dim=0, keepdim=True))
                if i in self.skip_layers:
                    self.eff[self.w_off[i]: self.b_off[i] + b].mul_(2.0)
        return self.eff

    def grads(self, flat: torch.Tensor) -> torch.Tensor:
        return self.eff_grad if self.active else flat.grad[self.lo: self.lo + self.n]

    def finish(self, flat: torch.Tensor):
        """Chain rule from the effective-weight gradients into (V, g, b); clears the staging buffer."""
        if not self.active:
            return
        with torch.no_grad():
            eg = self.eff_grad
            for i in self.skip_layers:
                a, b = self.shapes[i]
                eg[self.w_off[i]: self.b_off[i] + b].mul_(2.0)
            gr = flat.grad[self.lo: self.lo + self.n]
            gr += eg
            if self.weight_norm:
                for i, (a, b) in enumerate(self.shapes[:-1]):
                    sl = slice(self.w_off[i], self.w_off[i] + a * b)
                    v = flat.data[self.lo: self.lo + self.n][sl].view(a, b)
                    g = flat.data[self.g_off[i]: self.g_off[i] + b]
                    dw = eg[sl].view(a, b)
                    norm = v.norm(p=2, dim=0, keepdim=True)
                    dot = (dw * v).sum(dim=0, keepdim=True)
                    dv = (g / norm) * (dw - v * (dot / (norm * norm)))
                    gr[sl].view(a, b).add_(dv - dw)
                    flat.grad[self.g_off[i]: self.g_off[i] + b] += (dot / norm).view(-1)
            eg.zero_()


class DeepONet(base.Arch):
    """Same arguments as the reference (deeponet.py:71-89), including ``*_skip_connection`` / ``*_weight_norm`` (host-side
    reparametrisations of the sub-networks, like ``arch.MLP``)."""

    def __init__(
        self,
        u_key: str,
        y_key: str,
        G_key: str,
        num_loc: int,
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
        for wn, sk, name in ((branch_weight_norm, branch_skip_connection, "branch"), (trunk_weight_norm, trunk_skip_connection, "trunk")):
            if wn and sk:  # the reference picks WeightNormLinear first and then applies the skip to it (mlp.py:238-296)
                raise NotImplementedError(f"DeepONet({name}_weight_norm=True, {name}_skip_connection=True) is not supported yet")
        self.u_key, self.y_key = u_key, y_key
        self.input_keys = (u_key, y_key)
        self.output_keys = (G_key,)
        self.num_loc, self.num_features, self.use_bias = int(num_loc), int(num_features), bool(use_bias)
        self.branch_activation = act_mod.get_activation(branch_activation)
        self.trunk_activation = act_mod.get_activation(trunk_activation)
        for a in (self.branch_activation, self.trunk_activation):
            if a == "stan":
                raise NotImplementedError("DeepONet(*_activation='stan'): activations with a trainable parameter are "
                                          "supported by arch.MLP only")
            if a == "swish":
                act_mod.warn_fixed_swish()
        bw = [self.num_loc] + _hidden(branch_num_layers, branch_hidden_size) + [self.num_features]
        tw = [1] + _hidden(trunk_num_layers, trunk_hidden_size) + [self.num_features]
        feats = tuple(f"f{i}" for i in range(self.num_features))
        self._branch = NetSpec((u_key,), feats, [], [], [], bw, self.branch_activation, dense_in=True)
        self._trunk = NetSpec((y_key,), feats, [0], [0], [0.0], tw, self.trunk_activation)
        nb, nt = self._branch.n_params, self._trunk.n_params
        self._b_rng = (0, nb)
        t0 = (nb + 3) // 4 * 4
        self._t_rng = (t0, t0 + nt)
        self._bias_off = (t0 + nt + 3) // 4 * 4
        g0 = self._bias_off + (1 if self.use_bias else 0)
        self._rb = _SubnetReparam(bw, 0, branch_weight_norm, branch_skip_connection, g0)
        self._rt = _SubnetReparam(tw, t0, trunk_weight_norm, trunk_skip_connection, self._rb.g_end)
        self.flat = nn.Parameter(torch.zeros(self._rt.g_end, dtype=dtype))
        self.reset_parameters()
        self._plans = None

    # ---- parameters ------------------------------------------------------------------------------
    def _layers(self, which: str):
        net, (lo, _) = (self._branch, self._b_rng) if which == "branch_net" else (self._trunk, self._t_rng)
        off = lo
        n = len(net.widths) - 1
        for i, (a, b) in enumerate(zip(net.widths[:-1], net.widths[1:])):
            name = f"{which}.linears.{i}" if i < n - 1 else f"{which}.last_fc"
            yield name, (a, b), off, off + a * b
            off += a * b + b

    def reset_parameters(self):
        """Xavier-uniform weights, zero biases, b = 0 (Paddle nn.Linear defaults; deeponet.py:121-125)."""
        with torch.no_grad():
            self.flat.data.zero_()
            for which in ("branch_net", "trunk_net"):
                for _, (a, b), w0, w1 in self._layers(which):
                    lim = math.sqrt(6.0 / (a + b))
                    self.flat.data[w0:w1] = ((torch.rand(a * b, dtype=torch.float64) * 2 - 1) * lim).to(self.flat.dtype)
            for r in (self._rb, self._rt):  # WeightNormLinear._init_weights: g = 1
                for i, (a, b) in enumerate(r.shapes[:-1] if r.weight_norm else []):
                    self.flat.data[r.g_off[i]: r.g_off[i] + b] = 1

    @property
    def dtype(self) -> torch.dtype:
        return self.flat.dtype

    def state_dict(self, *args, **kwargs):  # reference-style keys
        out = OrderedDict()
        for which, r in (("branch_net", self._rb), ("trunk_net", self._rt)):
            for i, (name, (a, b), w0, w1) in enumerate(self._layers(which)):
                if r.weight_norm and i < len(r.g_off):  # WeightNormLinear: weight_v / weight_g (mlp.py:31-53)
                    out[f"{name}.weight_v"] = self.flat.data[w0:w1].view(a, b).detach().clone()
                    out[f"{name}.weight_g"] = self.flat.data[r.g_off[i]: r.g_off[i] + b].detach().clone()
                else:
                    out[f"{name}.weight"] = self.flat.data[w0:w1].view(a, b).detach().clone()
                out[f"{name}.bias"] = self.flat.data[w1: w1 + b].detach().clone()
        if self.use_bias:
            out["b"] = self.flat.data[self._bias_off: self._bias_off + 1].detach().clone()
        return out

    def load_state_dict(self, state_dict, strict: bool = True):
        missing = []
        with torch.no_grad():
            for which, r in (("branch_net", self._rb), ("trunk_net", self._rt)):
                for i, (name, (a, b), w0, w1) in enumerate(self._layers(which)):
                    wn = r.weight_norm and i < len(r.g_off)
                    slots = [(f"{name}.weight_v" if wn else f"{name}.weight", w0, w1), (f"{name}.bias", w1, w1 + b)]
                    if wn:
                        slots.append((f"{name}.weight_g", r.g_off[i], r.g_off[i] + b))
                    for key, lo, hi in slots:
                        if key not in state_dict:
                            missing.append(key)
                            continue
                        self.flat.data[lo:hi] = torch.as_tensor(state_dict[key]).reshape(-1).to(self.flat.dtype).to(self.flat.device)
            if self.use_bias:
                if "b" in state_dict:
                    self.flat.data[self._bias_off] = float(torch.as_tensor(state_dict["b"]).reshape(-1)[0])
                else:
                    missing.append("b")
        if strict and missing:
            raise KeyError(f"missing keys {missing}")
        return missing, []

    set_state_dict = load_state_dict

    # ---- native plans ----------------------------------------------------------------------------
    def _get_plans(self):
        from ..engine.plan import ResidualPlan

        if self._plans is None or self._plans[0].dtype != self.flat.dtype:
            self._plans = tuple(ResidualPlan(compile_residuals(net, {}, with_grad=False), self.flat.dtype, [], [])
                                for net in (self._branch, self._trunk))
        return self._plans

    def _features(self, x: Dict[str, torch.Tensor]):
        pb, pt = self._get_plans()
        dt = self.flat.dtype
        u = x[self.u_key].to(dt)
        y = x[self.y_key].to(dt)
        b = pb.forward({self.u_key: u}, self._rb.params(self.flat), want_jets=True, want_residuals=False)[0][0]
        t = pt.forward({self.y_key: y}, self._rt.params(self.flat), want_jets=True, want_residuals=False)[0][0]
        return u, y, b, t

    def _combine(self, b: torch.Tensor, t: torch.Tensor, bias) -> torch.Tensor:
        g = (b * _TORCH_ACT[self.trunk_activation](t)).sum(dim=-1, keepdim=True)  # einsum("bi,bi->b") + reshape [-1, 1]
        return g + bias if bias is not None else g

    def forward(self, x: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if self._input_transform is not None:
            x = self._input_transform(x)
        first = x[self.u_key]
        if first.device.type != "cuda" or self.flat.device != first.device:
            raise RuntimeError(
                "paddlescience_b200.arch.DeepONet.forward runs only on a CUDA (H100) device: the engine has no "
                f"CPU fallback (inputs on {first.device}, parameters on {self.flat.device})")
        _, _, b, t = self._features(x)
        bias = self.flat.data[self._bias_off: self._bias_off + 1] if self.use_bias else None
        out = {self.output_keys[0]: self._combine(b, t, bias)}
        if self._output_transform is not None:
            out = self._output_transform(x, out)
        return out

    def fused_train_forward(self, loss_fn, input_dict, label_dict, weight_dict) -> Dict[str, torch.Tensor]:
        """Loss of one constraint + accumulation of its gradient into ``self.flat.grad``.

        Replaces expression.py:96-129 + train.py:158 for this model without any framework autograd graph: native forward
        of both sub-nets with the adjoint's stash kept (``values_fwd_keep``), ONE head kernel for the product, the MSE and
        the two adjoint seeds dL/d(branch), dL/d(trunk) (``ppsci_b200_deeponet_head``), native adjoints of both sub-nets
        from the kept stash (``values_bwd_kept`` — the forward is not recomputed).  Batches larger than the plans'
        workspace chunk are processed slice by slice."""
        from ..engine import binding as B

        if self._input_transform is not None or self._output_transform is not None:
            raise NotImplementedError("input / output transforms are not supported on the fused DeepONet training path")
        if type(loss_fn).__name__ != "MSELoss":
            raise NotImplementedError(f"{type(loss_fn).__name__} has no fused head kernel; only MSELoss is on the hot path")
        flat = self.flat
        if flat.grad is None:
            flat.grad = torch.zeros_like(flat.data)
        key = self.output_keys[0]
        dt, dev = flat.dtype, flat.device
        u = input_dict[self.u_key].to(dt)
        y = input_dict[self.y_key].to(dt)
        if dev != u.device:
            raise ValueError(f"inputs are on {u.device}, parameters on {dev}")
        n = u.shape[0]
        label = label_dict[key].to(dt).reshape(-1).contiguous()
        weight = None
        if weight_dict is not None and key in weight_dict:
            weight = weight_dict[key].to(dt).reshape(-1)
        if "area" in input_dict:  # mse.py:92-93
            area = input_dict["area"].to(dt).reshape(-1)
            weight = area if weight is None else weight * area
        if weight is not None:
            weight = weight.expand(n).contiguous()
        red = getattr(loss_fn, "reduction", "mean")
        coef = float(loss_fn.weight_of(key) if hasattr(loss_fn, "weight_of") else 1.0) * (1.0 / n if red == "mean" else 1.0)
        pb, pt = self._get_plans()
        lib = pb.lib
        pbr, ptr_ = self._rb.params(flat), self._rt.params(flat)  # effective [W | b] under weight_norm / skip_connection
        gbr, gtr = self._rb.grads(flat), self._rt.grads(flat)
        loss_acc = torch.zeros(1, dtype=torch.float64, device=dev)
        bias = flat.data[self._bias_off: self._bias_off + 1] if self.use_bias else None
        dbias = flat.grad[self._bias_off: self._bias_off + 1] if self.use_bias else None
        act = B.ACT_IDS[self._trunk.act.lower()]
        chunk = min(pb.chunk_points, pt.chunk_points)
        stream = torch.cuda.current_stream(dev).cuda_stream if dev.type == "cuda" else 0
        for s0 in range(0, n, chunk):
            sl = slice(s0, min(n, s0 + chunk))
            if self.num_features % 4 == 0:
                # in place: the head reads the features where the forward left them (workspace) and writes the adjoints
                # where the adjoint call expects them — no copy kernels in between
                bf, bbar = pb.values_fwd_keep_inplace({self.u_key: u[sl]}, pbr)
                tf, tbar = pt.values_fwd_keep_inplace({self.y_key: y[sl]}, ptr_)
            else:
                bf = bbar = pb.values_fwd_keep({self.u_key: u[sl]}, pbr)
                tf = tbar = pt.values_fwd_keep({self.y_key: y[sl]}, ptr_)
            m = bf.shape[0]
            rc = lib.lib.ppsci_b200_deeponet_head(
                B.F64 if dt == torch.float64 else B.F32, act, bf.data_ptr(), tf.data_ptr(),
                bias.data_ptr() if bias is not None else None, label[sl].data_ptr(),
                weight[sl].data_ptr() if weight is not None else None, m, self.num_features, coef, None,
                loss_acc.data_ptr(), bbar.data_ptr(), tbar.data_ptr(), dbias.data_ptr() if dbias is not None else None, stream)
            lib.check(rc, "deeponet_head")
            pb.values_bwd_kept(pbr, gbr, bbar)  # bbar / tbar hold dL/d(branch), dL/d(trunk)
            pt.values_bwd_kept(ptr_, gtr, tbar)
        self._rb.finish(flat)
        self._rt.finish(flat)
        return {key: loss_acc[0].to(dt)}
