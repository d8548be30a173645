"""``DeepONet`` (reference: ppsci/arch/deeponet.py:28-154):  G(u)(y) = sum_i branch(u)_i * act(trunk(y))_i + b, and the
branch / trunk machinery it shares with ``HEDeepONets`` (``BranchTrunkArch``).

Both sub-networks run in the native kernels (values only, C = 1): the branch net reads its ``[N, num_loc]`` sensor
matrix as a dense first-layer operand (``dense_in``), the trunk net its coordinate column as an input seed.  The
combination, the loss and their derivatives are elementwise work on ``[N, num_features]`` done with torch on the
device; the weight gradients of the two MLPs come from ``ppsci_b200_values_fwd_bwd`` fed with dL/d(branch),
dL/d(trunk).  One flat parameter buffer  [branch | trunk | b]  so the flat optimizers apply unchanged.

Physics-informed constraints (expressions that differentiate G with respect to the trunk coordinate) take the jet path:
the trunk net carries Taylor jets along its inputs, the residual program runs in ``k_deeponet_jet_head`` between the
sub-networks' forward and adjoint passes (``jets_fwd_keep`` / ``jets_bwd_kept``)."""
from __future__ import annotations

import ctypes as C
import math
from collections import OrderedDict
from typing import Dict, List, NamedTuple, Sequence, Tuple, Union

import sympy as sp
import torch
from sympy.core.function import AppliedUndef
from torch import nn

from ..engine.compiler import CompiledResidual, NetSpec, compile_residuals
from . import activation as act_mod
from . import base
from .mlp import Reparam, hidden_sizes, stack_offsets

_TORCH_ACT = {
    "tanh": torch.tanh, "sin": torch.sin, "cos": torch.cos, "sigmoid": torch.sigmoid, "silu": torch.nn.functional.silu,
    "swish": torch.nn.functional.silu, "gelu": torch.nn.functional.gelu, "relu": torch.relu, "identity": lambda t: t,
    "elu": torch.nn.functional.elu, "selu": torch.nn.functional.selu, "leaky_relu": torch.nn.functional.leaky_relu,
    "siren": lambda t: torch.sin(30.0 * t),
}


class SubNet(NamedTuple):
    """The reference's ``mlp.MLP`` settings of one sub-network; ``prefix`` names its constructor arguments
    (``{prefix}_weight_norm``, ...)."""

    prefix: str
    num_layers: object
    hidden_size: object
    skip_connection: bool
    activation: str
    weight_norm: bool


class BranchTrunkArch(base.Arch):
    """Operators  G_k = sum_{i in block k} f_i * act(trunk(y))_i + b_k  (k < n_out, block k = features kF .. (k+1)F - 1)
    with f = branch(u) (DeepONet) or the product of several branch nets' features (HEDeepONets, he_deeponets.py:151-193;
    ChipDeepONets, chip_deeponets.py:175-199).

    One flat parameter buffer  [branch 1 | ... | trunk | b]  (each sub-network starts at a multiple of 4), then the
    weight-norm gains of every sub-network in the same order.  Physics-informed constraints and expression evaluation
    run through one native head (``k_deeponet_jet_head``): the trunk carries the jets of the compiled residual set, the
    branch nets run values only."""

    def _setup(self, branches: Sequence[Tuple[str, Tuple[str, ...], int, SubNet]], trunk: Tuple[str, Tuple[str, ...], SubNet],
               output_keys: Tuple[str, ...], num_features: int, use_bias: bool, dtype: torch.dtype):
        """``branches``: (reference name, input keys, input width, settings) of every branch net; ``trunk``: (reference
        name, input keys, settings) of the trunk net."""
        cls = type(self).__name__
        for sub in [b[3] for b in branches] + [trunk[2]]:
            if sub.weight_norm and sub.skip_connection:
                # the reference picks WeightNormLinear first and then applies the skip to it (mlp.py:238-296)
                p = sub.prefix
                raise NotImplementedError(f"{cls}({p}_weight_norm=True, {p}_skip_connection=True) is not supported yet")
        self.output_keys = tuple(output_keys)
        self.num_features, self.use_bias = int(num_features), bool(use_bias)
        self._branch_keys = [tuple(keys) for _, keys, _, _ in branches]
        self._branch_locs = [int(loc) for _, _, loc, _ in branches]
        self._trunk_keys = tuple(trunk[1])
        branch_acts = [act_mod.get_activation(sub.activation) for _, _, _, sub in branches]
        self.branch_activation = branch_acts[0]
        self.trunk_activation = act_mod.get_activation(trunk[2].activation)
        for a in branch_acts + [self.trunk_activation]:
            if a == "stan":
                raise NotImplementedError(f"{cls}(*_activation='stan'): activations with a trainable parameter are "
                                          "supported by arch.MLP only")
            if a == "swish":
                act_mod.warn_fixed_swish()
        n_out = len(self.output_keys)
        width = n_out * self.num_features
        feats = tuple(f"f{i}" for i in range(width))
        nets, lo = [], 0
        for (_, keys, loc, sub), act in zip(branches, branch_acts):
            bw = [int(loc)] + hidden_sizes(sub.num_layers, sub.hidden_size) + [width]
            nets.append((NetSpec((keys[0],), feats, [], [], [], bw, act, dense_in=True), sub.weight_norm, sub.skip_connection))
        n_in = len(self._trunk_keys)
        ts = trunk[2]
        tw = [n_in] + hidden_sizes(ts.num_layers, ts.hidden_size) + [width]
        nets.append((NetSpec(self._trunk_keys, feats, list(range(n_in)), [0] * n_in, [0.0] * n_in, tw, self.trunk_activation),
                     ts.weight_norm, ts.skip_connection))
        los = []
        for net, _, _ in nets:
            los.append(lo)
            lo = (lo + net.n_params + 3) // 4 * 4
        self._bias_off = lo
        off = self._bias_off + (n_out if self.use_bias else 0)  # the gains behind b, sub-network by sub-network
        self._nets, self._subnets, self._staged = [n for n, _, _ in nets], [], []
        for (net, wn, skip), lo in zip(nets, los):
            widths = net.widths
            shapes = list(zip(widths[:-1], widths[1:]))
            w_off, b_off, n = stack_offsets(shapes, 0)
            g_off = {}
            for i in range(len(shapes) - 1) if wn else ():  # WeightNormLinear on the hidden layers (mlp.py:234-246)
                g_off[i], off = off, off + shapes[i][1]
            # skip_connection as in arch.MLP: the pre-activation of every even hidden layer i >= 2 is doubled (2 W_i, 2 b_i)
            doubled = {i: (w_off[i], b_off[i] + shapes[i][1]) for i in range(2, len(shapes) - 1, 2)} if skip else {}
            self._subnets.append(Reparam(shapes, lo, n, g_off, wn, doubled))
            if wn or doubled:
                self._staged.append(self._subnets[-1])
        self._sub_names = [b[0] for b in branches] + [trunk[0]]
        self._eff = self._eff_grad = None  # staging buffers laid out like flat, allocated on first use
        self.flat = nn.Parameter(torch.zeros(off, dtype=dtype))
        self.reset_parameters()
        self._plans = None
        self._jet_heads = {}  # residual sets of physics-informed constraints -> _JetHead
        self._traced = {}  # (name, id(expression), extra keys) -> (expression, residual over the trunk inputs)
        syms = [sp.Symbol(k) for k in self.input_keys]
        self._out_fn = {k: sp.Function(k)(*syms) for k in self.output_keys}  # a label on an output with no expression
        tsyms = [sp.Symbol(k) for k in self._trunk_keys]
        self._trunk_fn = {k: sp.Function(k)(*tsyms) for k in self.output_keys}

    # ---- parameters ------------------------------------------------------------------------------
    def _layers(self):
        """(sub-network, layer index, reference name, (in, out), weight offset, bias offset) of every layer."""
        for which, r in zip(self._sub_names, self._subnets):
            for i, (a, b) in enumerate(r.shapes):
                name = f"{which}.linears.{i}" if i < len(r.shapes) - 1 else f"{which}.last_fc"
                yield r, i, name, (a, b), r.lo + r.w_off[i], r.lo + r.b_off[i]

    def reset_parameters(self):
        """Xavier-uniform weights, zero biases, b = 0 (Paddle nn.Linear defaults; deeponet.py:121-125)."""
        with torch.no_grad():
            self.flat.data.zero_()
            for r, i, _, (a, b), w0, w1 in self._layers():
                lim = math.sqrt(6.0 / (a + b))
                self.flat.data[w0:w1] = ((torch.rand(a * b, dtype=torch.float64) * 2 - 1) * lim).to(self.flat.dtype)
                if i in r.g_off:  # WeightNormLinear._init_weights: g = 1
                    self.flat.data[r.g_off[i]: r.g_off[i] + b] = 1

    @property
    def dtype(self) -> torch.dtype:
        return self.flat.dtype

    def state_dict(self, *args, **kwargs):  # reference-style keys
        out = OrderedDict()
        for r, i, name, (a, b), w0, w1 in self._layers():
            if i in r.g_off:  # WeightNormLinear: weight_v / weight_g (mlp.py:31-53)
                out[f"{name}.weight_v"] = self.flat.data[w0:w1].view(a, b).detach().clone()
                out[f"{name}.weight_g"] = self.flat.data[r.g_off[i]: r.g_off[i] + b].detach().clone()
            else:
                out[f"{name}.weight"] = self.flat.data[w0:w1].view(a, b).detach().clone()
            out[f"{name}.bias"] = self.flat.data[w1: w1 + b].detach().clone()
        if self.use_bias:
            out["b"] = self.flat.data[self._bias_off: self._bias_off + len(self.output_keys)].detach().clone()
        return out

    def load_state_dict(self, state_dict, strict: bool = True):
        missing = []
        n_out = len(self.output_keys)
        with torch.no_grad():
            for r, i, name, (a, b), w0, w1 in self._layers():
                wn = i in r.g_off
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
                    self.flat.data[self._bias_off: self._bias_off + n_out] = (
                        torch.as_tensor(state_dict["b"]).reshape(-1)[:n_out].to(self.flat.dtype).to(self.flat.device))
                else:
                    missing.append("b")
        if strict and missing:
            raise KeyError(f"missing keys {missing}")
        return missing, []

    set_state_dict = load_state_dict

    # ---- native plans ----------------------------------------------------------------------------
    def _get_plans(self):
        """Values-only plans of the branch nets, then of the trunk net."""
        from ..engine.plan import ResidualPlan

        if self._plans is None or self._plans[0].dtype != self.flat.dtype:
            self._plans = tuple(ResidualPlan(_no_program(net, []), self.flat.dtype, [], []) for net in self._nets)
        return self._plans

    def _sub_params(self):
        """Effective [W | b] of every sub-network (branches, then trunk): slices of ``flat``, or of the staging buffer
        for a sub-network that ``*_weight_norm`` / ``*_skip_connection`` reparametrise."""
        flat = self.flat.data
        if self._staged and (self._eff is None or self._eff.device != flat.device or self._eff.dtype != flat.dtype):
            self._eff, self._eff_grad = torch.empty_like(flat), torch.zeros_like(flat)
        with torch.no_grad():
            for r in self._staged:
                r.fill(flat, self._eff[r.lo: r.lo + r.n])
        return tuple((self._eff if r in self._staged else flat)[r.lo: r.lo + r.n] for r in self._subnets)

    def _sub_grads(self):
        """Buffers the native calls accumulate the sub-networks' weight gradients into (layout of ``_sub_params``)."""
        return tuple((self._eff_grad if r in self._staged else self.flat.grad)[r.lo: r.lo + r.n] for r in self._subnets)

    def _finish_sub_grads(self):
        """Chain rule of the reparametrised sub-networks into ``flat.grad``; clears the staging buffer."""
        with torch.no_grad():
            for r in self._staged:
                eg = self._eff_grad[r.lo: r.lo + r.n]
                r.chain(self.flat.data, self.flat.grad, eg)
                eg.zero_()

    def _branch_input(self, x: Dict[str, torch.Tensor], j: int) -> torch.Tensor:
        """Branch j's [N, input width] matrix (its input keys side by side, as MLP.concat_to_tensor)."""
        dt = self.flat.dtype
        keys = self._branch_keys[j]
        n = x[keys[0]].shape[0]
        return torch.cat([x[k].to(dt).reshape(n, -1) for k in keys], dim=1) if len(keys) > 1 else x[keys[0]].to(dt)

    def forward(self, x: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if self._input_transform is not None:
            x = self._input_transform(x)
        first = x[self.input_keys[0]]
        if first.device.type != "cuda" or self.flat.device != first.device:
            raise RuntimeError(
                f"paddlescience_b200.arch.{type(self).__name__}.forward runs only on a CUDA (H100) device: the engine has "
                f"no CPU fallback (inputs on {first.device}, parameters on {self.flat.device})")
        dt = self.flat.dtype
        plans, params = self._get_plans(), self._sub_params()
        feats = [plans[j].forward({self._branch_keys[j][0]: self._branch_input(x, j)}, params[j], want_jets=True,
                                  want_residuals=False)[0][0] for j in range(len(self._branch_keys))]
        t = plans[-1].forward({k: x[k].to(dt) for k in self._trunk_keys}, params[-1], want_jets=True, want_residuals=False)[0][0]
        prod = feats[0] * _TORCH_ACT[self.trunk_activation](t)  # he_deeponets.py:167-189: heat * act(trunk) * cold
        for f in feats[1:]:
            prod = prod * f
        n_out = len(self.output_keys)
        g = prod.view(prod.shape[0], n_out, self.num_features).sum(dim=-1)
        if self.use_bias:
            g = g + self.flat.data[self._bias_off: self._bias_off + n_out]
        out = {k: g[:, i: i + 1] for i, k in enumerate(self.output_keys)}
        if self._output_transform is not None:
            out = self._output_transform(x, out)
        return out

    def _check_fused(self, loss_fn):
        if self._input_transform is not None or self._output_transform is not None:
            raise NotImplementedError(f"input / output transforms are not supported on the fused {type(self).__name__} "
                                      "training path")
        if type(loss_fn).__name__ != "MSELoss":
            raise NotImplementedError(f"{type(loss_fn).__name__} has no fused head kernel; only MSELoss is on the hot path")

    # ---- residuals on the trunk inputs' Taylor jets -----------------------------------------------
    def _residual(self, name: str, e, extra_keys) -> sp.Basic:
        """sympy residual of one expression over the outputs as functions of the trunk inputs (cached per expression):
        traced with every output a function of all model inputs, then checked to use no derivative with respect to a
        branch input and no branch input wider than one column (after the outputs lose their branch arguments the
        former would silently read as 0; the latter has no column to read)."""
        from ..equation.pde.base import lookup_parameter
        from ..utils import symbolic

        key = (name, id(e), tuple(extra_keys))
        hit = self._traced.get(key)
        if hit is not None and hit[0] is e:
            return hit[1]
        cls = type(self).__name__
        src = e
        if isinstance(e, symbolic.CompiledExpr):
            e = e.expr
        elif not isinstance(e, sp.Basic):
            if not callable(e):
                raise TypeError(f"output_expr['{name}'] must be a sympy expression or a callable, got {type(e)}")
            e = symbolic.trace_to_sympy(e, self.input_keys, self.output_keys, list(extra_keys))
        e = sp.sympify(e)
        wide = {k: loc for keys, loc in zip(self._branch_keys, self._branch_locs) for k in keys if not (loc == 1 and len(keys) == 1)}
        branch = {k for keys in self._branch_keys for k in keys}
        trunk = "', '".join(self._trunk_keys)
        for d in e.atoms(sp.Derivative):
            for v, _ in d.variable_count:
                if str(v) in branch:
                    raise NotImplementedError(f"{cls} expression '{name}': derivatives with respect to the branch input "
                                              f"'{v}' are not supported (only the trunk inputs '{trunk}')")
        outs = set(self.output_keys)
        e = e.replace(lambda a: isinstance(a, AppliedUndef) and a.func.__name__ in outs,
                      lambda a: self._trunk_fn[a.func.__name__])
        for s_ in e.free_symbols:
            if str(s_) in wide:
                raise NotImplementedError(f"{cls} expression '{name}' uses the branch input '{s_}' itself, which has "
                                          f"{wide[str(s_)]} columns; only a one-column branch input can appear in an "
                                          f"expression, besides the outputs, their derivatives with respect to '{trunk}', "
                                          "the trunk inputs and extra input columns")
        learnable = sorted(str(s_) for s_ in e.free_symbols if lookup_parameter(str(s_)) is not None)
        if learnable:
            raise NotImplementedError(f"{cls} expression '{name}': learnable equation parameters {learnable} are "
                                      "not supported")
        self._traced[key] = (src, e)
        return e

    def _jet_head(self, exprs: Dict[str, object], extra_keys) -> "_JetHead":
        """The compiled residual set of ``exprs`` with its trunk plan and native head for the current dtype (cached)."""
        key = (tuple((name, id(e)) for name, e in exprs.items()), tuple(extra_keys), self.flat.dtype)
        hit = self._jet_heads.get(key)
        if hit is None or any(a is not b for a, b in zip(hit.sources, exprs.values())):
            hit = _JetHead(self, {k: self._residual(k, e, extra_keys) for k, e in exprs.items()}, list(exprs.values()))
            self._jet_heads[key] = hit
        return hit

    def _jet_run(self, head: "_JetHead", input_dict, labels, weights, coefs, loss_acc, residual_out, train: bool):
        """Chunked forward of every sub-network with the adjoint's stash kept (``jets_fwd_keep``), the jet head
        (``deeponet_jet_head_run``) and, when ``train``, every adjoint from the stash (``jets_bwd_kept``)."""
        from ..engine import binding as B

        flat = self.flat
        dt, dev = flat.dtype, flat.device
        us = [self._branch_input(input_dict, j) for j in range(len(self._branch_keys))]
        if dev != us[0].device:
            raise ValueError(f"inputs are on {us[0].device}, parameters are on {dev}")
        n = us[0].shape[0]
        xs = [input_dict[k].to(dt).reshape(-1).contiguous() for k in self._trunk_keys]
        cr = head.compiled
        aux = [input_dict[k].to(dt).reshape(-1).contiguous() for k in cr.aux_keys]
        pbs = self._get_plans()[:-1]
        pt = head.trunk_plan
        lib = pt.lib
        params = self._sub_params()
        grads = self._sub_grads() if train else None
        n_out = len(self.output_keys)
        bias = flat.data[self._bias_off: self._bias_off + n_out] if self.use_bias else None
        dbias = flat.grad[self._bias_off: self._bias_off + n_out] if (train and self.use_bias) else None
        a = B.DeepONetJetArgs()
        a.n_features = self.num_features
        a.bias = bias.data_ptr() if bias is not None else None
        for j, t in enumerate(xs):
            a.x_cols[j] = t.data_ptr()
        for i, t in enumerate(aux):
            a.aux_cols[i] = t.data_ptr()
        for k in range(len(cr.names)):
            lab = labels[k]
            if torch.is_tensor(lab):
                a.label_cols[k] = lab.data_ptr()
            else:
                a.label_const[k] = float(lab)
            a.weight_cols[k] = weights[k].data_ptr() if weights[k] is not None else None
            a.coef[k] = coefs[k]
            a.residual_out[k] = residual_out[k].data_ptr() if residual_out is not None else None
        a.loss_acc = loss_acc.data_ptr() if loss_acc is not None else None
        a.dbias = dbias.data_ptr() if dbias is not None else None
        chunk = min(p.chunk_points for p in pbs + (pt,))
        stream = torch.cuda.current_stream(dev).cuda_stream if dev.type == "cuda" else 0
        for s0 in range(0, n, chunk):
            sl = slice(s0, min(n, s0 + chunk))
            kept = [pb.jets_fwd_keep({self._branch_keys[j][0]: us[j][sl]}, params[j]) for j, pb in enumerate(pbs)]
            a.b, bbar, a.ldb, _ = kept[0]
            b2bar = b3bar = None
            if len(kept) > 1:
                a.b2, b2bar, a.ldb2, _ = kept[1]
            if len(kept) > 2:
                a.b3, b3bar, a.ldb3, _ = kept[2]
            a.t, tbar, a.ldt, a.tplane = pt.jets_fwd_keep({k: x[sl] for k, x in zip(self._trunk_keys, xs)}, params[-1])
            a.n = sl.stop - s0
            a.x_off = s0
            a.bbar, a.b2bar, a.b3bar, a.tbar = (bbar, b2bar, b3bar, tbar) if train else (None, None, None, None)
            lib.check(lib.lib.ppsci_b200_deeponet_jet_head_run(head.handle, C.byref(a), stream), "deeponet_jet_head_run")
            if train:
                for pb, g, p in zip(pbs + (pt,), grads, params):
                    pb.jets_bwd_kept(p, g)
        if train:
            self._finish_sub_grads()

    def _jet_train_forward(self, loss_fn, input_dict, label_dict, weight_dict, output_expr, extra_keys):
        """The losses of ``output_expr``'s slots (in the order of ``label_dict``; a label key without an expression is
        that output itself), whose residuals may differentiate the outputs with respect to the trunk inputs, and their
        gradient accumulated into ``self.flat.grad``.  Per slot: label column or constant, weight column (times
        ``area``), reduction and MSELoss weight, as mse.py:82-106."""
        flat = self.flat
        if flat.grad is None:
            flat.grad = torch.zeros_like(flat.data)
        dt, dev = flat.dtype, flat.device
        output_expr = output_expr or {}
        names = list(label_dict)
        for k in names:
            if k not in output_expr and k not in self.output_keys:
                raise KeyError(f"label '{k}' has neither an output expression nor a model output")
        exprs = {k: output_expr[k] if k in output_expr else self._out_fn[k] for k in names}
        head = self._jet_head(exprs, extra_keys)
        n = input_dict[self.input_keys[0]].shape[0]
        red = getattr(loss_fn, "reduction", "mean")
        area = input_dict["area"].to(dt).reshape(-1) if "area" in input_dict else None
        labels, weights, coefs = [], [], []
        for k in names:
            lab = label_dict[k]
            if torch.is_tensor(lab) and lab.numel() == n:
                labels.append(lab.to(dev, dt).reshape(-1).contiguous())
            else:
                labels.append(float(lab.reshape(-1)[0]) if torch.is_tensor(lab) else float(lab))
            w = weight_dict.get(k) if weight_dict else None
            if w is not None:
                w = (w.to(dev, dt).reshape(-1) if torch.is_tensor(w) else torch.full((1,), float(w), dtype=dt, device=dev))
            if area is not None:  # mse.py:92-93
                w = area if w is None else w * area
            weights.append(w.expand(n).contiguous() if w is not None else None)
            coefs.append(float(loss_fn.weight_of(k) if hasattr(loss_fn, "weight_of") else 1.0) * (1.0 / n if red == "mean" else 1.0))
        loss_acc = torch.zeros(len(names), dtype=torch.float64, device=dev)
        self._jet_run(head, input_dict, labels, weights, coefs, loss_acc, None, train=True)
        return {k: loss_acc[i].to(dt) for i, k in enumerate(names)}

    def evaluate_expressions(self, exprs: Dict[str, object], input_dict, extra_keys=(), outputs=None) -> Dict[str, torch.Tensor]:
        """Values [N, 1] of expressions over the outputs, their derivatives with respect to the trunk inputs, the inputs
        and extra columns (eval / visualisation), from one forward-only run of the jet head.  An expression that traces
        to exactly the output it is named after takes that output's value from ``outputs`` when given."""
        if self._input_transform is not None or self._output_transform is not None:
            raise NotImplementedError(f"input / output transforms are not supported on {type(self).__name__} expressions")
        res = {k: self._residual(k, e, extra_keys) for k, e in exprs.items()}
        out = {k: outputs[k] for k in exprs if outputs is not None and k in outputs and res[k] == self._trunk_fn.get(k)}
        pending = {k: e for k, e in exprs.items() if k not in out}
        if pending:
            head = self._jet_head(pending, extra_keys)
            first = input_dict[self.input_keys[0]]
            n = first.shape[0]
            vals = [torch.empty((n, 1), dtype=self.flat.dtype, device=first.device) for _ in pending]
            k = len(vals)
            self._jet_run(head, input_dict, [0.0] * k, [None] * k, [0.0] * k, None, vals, train=False)
            out.update(zip(pending, vals))
        return {k: out[k] for k in exprs}


class DeepONet(BranchTrunkArch):
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
        self.u_key, self.y_key = u_key, y_key
        self.input_keys = (u_key, y_key)
        self.num_loc = int(num_loc)
        branch = SubNet("branch", branch_num_layers, branch_hidden_size, branch_skip_connection, branch_activation,
                        branch_weight_norm)
        trunk = SubNet("trunk", trunk_num_layers, trunk_hidden_size, trunk_skip_connection, trunk_activation, trunk_weight_norm)
        self._setup([("branch_net", (u_key,), num_loc, branch)], ("trunk_net", (y_key,), trunk), (G_key,), num_features,
                    use_bias, dtype)
        self._branch, self._trunk = self._nets
        self._rb, self._rt = self._subnets

    def fused_train_forward(self, loss_fn, input_dict, label_dict, weight_dict, output_expr=None,
                            extra_keys=()) -> Dict[str, torch.Tensor]:
        """Loss of one constraint + accumulation of its gradient into ``self.flat.grad``.

        Replaces expression.py:96-129 + train.py:158 for this model without any framework autograd graph: native forward
        of both sub-nets with the adjoint's stash kept (``values_fwd_keep``), ONE head kernel for the product, the MSE and
        the two adjoint seeds dL/d(branch), dL/d(trunk) (``ppsci_b200_deeponet_head``), native adjoints of both sub-nets
        from the kept stash (``values_bwd_kept`` — the forward is not recomputed).  Batches larger than the plans'
        workspace chunk are processed slice by slice.

        ``output_expr`` (the constraint's expressions) with a key that is not a model output selects the residual path
        of physics-informed DeepONet: the expressions may differentiate G with respect to the trunk coordinate and use
        extra input columns (``extra_keys``); see ``_jet_train_forward``."""
        from ..engine import binding as B

        self._check_fused(loss_fn)
        if output_expr is not None and any(k not in self.output_keys for k in output_expr):
            return self._jet_train_forward(loss_fn, input_dict, label_dict, weight_dict, output_expr, extra_keys)
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
        pbr, ptr_ = self._sub_params()  # effective [W | b] under weight_norm / skip_connection
        gbr, gtr = self._sub_grads()
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
        self._finish_sub_grads()
        return {key: loss_acc[0].to(dt)}


def _no_program(net: NetSpec, dirs) -> CompiledResidual:
    """A sub-network whose output jets along ``dirs`` a head reads: no residual program, so no register file (its
    outputs may outnumber the program's 256 registers)."""
    return CompiledResidual(net=net, names=[], dirs=dirs, aux_keys=[], n_reg=0, prog=[], consts=[], res_reg=[], grad_res=[],
                            grad_in=[], grad_reg=[])


class _JetHead:
    """One compiled operator residual set for one dtype: the register program over the outputs' jets along the trunk
    inputs (compiled on a network with the trunk inputs and the model's outputs), the trunk plan built with that
    program's jet layout, and the native head (``ppsci_b200_deeponet_jet_head_create``) holding the program on the
    device."""

    def __init__(self, model: BranchTrunkArch, exprs: Dict[str, sp.Basic], sources):
        from ..engine import binding as B
        from ..engine.plan import ResidualPlan, _dtype_id

        self.sources = sources  # keeps the cache key's ids alive
        keys, outs = model._trunk_keys, tuple(model.output_keys)
        n_in = len(keys)
        net = NetSpec(keys, outs, list(range(n_in)), [0] * n_in, [0.0] * n_in, [n_in, len(outs)], model.trunk_activation)
        cr = compile_residuals(net, exprs)
        if len(cr.names) > B.MAX_RES:
            raise NotImplementedError(f"more than {B.MAX_RES} residuals per constraint")
        if len(cr.aux_keys) > B.MAX_IN:
            raise NotImplementedError(f"more than {B.MAX_IN} auxiliary columns")
        self.compiled = cr
        self.trunk_plan = ResidualPlan(_no_program(model._nets[-1], cr.dirs), model.flat.dtype, [], [])
        self.lib = self.trunk_plan.lib
        s = B.DeepONetHeadSpec()
        s.dtype = _dtype_id(model.flat.dtype)
        s.act = B.ACT_IDS[model.trunk_activation]
        s.n_out = len(outs)
        s.n_in = n_in
        s.n_dir = len(cr.dirs)
        for d, dr in enumerate(cr.dirs):
            s.dir_order[d] = dr.order
        s.n_aux = len(cr.aux_keys)
        s.n_reg = cr.n_reg
        s.n_ops = len(cr.prog)
        self._prog = (C.c_int32 * max(1, 4 * len(cr.prog)))(*[x for op in cr.prog for x in op])
        self._consts = (C.c_double * max(1, len(cr.consts)))(*cr.consts)
        self._gres = (C.c_int32 * max(1, len(cr.grad_res)))(*cr.grad_res)
        self._gin = (C.c_int32 * max(1, len(cr.grad_in)))(*cr.grad_in)
        self._greg = (C.c_int32 * max(1, len(cr.grad_reg)))(*cr.grad_reg)
        s.prog = C.cast(self._prog, C.POINTER(C.c_int32))
        s.n_consts = len(cr.consts)
        s.consts = C.cast(self._consts, C.POINTER(C.c_double))
        s.n_res = len(cr.names)
        for k, r in enumerate(cr.res_reg):
            s.res_reg[k] = r
        s.n_grad = len(cr.grad_res)
        s.grad_res = C.cast(self._gres, C.POINTER(C.c_int32))
        s.grad_in = C.cast(self._gin, C.POINTER(C.c_int32))
        s.grad_reg = C.cast(self._greg, C.POINTER(C.c_int32))
        handle = C.c_void_p()
        self.lib.check(self.lib.lib.ppsci_b200_deeponet_jet_head_create(C.byref(s), C.byref(handle)), "deeponet_jet_head_create")
        self.handle = handle

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.lib.ppsci_b200_deeponet_jet_head_destroy(self.handle)
                self.handle = None
        except Exception:
            pass
