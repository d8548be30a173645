"""``ExpressionSolver`` — the drop-in seam of the hot path.

Reference: ppsci/utils/expression.py:40-212.  ``train_forward`` keeps the reference signature
and return value, but each constraint is ONE call into the native library that evaluates the
network jets, the residual program, the MSE *and* accumulates the weight gradient into
``model.flat.grad`` (so the reference's separate ``total_loss.backward()``,
ppsci/solver/train.py:158, has nothing left to do).  Loss values stay on the device: the
per-key ``.item()`` syncs of expression.py:122 are gone; ``losses_constraint`` holds lazy
0-dim tensors that the logger converts only when it prints."""
from __future__ import annotations

from typing import Callable, Dict, Optional, Tuple

import sympy as sp
import torch
from torch import nn

from ..engine.compiler import compile_residuals
from ..engine.plan import ResidualPlan
from . import symbolic


def _learnable_parameters(exprs: Dict[str, sp.Basic]) -> Dict[str, "torch.nn.Parameter"]:
    """Free symbols of the expressions that name a learnable equation parameter (``PDE.create_parameter``): what the
    reference receives as ``extra_parameters`` and turns into ParameterNodes (symbolic.py:798, 849-858)."""
    from ..equation.pde.base import lookup_parameter

    found = {}
    for e in exprs.values():
        for s_ in e.free_symbols:
            p = lookup_parameter(str(s_))
            if p is not None:
                found[str(s_)] = p
    return found


def _with_parameters(inputs: Dict[str, torch.Tensor], params: Dict[str, "torch.nn.Parameter"]):
    if not params:
        return inputs
    merged = dict(inputs)
    merged.update(params)
    return merged


def _collect_parameter_grads(plan: ResidualPlan, params: Dict[str, "torch.nn.Parameter"], device):
    """dLoss/dparameter from the plan's fp64 accumulators into ``param.grad`` (accumulating, like backward())."""
    if not params:
        return
    buf = plan.param_grad_buffer(device)
    for i, k in enumerate(plan.compiled.aux_keys):
        p = params.get(k)
        if p is None:
            continue
        g = buf[i].to(p.dtype).reshape(p.shape).to(p.device)
        p.grad = g.clone() if p.grad is None else p.grad + g
    buf.zero_()


class CompiledConstraint:
    """Residual plan(s) of one constraint, built lazily per dtype."""

    def __init__(self, model, cst, extra_keys=()):
        self.model = model
        self.cst = cst
        self.exprs = _constraint_exprs(model, cst, extra_keys)  # the loss iterates label keys (mse.py:85); same order
        self.names = list(self.exprs)
        # MSELossWithL2Decay: penalty slots (mse.py:259-266) — reduction "sum", their own weight, no per-point weights
        self.reg = dict(getattr(cst.loss, "regularization_dict", None) or {})
        self.parameters = _learnable_parameters(self.exprs)
        self.compiled = compile_residuals(model.net_spec(), self.exprs, param_keys=list(self.parameters))
        self._plans: Dict[torch.dtype, ResidualPlan] = {}
        self._key_plans: Dict[tuple, ResidualPlan] = {}

    def plan_for_key(self, dtype, k: int) -> ResidualPlan:
        """The same residual program with a one-hot loss weight: the adjoint yields d(loss of residual k)/d(params) alone
        (per-equation gradients for mtl.PCGrad and friends; the reference calls losses[key].backward() per key)."""
        if (dtype, k) not in self._key_plans:
            reds, lw = self._loss_spec()
            lw = [w if j == k else 0.0 for j, w in enumerate(lw)]
            self._key_plans[(dtype, k)] = ResidualPlan(self.compiled, dtype, reds, lw)
        return self._key_plans[(dtype, k)]

    def strip_penalty_slots(self, labels, weights):
        """MSELossWithL2Decay: a penalty slot is ``sum(out^2)`` — no label, no per-point weight / area (mse.py:262-264)."""
        if not self.reg:
            return labels, weights
        labels = {k: v for k, v in (labels or {}).items() if k not in self.reg}
        weights = {k: v for k, v in weights.items() if k not in self.reg} if weights else weights
        return labels, weights

    def _loss_spec(self):
        """Per residual slot: (reduction, loss weight)."""
        loss = self.cst.loss
        red = getattr(loss, "reduction", "mean")
        reds = ["sum" if key in self.reg else red for key in self.names]
        lw = [float(self.reg[key]) if key in self.reg else (loss.weight_of(key) if hasattr(loss, "weight_of") else 1.0)
              for key in self.names]
        return reds, lw

    def plan(self, dtype) -> ResidualPlan:
        if dtype not in self._plans:
            loss = self.cst.loss
            if type(loss).__name__ not in ("MSELoss", "CausalMSELoss", "MSELossWithL2Decay"):
                raise NotImplementedError(f"{type(loss).__name__} has no fused head kernel; only MSELoss / CausalMSELoss / "
                                          "MSELossWithL2Decay are on the hot path")
            reds, lw = self._loss_spec()
            self._plans[dtype] = ResidualPlan(self.compiled, dtype, reds, lw)
        return self._plans[dtype]


def _constraint_exprs(model, cst, extra_keys) -> Dict[str, sp.Basic]:
    """sympy residual expressions of one constraint, keyed and ordered like its label dict (mse.py:85)."""
    exprs: Dict[str, sp.Basic] = {}
    out_keys = tuple(model.output_keys)
    for name, e in cst.output_expr.items():
        if isinstance(e, symbolic.CompiledExpr):
            exprs[name] = e.expr
        elif isinstance(e, sp.Basic):
            exprs[name] = e
        elif callable(e):
            exprs[name] = symbolic.trace_to_sympy(e, model.input_keys, out_keys, extra_keys)
        else:
            raise TypeError(f"output_expr['{name}'] must be a sympy expression or a callable, got {type(e)}")
    names = [k for k in cst.output_keys if k in exprs] if hasattr(cst, "output_keys") else list(exprs)
    for reg_key in (getattr(cst.loss, "regularization_dict", None) or {}):  # MSELossWithL2Decay: output_dict[reg_key]
        if reg_key not in exprs:
            if reg_key not in out_keys:
                raise KeyError(f"regularization key '{reg_key}' is neither an output expression nor a model output")
            exprs[reg_key] = sp.Function(reg_key)(*[sp.Symbol(k) for k in model.input_keys])
        if reg_key not in names:
            names.append(reg_key)
    # a registered output transform is part of the function being trained (mlp.py:313-314): rewrite the residuals in
    # terms of the bare network the kernels differentiate
    return {k: symbolic.apply_output_transform(model, exprs[k]) for k in names}


class BatchedConstraints:
    """Several constraints that share one MLP evaluated by ONE native call (SURVEY section 8(f) rank 1; the reference
    loops ``for i, cst_name in enumerate(constraint)`` in expression.py:89-129 — for LDC that is the interior equation
    plus four ~100-point wall constraints, i.e. five times the per-call launch train for 0.1 % more points).

    The point sets are concatenated; every residual of every constraint becomes one slot of a single residual program
    (shared jet directions, common sub-expressions merged by the compiler); a slot only counts on its own constraint's
    range because its per-point weight column is zero elsewhere.  "mean" of constraint i over its own N_i points is
    expressed through the weights: w(p) = N_total / N_i on the range, with the call normalised by N_total."""

    def __init__(self, model, csts: Dict[str, "object"], input_dicts):
        from ..engine import binding as B

        self.model = model
        self.cst_names = list(csts)
        self.slots = []  # (constraint index, key, slot name)
        exprs: Dict[str, sp.Basic] = {}
        self.reductions, self.loss_weights = [], []
        for i, (cname, cst) in enumerate(csts.items()):
            if type(cst.loss).__name__ != "MSELoss":
                raise NotImplementedError(f"{type(cst.loss).__name__} has no fused head kernel; only MSELoss is on the hot path")
            extra = [k for k in (input_dicts[i] or {}) if k not in model.input_keys]
            for key, e in _constraint_exprs(model, cst, extra).items():
                slot = f"{cname}::{key}"
                exprs[slot] = e
                self.slots.append((i, key, slot))
                self.reductions.append(getattr(cst.loss, "reduction", "mean"))
                self.loss_weights.append(cst.loss.weight_of(key) if hasattr(cst.loss, "weight_of") else 1.0)
        if len(self.slots) > B.MAX_RES:
            raise NotImplementedError(f"{len(self.slots)} residuals in one batch (max {B.MAX_RES})")
        self.parameters = _learnable_parameters(exprs)
        self.compiled = compile_residuals(model.net_spec(), exprs, param_keys=list(self.parameters))
        self._plans: Dict[torch.dtype, ResidualPlan] = {}
        self._mask_cache = {}

    def plan(self, dtype) -> ResidualPlan:
        if dtype not in self._plans:
            self._plans[dtype] = ResidualPlan(self.compiled, dtype, self.reductions, self.loss_weights)
        return self._plans[dtype]

    def run(self, input_dicts, label_dicts, weight_dicts, params, grads):
        """Returns the per-slot loss vector (device tensor, no host sync)."""
        dtype, dev = params.dtype, params.device
        plan = self.plan(dtype)
        cr = self.compiled
        ns = [next(iter(d.values())).shape[0] for d in input_dicts]
        offs = [0]
        for n in ns:
            offs.append(offs[-1] + n)
        ntot = offs[-1]
        cols = {}
        for k in list(cr.net.input_keys) + list(cr.aux_keys):
            if k in self.parameters:  # a learnable scalar, not a data column
                cols[k] = self.parameters[k]
                continue
            buf = torch.zeros(ntot, 1, dtype=dtype, device=dev)
            for i, d in enumerate(input_dicts):
                if k in d:
                    buf[offs[i]: offs[i + 1]] = d[k].to(dtype).reshape(-1, 1)
            cols[k] = buf
        labels, weights = {}, {}
        for (i, key, slot), red in zip(self.slots, self.reductions):
            lab = torch.zeros(ntot, 1, dtype=dtype, device=dev)
            lv = label_dicts[i][key]
            lab[offs[i]: offs[i + 1]] = lv.to(dtype).reshape(-1, 1) if torch.is_tensor(lv) else float(lv)
            labels[slot] = lab
            w = torch.zeros(ntot, 1, dtype=dtype, device=dev)
            scale = (ntot / ns[i]) if red == "mean" else 1.0  # mean over the constraint's own points
            wi = weight_dicts[i].get(key) if weight_dicts[i] else None
            rng = w[offs[i]: offs[i + 1]]
            rng.fill_(scale)
            if wi is not None:
                rng.mul_(wi.to(dtype).reshape(-1, 1) if torch.is_tensor(wi) else float(wi))
            if "area" in input_dicts[i]:  # mse.py:92-93
                rng.mul_(input_dicts[i]["area"].to(dtype).reshape(-1, 1))
            weights[slot] = w
        out = plan.loss_fwd_bwd(cols, params, grads, labels=labels, weights=weights, n_norm=ntot).clone()
        if grads is not None:
            _collect_parameter_grads(plan, self.parameters, dev)
        return out


class ExpressionSolver(nn.Module):
    """Expression computing helper (same public methods as the reference)."""

    batch_constraints: bool = True  # constraints sharing the MLP go through ONE native call (BatchedConstraints)

    nvtx_flag: bool = False

    def __init__(self):
        super().__init__()
        self._compiled: Dict[int, CompiledConstraint] = {}
        self._eval_exprs: Dict[tuple, symbolic.CompiledExpr] = {}  # (id(expr), name, id(model), extra keys) -> compiled
        self._batched: Dict[tuple, BatchedConstraints] = {}

    def forward(self, *args, **kwargs):
        raise NotImplementedError("Use train_forward/eval_forward/visu_forward instead of forward.")

    def compiled_for(self, model, cst, input_dict=None) -> CompiledConstraint:
        key = id(cst)
        if key not in self._compiled:
            extra = [k for k in (input_dict or {}) if k not in model.input_keys]
            self._compiled[key] = CompiledConstraint(model, cst, extra)
        return self._compiled[key]

    def train_forward(
        self,
        expr_dicts: Tuple[Dict[str, Callable], ...],
        input_dicts: Tuple[Dict[str, torch.Tensor], ...],
        model,
        constraint: Dict[str, "object"],
        label_dicts: Tuple[Dict[str, torch.Tensor], ...],
        weight_dicts: Tuple[Dict[str, torch.Tensor], ...],
        per_key_grads: bool = False,
    ):
        """Returns (losses_all, losses_constraint) like the reference; additionally the weight
        gradient of  sum(losses_all)  has been accumulated into ``model.flat.grad``.

        ``per_key_grads=True`` (loss aggregators that need the gradient of every loss term, mtl.PCGrad): nothing is
        accumulated into ``model.flat.grad``; a third value ``{key: flat gradient of losses_all[key]}`` is returned, each
        produced by one fused call with a one-hot loss weight."""
        losses_all: Dict[str, torch.Tensor] = {}
        losses_constraint: Dict[str, torch.Tensor] = {}
        if per_key_grads:
            if hasattr(model, "fused_train_forward"):
                raise NotImplementedError("per-term gradients are implemented for the MLP family of models")
            if getattr(model, "_input_transform", None) is not None:
                raise NotImplementedError(f"{type(model).__name__}: a registered input transform is not traced into the fused "
                                          "residual kernels")
            flat = model.flat
            params = model.engine_params()
            # reparametrised models (weight_norm / random_weight / fourier / skip_connection): the kernels fill the
            # staging buffer, finish_grads() chains it into flat.grad — borrowed per term and restored afterwards
            staged = bool(getattr(model, "_has_eff", False))
            saved = None
            if staged:
                if flat.grad is None:
                    flat.grad = torch.zeros_like(flat.data)
                saved = flat.grad.clone()
            grads_by_key: Dict[str, torch.Tensor] = {}
            for i, cst_name in enumerate(constraint):
                cst = constraint[cst_name]
                cc = self.compiled_for(model, cst, input_dicts[i])
                weights = weight_dicts[i]
                if "area" in input_dicts[i]:
                    area = input_dicts[i]["area"]
                    weights = {k: (weights[k] * area if weights and k in weights else area) for k in cc.names}
                labels_i, weights = cc.strip_penalty_slots(label_dicts[i], weights)
                if cc.parameters:
                    raise NotImplementedError("per-term gradients with learnable equation parameters are not supported yet")
                if type(cst.loss).__name__ == "CausalMSELoss":
                    weights = self._causal_weights(cst, cc, cc.plan(flat.dtype), input_dicts[i], labels_i, weights, params)
                for k, key in enumerate(cc.names):
                    g = grads_by_key.setdefault(key, torch.zeros_like(flat.data))
                    if staged:
                        flat.grad.zero_()
                        lv = cc.plan_for_key(flat.dtype, k).loss_fwd_bwd(input_dicts[i], params, model.engine_grads(),
                                                                         labels=labels_i, weights=weights)[k].clone()
                        model.finish_grads()
                        g.add_(flat.grad)
                    else:
                        lv = cc.plan_for_key(flat.dtype, k).loss_fwd_bwd(input_dicts[i], params, g, labels=labels_i,
                                                                         weights=weights)[k].clone()
                    losses_all[key] = losses_all[key] + lv if key in losses_all else lv
                    losses_constraint[cst_name] = losses_constraint[cst_name] + lv if cst_name in losses_constraint else lv
            if staged:
                flat.grad.copy_(saved)
            return losses_all, losses_constraint, grads_by_key
        if hasattr(model, "fused_train_forward"):  # models that combine several native networks (DeepONet)
            for i, cst_name in enumerate(constraint):
                cst = constraint[cst_name]
                extra = [k for k in input_dicts[i] if k not in model.input_keys]
                losses = model.fused_train_forward(cst.loss, input_dicts[i], label_dicts[i], weight_dicts[i],
                                                   cst.output_expr, extra)
                losses_constraint[cst_name] = sum(losses.values())
                for key, v in losses.items():
                    losses_all[key] = losses_all[key] + v if key in losses_all else v
            return losses_all, losses_constraint
        if getattr(model, "_input_transform", None) is not None:
            # MLP.forward (eval / predict / validators) applies the registered transforms; the fused residual kernels
            # differentiate the bare network.  Output transforms are traced into the residual program
            # (symbolic.apply_output_transform); an input transform would change the jet seeds.  Training a different
            # function than the one evaluated must not be silent.
            raise NotImplementedError(f"{type(model).__name__}: a registered input transform is not traced into the fused "
                                      "residual kernels; express it inside the constraint's output_expr (or the "
                                      "equation) instead")
        flat = model.flat
        params, grads = model.engine_params(), model.engine_grads()  # effective weights / staging grads under weight_norm
        if self.batch_constraints and len(constraint) > 1:
            from ..engine import binding as B

            n_slots = sum(len([k for k in cst.output_expr]) for cst in constraint.values())
            if n_slots <= B.MAX_RES and all(type(c.loss).__name__ == "MSELoss" for c in constraint.values()):
                bkey = tuple(id(c) for c in constraint.values())
                if bkey not in self._batched:
                    self._batched[bkey] = BatchedConstraints(model, constraint, input_dicts)
                bc = self._batched[bkey]
                loss_vec = bc.run(input_dicts, label_dicts, weight_dicts, params, grads)
                for k, (i, key, _) in enumerate(bc.slots):
                    cname = bc.cst_names[i]
                    losses_constraint[cname] = losses_constraint[cname] + loss_vec[k] if cname in losses_constraint else loss_vec[k]
                    losses_all[key] = losses_all[key] + loss_vec[k] if key in losses_all else loss_vec[k]
                model.finish_grads()
                return losses_all, losses_constraint
        for i, cst_name in enumerate(constraint):
            cst = constraint[cst_name]
            use_nvtx = self.nvtx_flag and flat.is_cuda
            if use_nvtx:
                torch.cuda.nvtx.range_push(f"Constraint {cst_name}")
            cc = self.compiled_for(model, cst, input_dicts[i])
            plan = cc.plan(flat.dtype)
            weights = weight_dicts[i]
            if "area" in input_dicts[i]:  # mse.py:92-93 multiplies by the area column when present
                area = input_dicts[i]["area"]
                weights = {k: (weights[k] * area if weights and k in weights else area) for k in cc.names}
            labels_i, weights = cc.strip_penalty_slots(label_dicts[i], weights)
            if type(cst.loss).__name__ == "CausalMSELoss":
                weights = self._causal_weights(cst, cc, plan, input_dicts[i], labels_i, weights, params)
            loss_vec = plan.loss_fwd_bwd(_with_parameters(input_dicts[i], cc.parameters), params, grads, labels=labels_i,
                                         weights=weights)
            loss_vec = loss_vec.clone()
            _collect_parameter_grads(plan, cc.parameters, flat.device)
            losses_constraint[cst_name] = loss_vec.sum()
            for k, key in enumerate(cc.names):
                losses_all[key] = losses_all[key] + loss_vec[k] if key in losses_all else loss_vec[k]
            if use_nvtx:
                torch.cuda.nvtx.range_pop()
        model.finish_grads()  # weight_norm chain rule into model.flat.grad (no-op otherwise)
        return losses_all, losses_constraint

    @staticmethod
    def _causal_weights(cst, cc, plan, input_dict, label_dict, weights, params):
        """CausalMSELoss (mse.py:157-190): chunk weights exp(-tol * sum of the earlier chunks' mean losses), without
        gradient.  One forward-only native call gives the residuals they are formed from; the fused call then takes them
        as (part of) its per-point weight column."""
        _, res = plan.forward(_with_parameters(input_dict, cc.parameters), params, want_jets=False)
        out = {}
        for key in cc.names:
            e2 = (res[key] - label_dict[key].to(res[key].dtype)) ** 2
            if weights and key in weights:
                e2 = e2 * weights[key]
            cw = cst.loss.causal_weights(e2)
            out[key] = weights[key] * cw if weights and key in weights else cw
        return out

    def eval_forward(self, expr_dict, input_dict, model, validator, label_dict, weight_dict):
        """Forward for evaluation (expression.py:133-180): outputs + expressions + validator loss."""
        output_dict = model({k: input_dict[k] for k in model.input_keys})
        if hasattr(model, "evaluate_expressions"):  # operator networks: expressions through their jet head
            if expr_dict:  # a pass-through is an expression that traces to exactly its output, whatever its form
                extra = [k for k in input_dict if k not in model.input_keys]
                output_dict.update(model.evaluate_expressions(expr_dict, input_dict, extra, outputs=output_dict))
            expr_dict = {}
        for name, expr in expr_dict.items():
            if name in output_dict and not isinstance(expr, (sp.Basic, symbolic.CompiledExpr)):
                continue  # plain "lambda out: out['u']" style pass-through
            if isinstance(expr, symbolic.CompiledExpr):
                ce = expr
            else:  # compile once per (expression, model): sympy CSE + plan_create + workspace are not per-batch work
                extra = tuple(k for k in input_dict if k not in model.input_keys)
                ck = (id(expr), name, id(model), extra)
                ce = self._eval_exprs.get(ck)
                if ce is None or ce._src is not expr:
                    ce = symbolic.CompiledExpr(
                        expr if isinstance(expr, sp.Basic) else symbolic.trace_to_sympy(
                            expr, model.input_keys, model.output_keys, list(extra)), model, name)
                    ce._src = expr  # keeps the key's id() alive and guards against id reuse
                    self._eval_exprs[ck] = ce
            output_dict[name] = ce(input_dict)
        if "area" in input_dict:
            output_dict["area"] = input_dict["area"]
        losses = validator.loss(output_dict, label_dict, weight_dict) if validator is not None else {}
        return output_dict, losses

    def visu_forward(self, expr_dict, input_dict, model):
        output_dict, _ = self.eval_forward(expr_dict or {}, input_dict, model, None, None, None)
        return output_dict
