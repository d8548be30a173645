"""Optimizer factories with the reference's call convention ``Adam(lr, ...)(model)``
(ppsci/optimizer/optimizer.py:179-248).  The step itself is one fused CUDA kernel over the flat
parameter / gradient buffers (``ppsci_b200_adam_step``, csrc/kernels_simt.cuh ``k_adam``)."""
from __future__ import annotations

from typing import Optional, Tuple, Union

import torch

from ..engine import binding as B


class ClipGradByGlobalNorm:
    """paddle.nn.ClipGradByGlobalNorm: every gradient of the optimizer is scaled by ``clip_norm / max(global_norm, clip_norm)``."""

    def __init__(self, clip_norm: float):
        self.clip_norm = float(clip_norm)


class ClipGradByNorm:
    """paddle.nn.ClipGradByNorm: each parameter TENSOR's gradient is scaled by ``clip_norm / max(its norm, clip_norm)``."""

    def __init__(self, clip_norm: float):
        self.clip_norm = float(clip_norm)


class ClipGradByValue:
    """paddle.nn.ClipGradByValue: gradients are clamped to ``[min, max]`` (``min`` defaults to ``-max``)."""

    def __init__(self, max: float, min: Optional[float] = None):  # noqa: A002 (paddle's argument names)
        self.max = float(max)
        self.min = -float(max) if min is None else float(min)


def clip_gradients(grad_clip, flat_grad: torch.Tensor, segments, extra_grads=(), grad_scale: float = 1.0) -> None:
    """Apply a paddle-style gradient clipping object (matched by class name, so ``paddle.nn.ClipGradBy*`` instances work
    too) in place, on the device, without a host synchronisation.  ``grad_scale`` is the factor the fused Adam kernel
    applies to the raw gradient first (1 / world size, 1 / update_freq): the clipping thresholds refer to the scaled
    gradient, like paddle's, which clips what the optimizer consumes.  ``segments``: (start, stop) of every parameter
    tensor inside the flat buffer (ClipGradByNorm is per tensor)."""
    if grad_clip is None:
        return
    kind = type(grad_clip).__name__
    gs = float(grad_scale)
    grads = [flat_grad] + [g for g in extra_grads if g is not None]
    if kind == "ClipGradByGlobalNorm":
        clip = float(grad_clip.clip_norm)
        total = torch.sqrt(sum((g.double() ** 2).sum() for g in grads)) * abs(gs)
        scale = clip / torch.clamp(total, min=clip)
        for g in grads:
            g.mul_(scale.to(g.dtype))
    elif kind == "ClipGradByNorm":
        clip = float(grad_clip.clip_norm)
        views = [flat_grad[a:b] for a, b in segments] + grads[1:]
        for v in views:
            n = v.double().norm() * abs(gs)
            v.mul_((clip / torch.clamp(n, min=clip)).to(v.dtype))
    elif kind == "ClipGradByValue":
        lo, hi = float(grad_clip.min), float(grad_clip.max)
        for g in grads:
            g.clamp_(min=lo / gs, max=hi / gs) if gs > 0 else g.clamp_(min=hi / gs, max=lo / gs)
    else:
        raise NotImplementedError(f"grad_clip of type {kind} is not supported (ClipGradByGlobalNorm / ByNorm / ByValue)")


class FlatAdam:
    """Adam over ``model.flat`` (paddle.optimizer.Adam semantics: L2 ``weight_decay`` folded into
    the gradient, bias-corrected moments, no amsgrad)."""

    def __init__(self, model, learning_rate, beta1=0.9, beta2=0.999, epsilon=1e-8, weight_decay=None, decoupled=False,
                 extra_params=(), grad_clip=None):
        self.model = model
        self.grad_clip = grad_clip  # paddle-style clipping object, applied to the gradients right before the fused step
        # learnable equation parameters (``Adam(lr)((model, equation))``, ppsci/optimizer/optimizer.py:225-248 collects the
        # parameters of every entry of model_list): each is stepped by the same fused kernel, one tiny launch per scalar
        self.extra_params = list(extra_params)
        self._extra_state = {}
        self._lr = learning_rate
        self.beta1, self.beta2, self.epsilon = beta1, beta2, epsilon
        self.weight_decay = float(weight_decay) if weight_decay else 0.0
        if self.weight_decay < 0:
            raise ValueError("weight_decay must be non-negative")
        self.decoupled = bool(decoupled)
        if self.decoupled:  # the native step reads a negative coefficient as "decoupled" (include/ppsci_b200.h)
            self.weight_decay = -self.weight_decay
        self.t = 0
        self.exp_avg: Optional[torch.Tensor] = None
        self.exp_avg_sq: Optional[torch.Tensor] = None
        self.grad_scale = 1.0

    def get_lr(self) -> float:
        return float(self._lr() if callable(self._lr) else self._lr)

    def set_lr(self, lr: float):
        self._lr = lr

    @property
    def _learning_rate(self):
        return self._lr

    def _ensure_state(self):
        p = self.model.flat
        if self.exp_avg is None or self.exp_avg.device != p.device or self.exp_avg.dtype != p.dtype:
            self.exp_avg = torch.zeros_like(p.data)
            self.exp_avg_sq = torch.zeros_like(p.data)

    def step(self):
        p = self.model.flat
        if p.grad is None:
            return
        if p.device.type != "cuda":
            raise RuntimeError("FlatAdam.step needs parameters on a CUDA (H100) device: no CPU fallback")
        self._ensure_state()
        self.t += 1
        self._clip()
        lib = B.get_library()
        dtype = B.F64 if p.dtype == torch.float64 else B.F32
        rc = lib.lib.ppsci_b200_adam_step(dtype, p.data.data_ptr(), p.grad.data_ptr(), self.exp_avg.data_ptr(),
                                          self.exp_avg_sq.data_ptr(), p.numel(), self.get_lr(), self.beta1, self.beta2,
                                          self.epsilon, self.weight_decay, self.t, self.grad_scale,
                                          torch.cuda.current_stream(p.device).cuda_stream)
        lib.check(rc, "adam_step")
        for q in self.extra_params:
            if q.grad is None:
                continue
            if q.device.type != "cuda":
                raise RuntimeError("learnable equation parameters must live on the CUDA device of the model")
            st = self._extra_state.get(id(q))
            if st is None or st[0].device != q.device or st[0].dtype != q.dtype:
                st = self._extra_state[id(q)] = (torch.zeros_like(q.data), torch.zeros_like(q.data))
            qd = B.F64 if q.dtype == torch.float64 else B.F32
            rc = lib.lib.ppsci_b200_adam_step(qd, q.data.data_ptr(), q.grad.data_ptr(), st[0].data_ptr(), st[1].data_ptr(),
                                              q.numel(), self.get_lr(), self.beta1, self.beta2, self.epsilon,
                                              self.weight_decay, self.t, self.grad_scale,
                                              torch.cuda.current_stream(q.device).cuda_stream)
            lib.check(rc, "adam_step (equation parameter)")

    # -- the same step split for CUDA-graph replay (solver/graph_step.py): ``step_dev`` is the launch (recorded once,
    #    every scalar that changes per step is read from ``hyper_dev``), ``advance`` the host-side bookkeeping that
    #    produces those scalars for the coming step.
    def _param_segments(self):
        """(start, stop) of every parameter tensor inside ``model.flat`` (weights, biases, gains, ... each on its own)."""
        m = self.model
        segs = []
        if hasattr(m, "_shapes"):
            for i, (a, b) in enumerate(m._shapes):
                segs.append((m._w_off[i], m._w_off[i] + a * b))
                segs.append((m._b_off[i], m._b_off[i] + b))
        covered = max((hi for _, hi in segs), default=0)
        if covered < m.flat.numel():
            segs.append((covered, m.flat.numel()))  # gains / alphas / betas / fourier kernel: one segment
        return segs

    def _clip(self):
        if self.grad_clip is not None and self.model.flat.grad is not None:
            clip_gradients(self.grad_clip, self.model.flat.grad, self._param_segments(),
                           [q.grad for q in self.extra_params], self.grad_scale)

    def advance(self):
        """t += 1; returns [lr, 1 - beta1^t, 1 - beta2^t, grad_scale] of this step."""
        self.t += 1
        return [self.get_lr(), 1.0 - self.beta1 ** self.t, 1.0 - self.beta2 ** self.t, float(self.grad_scale)]

    def step_dev(self, hyper_dev: torch.Tensor, zero_grads: bool = True):
        if self.extra_params:
            raise NotImplementedError("CUDA-graph replay (to_static) with learnable equation parameters is not supported yet")
        p = self.model.flat
        if p.device.type != "cuda":
            raise RuntimeError("FlatAdam.step_dev needs parameters on a CUDA (H100) device: no CPU fallback")
        if hyper_dev.dtype != torch.float64 or hyper_dev.numel() < 4 or hyper_dev.device != p.device:
            raise ValueError("hyper_dev must be a float64 tensor of 4 values on the parameters' device")
        self._ensure_state()
        self._clip()  # device-side vector operations: recorded into the graph with the step
        lib = B.get_library()
        dtype = B.F64 if p.dtype == torch.float64 else B.F32
        rc = lib.lib.ppsci_b200_adam_step_dev(dtype, p.data.data_ptr(), p.grad.data_ptr(), self.exp_avg.data_ptr(),
                                              self.exp_avg_sq.data_ptr(), p.numel(), hyper_dev.data_ptr(), self.beta1,
                                              self.beta2, self.epsilon, self.weight_decay, 1 if zero_grads else 0,
                                              torch.cuda.current_stream(p.device).cuda_stream)
        lib.check(rc, "adam_step_dev")

    def clear_grad(self):
        if self.model.flat.grad is not None:
            self.model.flat.grad.zero_()
        for q in self.extra_params:
            if q.grad is not None:
                q.grad.zero_()

    zero_grad = clear_grad

    def state_dict(self):
        # like paddle's optimizer state ("LR_Scheduler" entry): a resumed run continues the warm-up / decay where it
        # stopped instead of replaying it from step 0
        sd = {"t": self.t, "exp_avg": self.exp_avg, "exp_avg_sq": self.exp_avg_sq}
        if self.extra_params:
            sd["extra"] = [self._extra_state.get(id(q)) for q in self.extra_params]
        if hasattr(self._lr, "state_dict"):
            sd["LR_Scheduler"] = self._lr.state_dict()
        return sd

    def set_state_dict(self, sd):
        self.t = int(sd["t"])
        self.exp_avg, self.exp_avg_sq = sd["exp_avg"], sd["exp_avg_sq"]
        for q, st in zip(self.extra_params, sd.get("extra", [])):
            if st is not None:
                self._extra_state[id(q)] = (st[0], st[1])
        if "LR_Scheduler" in sd and hasattr(self._lr, "set_state_dict"):
            self._lr.set_state_dict(sd["LR_Scheduler"])


class Adam:
    """``ppsci.optimizer.Adam`` factory (optimizer.py:179-248)."""

    def __init__(self, learning_rate=1e-3, beta1: float = 0.9, beta2: float = 0.999, epsilon: float = 1e-8,
                 weight_decay=None, grad_clip=None, lazy_mode: bool = False, amsgrad: bool = False):
        self.grad_clip = grad_clip
        if amsgrad:
            raise NotImplementedError("amsgrad is not supported yet")
        self.learning_rate, self.beta1, self.beta2, self.epsilon = learning_rate, beta1, beta2, epsilon
        self.weight_decay = weight_decay

    def __call__(self, model_list):
        extra = []
        if isinstance(model_list, (tuple, list)):
            # (model, equation, ...): entries without a flat parameter buffer contribute their learnable scalars
            models = [m for m in model_list if hasattr(m, "flat")]
            for m in model_list:
                if not hasattr(m, "flat"):
                    if not hasattr(m, "learnable_parameters"):
                        raise TypeError(f"{type(m).__name__} is neither a model nor an equation with learnable parameters")
                    extra += list(m.learnable_parameters)
            if len(models) != 1:
                raise NotImplementedError("one optimizer over several models is not supported yet")
            model_list = models[0]
        return FlatAdam(model_list, self.learning_rate, self.beta1, self.beta2, self.epsilon, self.weight_decay,
                        decoupled=getattr(self, "_decoupled", False), extra_params=extra, grad_clip=self.grad_clip)


class AdamW(Adam):
    """``ppsci.optimizer.AdamW`` factory (optimizer.py:386-496): Adam with DECOUPLED weight decay —
    ``p <- p (1 - lr * weight_decay)`` before the Adam update, in the same fused kernel.  The per-parameter exclusions
    (``no_weight_decay_name``, ``one_dim_param_no_weight_decay``) have no counterpart on the flat parameter buffer."""

    def __init__(self, learning_rate=1e-3, beta1: float = 0.9, beta2: float = 0.999, epsilon: float = 1e-8,
                 weight_decay: float = 0.001, grad_clip=None, no_weight_decay_name=None,
                 one_dim_param_no_weight_decay: bool = False, amsgrad: bool = False):
        if no_weight_decay_name or one_dim_param_no_weight_decay:
            raise NotImplementedError("AdamW: per-parameter weight-decay exclusions are not supported on the flat buffer")
        super().__init__(learning_rate, beta1, beta2, epsilon, weight_decay, grad_clip, False, amsgrad)
        self._decoupled = True


class FlatLBFGS:
    """L-BFGS over ``model.flat`` (reference: ppsci/optimizer/optimizer.py:250-323 wraps ``paddle.optimizer.LBFGS``,
    driven by the closure loop of ppsci/solver/train.py:216-319).  The two-loop recursion and the strong-Wolfe line
    search are vector operations on the single flat parameter buffer (``torch.optim.LBFGS`` semantics); every
    closure evaluation is one fused native loss + weight-gradient call per constraint."""

    is_lbfgs = True

    def __init__(self, model, learning_rate=1.0, max_iter=1, max_eval=None, tolerance_grad=1e-7, tolerance_change=1e-9,
                 history_size=100, line_search_fn="strong_wolfe"):
        self.model = model
        self._opt = torch.optim.LBFGS([model.flat], lr=float(learning_rate() if callable(learning_rate) else learning_rate),
                                      max_iter=max_iter, max_eval=max_eval, tolerance_grad=tolerance_grad,
                                      tolerance_change=tolerance_change, history_size=history_size,
                                      line_search_fn=line_search_fn)
        self._lr = learning_rate
        self.grad_scale = 1.0

    def get_lr(self) -> float:
        return float(self._opt.param_groups[0]["lr"])

    def set_lr(self, lr: float):
        self._opt.param_groups[0]["lr"] = float(lr)

    def step(self, closure):
        if self.model.flat.device.type != "cuda":
            raise RuntimeError("FlatLBFGS.step needs parameters on a CUDA (H100) device: no CPU fallback")
        if callable(self._lr):
            self.set_lr(self._lr())
        return self._opt.step(closure)

    def clear_grad(self):
        if self.model.flat.grad is not None:
            self.model.flat.grad.zero_()

    zero_grad = clear_grad

    def state_dict(self):
        sd = self._opt.state_dict()
        if hasattr(self._lr, "state_dict"):
            sd["LR_Scheduler"] = self._lr.state_dict()
        return sd

    def set_state_dict(self, sd):
        sd = dict(sd)
        lr_sd = sd.pop("LR_Scheduler", None)
        self._opt.load_state_dict(sd)
        if lr_sd is not None and hasattr(self._lr, "set_state_dict"):
            self._lr.set_state_dict(lr_sd)


class LBFGS:
    """``ppsci.optimizer.LBFGS`` factory (optimizer.py:250-323), same arguments and defaults."""

    def __init__(self, learning_rate: float = 1.0, max_iter: int = 1, max_eval: Optional[int] = None,
                 tolerance_grad: float = 1e-07, tolerance_change: float = 1e-09, history_size: int = 100,
                 line_search_fn: Optional[str] = "strong_wolfe"):
        if line_search_fn not in (None, "strong_wolfe"):
            raise ValueError(f"line_search_fn should be 'strong_wolfe' or None, but got {line_search_fn}")
        self.lr, self.max_iter, self.max_eval = learning_rate, max_iter, max_eval
        self.tolerance_grad, self.tolerance_change = tolerance_grad, tolerance_change
        self.history_size, self.line_search_fn = history_size, line_search_fn

    def __call__(self, model_list):
        if isinstance(model_list, (tuple, list)):
            if len(model_list) != 1:
                raise NotImplementedError("one optimizer over several models is not supported yet")
            model_list = model_list[0]
        return FlatLBFGS(model_list, self.lr, self.max_iter, self.max_eval, self.tolerance_grad, self.tolerance_change,
                         self.history_size, self.line_search_fn)
