"""``jacobian`` / ``hessian`` / ``clear`` with the reference's signatures
(ppsci/autodiff/ad.py:95-103, 254-264, 326-341).

The reference implements them as cached reverse-mode ``paddle.grad(create_graph=True)`` sweeps.
Here derivatives w.r.t. network inputs are produced by forward Taylor jets inside the CUDA
kernels, so these functions act on *symbolic proxies* (``SymTensor``): a Python-callable
equation such as ``AllenCahn`` (ppsci/equation/pde/allen_cahn.py:56-62) is called ONCE with
proxies, the resulting sympy expression is compiled (engine/compiler.py) and no autograd graph
ever exists on the hot path.  Passing real tensors raises ``TypeError`` — loudly, instead of a
silent slow path.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Union

import sympy as sp
import torch


class SymTensor:
    """A stand-in for an ``[N, 1]`` tensor that records sympy arithmetic."""

    __array_priority__ = 1000

    def __init__(self, expr):
        self.expr = sp.sympify(expr)

    # shape mimicry, enough for user code that inspects it
    shape = (None, 1)
    ndim = 2

    @staticmethod
    def _unwrap(o):
        if isinstance(o, SymTensor):
            return o.expr
        if isinstance(o, (int, float)):
            return sp.sympify(o)
        if isinstance(o, torch.Tensor) and o.numel() == 1:
            return sp.Float(float(o))
        if isinstance(o, sp.Basic):
            return o
        raise TypeError(f"cannot combine a symbolic tensor with {type(o).__name__}; "
                        "equations traced by the engine may only mix proxies, python numbers and sympy objects")

    def __add__(self, o): return SymTensor(self.expr + self._unwrap(o))
    def __radd__(self, o): return SymTensor(self._unwrap(o) + self.expr)
    def __sub__(self, o): return SymTensor(self.expr - self._unwrap(o))
    def __rsub__(self, o): return SymTensor(self._unwrap(o) - self.expr)
    def __mul__(self, o): return SymTensor(self.expr * self._unwrap(o))
    def __rmul__(self, o): return SymTensor(self._unwrap(o) * self.expr)
    def __truediv__(self, o): return SymTensor(self.expr / self._unwrap(o))
    def __rtruediv__(self, o): return SymTensor(self._unwrap(o) / self.expr)
    def __pow__(self, o): return SymTensor(self.expr ** self._unwrap(o))
    def __rpow__(self, o): return SymTensor(self._unwrap(o) ** self.expr)
    def __neg__(self): return SymTensor(-self.expr)
    # comparisons are conditions of torch.where; the residual compiler takes equalities only and names that form for
    # the others
    def __eq__(self, o): return SymTensor(sp.Eq(self.expr, self._unwrap(o)))
    def __ne__(self, o): return SymTensor(sp.Ne(self.expr, self._unwrap(o)))
    def __lt__(self, o): return SymTensor(sp.Lt(self.expr, self._unwrap(o)))
    def __le__(self, o): return SymTensor(sp.Le(self.expr, self._unwrap(o)))
    def __gt__(self, o): return SymTensor(sp.Gt(self.expr, self._unwrap(o)))
    def __ge__(self, o): return SymTensor(sp.Ge(self.expr, self._unwrap(o)))
    __hash__ = object.__hash__
    def __pos__(self): return self
    def __repr__(self): return f"SymTensor({self.expr})"

    def detach(self): return SymTensor(sp.Function("detach")(self.expr))
    def pow(self, o): return self.__pow__(o)
    def square(self): return SymTensor(self.expr ** 2)
    def sin(self): return SymTensor(sp.sin(self.expr))
    def cos(self): return SymTensor(sp.cos(self.expr))
    def exp(self): return SymTensor(sp.exp(self.expr))
    def tanh(self): return SymTensor(sp.tanh(self.expr))
    def log(self): return SymTensor(sp.log(self.expr))
    def sqrt(self): return SymTensor(sp.sqrt(self.expr))
    def abs(self): return SymTensor(sp.Abs(self.expr))

    _TORCH_UNARY = {
        torch.sin: sp.sin, torch.cos: sp.cos, torch.exp: sp.exp, torch.tanh: sp.tanh, torch.log: sp.log,
        torch.sqrt: sp.sqrt, torch.abs: sp.Abs, torch.sinh: sp.sinh, torch.cosh: sp.cosh, torch.tan: sp.tan,
        torch.square: lambda e: e ** 2, torch.neg: lambda e: -e,
    }

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func in cls._TORCH_UNARY and len(args) == 1:
            return SymTensor(cls._TORCH_UNARY[func](cls._unwrap(args[0])))
        if func in (torch.pow,):
            return SymTensor(cls._unwrap(args[0]) ** cls._unwrap(args[1]))
        if func in (torch.add, torch.sub, torch.mul, torch.div, torch.true_divide):
            a, b = cls._unwrap(args[0]), cls._unwrap(args[1])
            return SymTensor({torch.add: a + b, torch.sub: a - b, torch.mul: a * b}.get(func, a / b))
        if func in (torch.maximum,):
            return SymTensor(sp.Max(cls._unwrap(args[0]), cls._unwrap(args[1])))
        if func in (torch.minimum,):
            return SymTensor(sp.Min(cls._unwrap(args[0]), cls._unwrap(args[1])))
        if func is torch.where and len(args) == 3 and not kwargs:
            cond, a, b = (cls._unwrap(t) for t in args)
            return SymTensor(sp.Piecewise((a, cond), (b, True)))
        raise NotImplementedError(
            f"torch function {getattr(func, '__name__', func)} cannot be traced into a residual program")


def _need_sym(t, what: str):
    if not isinstance(t, SymTensor):
        raise TypeError(
            f"{what} must be a symbolic proxy: in this engine input-derivatives are computed by forward "
            "Taylor jets inside the CUDA kernels, so jacobian/hessian are only meaningful while an equation "
            "callable is being traced (Solver / lambdify do that automatically); there is no autograd "
            "graph through the network to differentiate real tensors.")


def _diff(expr: sp.Basic, x: sp.Basic, order: int) -> sp.Basic:
    """d^order expr / dx^order with the product / chain rule expanded down to derivatives of network outputs
    (``jacobian(nu * u__x, x)`` or ``jacobian(u * u, x)`` in a user PDE callable — the reference differentiates
    whatever tensor it is handed, ad.py:56-77).  A bare network output stays an unevaluated ``Derivative`` node,
    which is what the residual compiler lowers to jet registers."""
    return sp.diff(expr, x, order)


class Jacobians:
    """``jacobian(ys, xs, i=0, j=None, retain_graph=None, create_graph=True)`` — ad.py:95-160."""

    def __call__(self, ys, xs: Union[SymTensor, Sequence[SymTensor]], i: int = 0, j: Optional[int] = None,
                 retain_graph: Optional[bool] = None, create_graph: bool = True):
        _need_sym(ys, "ys")
        if i != 0:
            raise ValueError(f"i={i} is not valid: ys is a single-column proxy")  # ad.py:66-69 analogue
        if isinstance(xs, (list, tuple)):
            for x in xs:
                _need_sym(x, "xs[k]")
            return [SymTensor(_diff(ys.expr, x.expr, 1)) for x in xs]
        _need_sym(xs, "xs")
        if j not in (None, 0):
            raise ValueError(f"j={j} is not valid: xs is a single-column proxy")
        return SymTensor(_diff(ys.expr, xs.expr, 1))

    def _clear(self):
        pass


class Hessians:
    """``hessian(ys, xs, component=None, i=0, j=0, ...)`` — ad.py:254-303."""

    def __call__(self, ys, xs, component: Optional[int] = None, i: int = 0, j: int = 0, grad_y=None,
                 retain_graph: Optional[bool] = None, create_graph: bool = True):
        _need_sym(ys, "ys")
        _need_sym(xs, "xs")
        if component not in (None, 0) or i != 0 or j != 0:
            raise ValueError("component / i / j must be 0 for single-column proxies")
        return SymTensor(_diff(ys.expr, xs.expr, 2))

    def _clear(self):
        pass


jacobian = Jacobians()
hessian = Hessians()


def clear():
    """ad.py:326-341 clears the per-iteration grad caches; nothing is cached here."""
    jacobian._clear()
    hessian._clear()
