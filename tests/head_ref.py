"""Test helper: an fp64 reference of one residual-head call (k_head), evaluated on the output jets the head read.

After a fused call the plan's workspace still holds the output jets Y that k_head read and the output-jet adjoints Ybar
it wrote (``layer_ref.stash_views``).  From Y this module recomputes, independently of the compiler's lowering, CSE,
register allocation and emission, everything the head produces:

* each residual r_k, by evaluating the user's sympy expression with ``oracle.ppsci_oracle.eval_expr`` on fp64 tensors,
  a ``Piecewise`` per group of points that take the same branches (conditions by ``tests/chip_deeponet_ref.
  eval_piecewise``), so an untaken branch is never evaluated: an output binds to Y[0, :, j], a
  derivative D^alpha of output j to sum_{(d, c) in combos[alpha]} c k! Y[channel(d, k), :, j], inputs, aux columns and
  learnable parameters to fp64 leaves;
* each slot's loss coef_k sum_p w e^2, e = r - label, coef = loss_weight / n_norm (mean) or loss_weight (sum);
* Ybar = dLoss/dY and dLoss/d(parameter) by torch.autograd.grad of the total loss (the head's
  sum_k 2 coef_k w e_k dr_k/dY).

Every residual also gets a first-order running-error bound M, propagated through the same tree (add / sub:
M(a) + M(b) + |a +- b|; mul: |b| M(a) + |a| M(b) + |ab|; unary f: |f'(a)| M(a) + |f(a)|; leaves 0, constants |c|, a
derivative leaf the size of its lowered sum), so that |r - r_ref| / (u M) is the error in units of the rounding of the
residual's own terms.  Ybar is measured per (channel, output) plane against the plane's largest |ref|, dLoss/dparameter
against sum_p |term_p|, the losses relatively (their terms are all positive).

``gen_residuals`` builds seeded random residual sets over the operator set the tracer offers, with domain guards that keep
every value finite; half of them are written as torch callables and traced through ``ad.SymTensor``.
"""
from __future__ import annotations

import math
import random
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import sympy as sp
import torch
from sympy.core.function import AppliedUndef

from oracle import ppsci_oracle as O
from paddlescience_b200.autodiff import ad
from paddlescience_b200.engine import binding as B
from paddlescience_b200.engine.compiler import DETACH_FUNC_NAME, compile_residuals, cvt_to_key
from paddlescience_b200.engine.plan import ResidualPlan
from tests.cases import make_net
from tests.chip_deeponet_ref import eval_piecewise
from tests.layer_ref import all_layouts, last_chunk, param_blocks, stash_views

U32 = 2.0 ** -24
U64 = 2.0 ** -53
OP_NAMES = {v: k for k, v in B.OPS.items()}


def _is_detach(e) -> bool:
    return isinstance(e, AppliedUndef) and e.func.__name__ == DETACH_FUNC_NAME


# ------------------------------------------------------------------------------------------------------------------
# binding of the user expression's atoms
# ------------------------------------------------------------------------------------------------------------------
def bind(cr, exprs: Sequence[sp.Basic], Y: torch.Tensor, X: torch.Tensor, aux: Dict[str, torch.Tensor]):
    """(expressions with every Derivative replaced by a symbol, data, leaf bounds M).  Y [C, n, n_out] fp64 (may
    require grad), X [n_in, n] fp64, aux {name: [n] column or [n] expanded parameter}."""
    net = cr.net
    in_index = {k: i for i, k in enumerate(net.input_keys)}
    out_index = {k: j for j, k in enumerate(net.output_keys)}
    data: Dict[str, torch.Tensor] = {}
    leafM: Dict[str, torch.Tensor] = {}
    for j, k in enumerate(net.output_keys):  # an [n] column first: eval_expr shapes constants like its first entry
        data[k] = Y[0, :, j]
    for i, k in enumerate(net.input_keys):
        data[k] = X[i]
    data.update(aux)
    out = []
    for e in exprs:
        subs = {}
        for d in e.atoms(sp.Derivative):
            f = d.args[0].args[0] if _is_detach(d.args[0]) else d.args[0]
            j = out_index[f.func.__name__]
            alpha = [0] * len(in_index)
            for s, o in d.variable_count:
                alpha[in_index[str(s)]] += int(o)
            k = sum(alpha)
            key = "_D_" + cvt_to_key(d)
            terms = [float(c) * math.factorial(k) * Y[cr.channel_of(dd, k), :, j] for dd, c in cr.combos[tuple(alpha)]]
            data[key] = sum(terms[1:], terms[0])
            leafM[key] = sum(t.detach().abs() for t in terms) * (len(terms) + 1)
            subs[d] = sp.Symbol(key)
        out.append(e.xreplace(subs))
    return out, data, leafM


def _resolve(e: sp.Basic, truth: Dict[sp.Basic, bool]) -> sp.Basic:
    """``e`` with every Piecewise replaced by the branch the condition values ``truth`` select."""
    if isinstance(e, sp.Piecewise):
        for val, cond in e.args:
            if cond == sp.true or truth[cond]:
                return _resolve(val, truth)
    if not e.args:
        return e
    return e.func(*[_resolve(a, truth) for a in e.args])


def branch_groups(e: sp.Basic, data: Dict[str, torch.Tensor], n: int):
    """[(point indices, ``e`` without Piecewise)]: the points grouped by the values of every condition of a where.  Each
    group evaluates only its own branches, so the NaN / Inf of an untaken branch reaches neither the value nor autograd
    (a torch.where would hand it to the gradient as 0 * inf)."""
    conds = sorted({c for pw in e.atoms(sp.Piecewise) for _, c in pw.args if c != sp.true}, key=str)
    dev = next(iter(data.values())).device
    if not conds:
        return [(torch.arange(n, device=dev), e)]
    masks = [(eval_piecewise(c.lhs, data).detach() == eval_piecewise(c.rhs, data).detach()).expand(n) for c in conds]
    code = sum(m.long() << i for i, m in enumerate(masks))
    out = []
    for v in torch.unique(code).tolist():
        idx = torch.nonzero(code == v).view(-1)
        out.append((idx, _resolve(e, {c: bool((v >> i) & 1) for i, c in enumerate(conds)})))
    return out


def _take(data: Dict[str, torch.Tensor], idx: torch.Tensor, n: int) -> Dict[str, torch.Tensor]:
    return {k: (v[idx] if v.dim() == 1 and v.shape[0] == n else v) for k, v in data.items()}


# ------------------------------------------------------------------------------------------------------------------
# running-error bound
# ------------------------------------------------------------------------------------------------------------------
_DF = {sp.sin: torch.cos, sp.cos: lambda a: -torch.sin(a), sp.tanh: lambda a: 1 - torch.tanh(a) ** 2,
       sp.exp: torch.exp, sp.log: lambda a: 1 / a, sp.sinh: torch.cosh, sp.cosh: torch.sinh}
_F = {sp.sin: torch.sin, sp.cos: torch.cos, sp.tanh: torch.tanh, sp.exp: torch.exp, sp.log: torch.log,
      sp.sinh: torch.sinh, sp.cosh: torch.cosh}


def bound(e: sp.Basic, data: Dict[str, torch.Tensor], leafM: Dict[str, torch.Tensor], n: int,
          fragile: Optional[List[torch.Tensor]] = None, u: float = U32) -> Tuple[torch.Tensor, torch.Tensor]:
    """(value, M) of ``e`` (detached fp64 [n]).  ``fragile`` collects, per branch node (Abs, Max, Min), the points
    whose branch a rounding of u M could flip: there the kernel may take the other partial."""
    z = torch.zeros(n, dtype=torch.float64, device=next(iter(data.values())).device)

    def rec(e):
        if isinstance(e, (sp.Symbol, AppliedUndef)) and not _is_detach(e):
            nm = str(e) if isinstance(e, sp.Symbol) else e.func.__name__
            return data[nm].detach() + z, leafM.get(nm, z)
        if _is_detach(e):
            return rec(e.args[0])
        if e.is_Number or isinstance(e, sp.NumberSymbol):
            return z + float(e), z + abs(float(e))
        if isinstance(e, sp.Add):
            v, M = rec(e.args[0])
            for a in e.args[1:]:
                va, Ma = rec(a)
                v = v + va
                M = M + Ma + v.abs()
            return v, M
        if isinstance(e, sp.Mul):
            v, M = rec(e.args[0])
            for a in e.args[1:]:
                va, Ma = rec(a)
                M = va.abs() * M + v.abs() * Ma
                v = v * va
                M = M + v.abs()
            return v, M
        if isinstance(e, sp.Pow):
            a, Ma = rec(e.args[0])
            ex = e.args[1]
            if ex.is_Number:
                p = float(ex)
                f = a ** p
                # powi: one rounding per multiplication of the square-and-multiply, one more for 1 / r
                k = abs(int(p)) if ex.is_Integer else 0
                nr = max(1, k.bit_length() + bin(k).count("1") - 1 + (p < 0)) if ex.is_Integer else 1
                return f, (p * a ** (p - 1)).abs() * Ma + nr * f.abs()
            b, Mb = rec(ex)
            f = a ** b
            return f, (b * a ** (b - 1)).abs() * Ma + (f * torch.log(a)).abs() * Mb + f.abs()
        for cls, fn in _F.items():
            if isinstance(e, cls):
                a, Ma = rec(e.args[0])
                f = fn(a)
                return f, _DF[cls](a).abs() * Ma + f.abs()
        if isinstance(e, sp.tan):  # sin / cos: three roundings
            a, Ma = rec(e.args[0])
            f = torch.tan(a)
            return f, (1 + f * f) * Ma + 3 * f.abs()
        if isinstance(e, sp.Abs):
            a, Ma = rec(e.args[0])
            if fragile is not None:
                fragile.append((a.abs() <= 64 * u * Ma) & (Ma > 0))
            return a.abs(), Ma
        if isinstance(e, (sp.Max, sp.Min)):
            v, M = rec(e.args[0])
            for t in e.args[1:]:
                b, Mb = rec(t)
                if fragile is not None:
                    fragile.append(((v - b).abs() <= 64 * u * (M + Mb)) & (M + Mb > 0))
                pick = (v >= b) if isinstance(e, sp.Max) else (v <= b)
                v, M = torch.where(pick, v, b), torch.where(pick, M, Mb)
            return v, M
        if isinstance(e, (sp.sign, sp.Heaviside)):
            a, _ = rec(e.args[0])
            return (torch.sign(a) if isinstance(e, sp.sign) else torch.heaviside(a, z + 0.5)), z
        if isinstance(e, sp.Piecewise):
            (val, cond), rest = e.args[0], e.args[1:]
            if cond == sp.true:
                return rec(val)
            c = rec(cond.lhs)[0] == rec(cond.rhs)[0]
            va, Ma = rec(val)
            vb, Mb = rec(sp.Piecewise(*rest))
            return torch.where(c, va, vb), torch.where(c, Ma, Mb)
        raise NotImplementedError(f"bound: {type(e).__name__}")

    return rec(e)


# ------------------------------------------------------------------------------------------------------------------
# the reference of one head call
# ------------------------------------------------------------------------------------------------------------------
@dataclass
class Slot:
    """Loss options of one residual slot, as ``ResidualPlan.loss_fwd_bwd`` takes them."""
    label: Optional[str] = None  # None, "col" (a label column) or "const" (a label constant)
    weight: bool = False  # a per-point weight column
    reduction: str = "mean"
    loss_weight: float = 1.0
    out: bool = False  # the residual is also written to residual_out


@dataclass
class HeadRef:
    r: torch.Tensor  # [n_res, n]
    M: torch.Tensor  # [n_res, n] running-error bound
    loss: torch.Tensor  # [n_res]
    ybar: torch.Tensor  # [C, n, n_out]
    pgrad: Dict[str, torch.Tensor] = field(default_factory=dict)  # name -> scalar
    pgrad_abs: Dict[str, torch.Tensor] = field(default_factory=dict)  # name -> sum_p |term_p|
    fragile: Optional[torch.Tensor] = None  # [n] points where a branch could flip


def head_reference(cr, exprs: Sequence[sp.Basic], Y: torch.Tensor, X: torch.Tensor, aux: Dict[str, torch.Tensor],
                   params: Dict[str, float], labels: Sequence[torch.Tensor], weights: Sequence[Optional[torch.Tensor]],
                   slots: Sequence[Slot], n_norm: int, u: float) -> HeadRef:
    """fp64 reference of one head call.  Y [C, n, n_out] as the head read it, X [n_in, n], aux {name: [n]} data columns,
    params {name: value} learnable scalars, labels [n] per slot (zeros when none), weights [n] per slot or None."""
    n = Y.shape[1]
    Y64 = Y.double().detach().requires_grad_(True)
    dev = Y64.device
    P = {k: torch.full((n,), float(v), dtype=torch.float64, device=dev, requires_grad=True) for k, v in params.items()}
    data_aux = {k: v.double() for k, v in aux.items()}
    data_aux.update(P)
    sub, data, leafM = bind(cr, exprs, Y64, X.double(), data_aux)
    rs, Ms, frag = [], [], []
    total = torch.zeros((), dtype=torch.float64, device=dev)
    losses = []
    zero = torch.zeros(n, dtype=torch.float64, device=dev)
    for k, e in enumerate(sub):
        r, M = zero, zero
        for idx, eg in branch_groups(e, data, n):
            m = idx.numel()
            dg, lg = _take(data, idx, n), _take(leafM, idx, n)
            rg = O.eval_expr(eg, dg) + torch.zeros(m, dtype=torch.float64, device=dev)  # a constant residual
            fg: List[torch.Tensor] = []
            _, Mg = bound(eg, dg, lg, m, fg, u)
            r = r.index_put((idx,), rg)
            M = M.index_put((idx,), Mg)
            frag += [torch.zeros(n, dtype=torch.bool, device=dev).index_put((idx,), f) for f in fg]
        s = slots[k]
        coef = s.loss_weight / n_norm if s.reduction == "mean" else s.loss_weight
        err = r - labels[k].double()
        w = weights[k].double() if weights[k] is not None else 1.0
        lk = coef * (w * err * err).sum()
        losses.append(lk.detach())
        total = total + lk
        rs.append(r.detach())
        Ms.append(M)
    leaves = [Y64] + list(P.values())
    grads = torch.autograd.grad(total, leaves, allow_unused=True)
    ybar = grads[0] if grads[0] is not None else torch.zeros_like(Y64)
    pg, pga = {}, {}
    for (k, _), g in zip(P.items(), grads[1:]):
        g = g if g is not None else torch.zeros(n, dtype=torch.float64, device=dev)
        pg[k], pga[k] = g.sum(), g.abs().sum()
    fr = torch.stack(frag).any(0) if frag else torch.zeros(n, dtype=torch.bool, device=dev)
    return HeadRef(torch.stack(rs), torch.stack(Ms), torch.stack(losses), ybar.detach(), pg, pga, fr)


def errors(ref: HeadRef, u: float, r: Optional[torch.Tensor] = None, loss: Optional[torch.Tensor] = None,
           ybar: Optional[torch.Tensor] = None, pgrad: Optional[Dict[str, float]] = None,
           slots_out: Optional[Sequence[int]] = None) -> Dict[str, float]:
    """Errors in units of u: "res" max |r - r_ref| / (u M) over the slots ``slots_out`` of r [n_res, n]; "loss"
    relative; "ybar" per (channel, output) plane / its largest |ref| (points where a branch could flip left out);
    "pgrad" / sum_p |term_p|.  An element whose scale is zero must be exact (else inf)."""
    def ratio(d, s):
        return float(torch.where(s > 0, d / s.clamp_min(1e-300), torch.where(d > 0, math.inf, 0.0)).max()) / u

    e = {}
    if r is not None:
        ks = list(slots_out) if slots_out is not None else list(range(ref.r.shape[0]))
        if ks:
            d = (r[ks].double() - ref.r[ks]).abs()
            bad = ~torch.isfinite(r[ks].double())
            e["res"] = math.inf if bool(bad.any()) else ratio(d, ref.M[ks])
    if loss is not None:
        e["loss"] = ratio((loss.double() - ref.loss).abs(), ref.loss.abs())
    if ybar is not None:
        keep = ~ref.fragile
        yb, yr = ybar.double()[:, keep], ref.ybar[:, keep]
        if not bool(torch.isfinite(yb).all()):
            e["ybar"] = math.inf
        else:
            num = (yb - yr).abs().amax(1) if yb.shape[1] else torch.zeros(yr.shape[0], yr.shape[2], dtype=torch.float64)
            den = yr.abs().amax(1) if yr.shape[1] else torch.zeros_like(num)
            e["ybar"] = ratio(num, den)
    if pgrad:
        e["pgrad"] = max(ratio(torch.tensor(abs(float(pgrad[k]) - float(ref.pgrad[k]))), ref.pgrad_abs[k].cpu())
                         for k in pgrad)
    return e


# ------------------------------------------------------------------------------------------------------------------
# random residual programs
# ------------------------------------------------------------------------------------------------------------------
def layout_alphas(layout: str) -> List[Tuple[int, ...]]:
    """The derivative multi-indices the layout's own equation reads (so a program over them keeps its jet layout)."""
    spec = all_layouts()[layout]
    in_index = {k: i for i, k in enumerate(spec["in_keys"])}
    out = set()
    for e in spec["exprs"]().values():
        for d in sp.sympify(e).atoms(sp.Derivative):
            a = [0] * len(in_index)
            for s, o in d.variable_count:
                a[in_index[str(s)]] += int(o)
            out.add(tuple(a))
    return sorted(out)


def anchor(layout: str, out_key: str = "u") -> sp.Basic:
    """0.01 times the sum of every derivative the layout reads, of output ``out_key``: keeps the jet layout's C."""
    spec = all_layouts()[layout]
    syms = sp.symbols(spec["in_keys"])
    f = sp.Function(out_key)(*syms)
    terms = [f.diff(*[s for s, o in zip(syms, a) for _ in range(o)]) for a in layout_alphas(layout)]
    return sp.Float(0.01) * sp.Add(*terms) if terms else sp.Float(0.01) * f


class _Gen:
    """Random expressions over ``leaves``; ``S`` wraps a sympy atom for the tracing mode (ad.SymTensor and torch ops)
    or leaves it as is (sympy mode)."""

    def __init__(self, rng: random.Random, leaves, aux_masks: Sequence[str], traced: bool):
        self.rng, self.leaves, self.masks, self.traced = rng, leaves, list(aux_masks), traced

    def leaf(self):
        return self.rng.choice(self.leaves)

    def c(self, lo=-1.5, hi=1.5):
        return round(self.rng.uniform(lo, hi), 3)

    def expr(self, depth: int):
        rng, T = self.rng, self.traced
        if depth <= 0 or rng.random() < 0.2:
            return self.leaf()
        k = rng.randrange(22)
        a = self.expr(depth - 1)
        if k == 0:
            return a + self.expr(depth - 1)
        if k == 1:
            return a * self.expr(depth - 1)
        if k == 2:
            return a - self.c() * self.expr(depth - 1)
        if k == 3:
            return torch.log(1 + a * a) if T else sp.log(1 + a * a)
        if k == 4:
            return torch.sqrt(1 + a * a) if T else sp.sqrt(1 + a * a)
        if k == 5:
            return (1 + a * a) ** 1.5 if T else (1 + a * a) ** sp.Rational(3, 2)
        if k == 6:  # a Y-dependent exponent: pow's log partial
            b = self.expr(depth - 1)
            return (1 + a * a) ** torch.sin(b) if T else (1 + a * a) ** sp.sin(b)
        if k == 7:
            return a ** rng.choice([2, 3, 4, 5])
        if k == 8:  # negative powers of a base bounded away from 0
            base = (2 + torch.sin(a)) if T else (2 + sp.sin(a))
            return base ** rng.choice([-1, -2, -3])
        if k == 9:
            den = (2 + torch.sin(self.expr(depth - 1))) if T else (2 + sp.sin(self.expr(depth - 1)))
            return a / den
        if k == 10:
            return torch.tan(0.5 * torch.tanh(a)) if T else sp.tan(sp.Float(0.5) * sp.tanh(a))
        if k == 11:
            return torch.sinh(torch.tanh(a)) if T else sp.sinh(sp.tanh(a))
        if k == 12:
            return torch.cosh(torch.tanh(a)) if T else sp.cosh(sp.tanh(a))
        if k == 13:
            return torch.exp(torch.tanh(a)) if T else sp.exp(sp.tanh(a))
        if k == 14:
            return torch.abs(a) if T else sp.Abs(a)
        if k == 15:
            b = self.expr(depth - 1)
            return torch.maximum(a, b) if T else sp.Max(a, b)
        if k == 16:
            b = self.expr(depth - 1)
            return torch.minimum(a, b) if T else sp.Min(a, b)
        if k == 17:
            return a.detach() if T else sp.Function(DETACH_FUNC_NAME)(a)
        if k == 18 and self.masks:
            m = sp.Symbol(self.rng.choice(self.masks))
            b = self.expr(depth - 1)
            if T:
                return torch.where(ad.SymTensor(m) == 1.0, a, b)
            return sp.Piecewise((a, sp.Eq(m, 1)), (b, True))
        if k == 19:
            return torch.sin(a) if T else sp.sin(a)
        if k == 20:
            return torch.cos(a) if T else sp.cos(a)
        return torch.tanh(a) if T else sp.tanh(a)


def gen_residuals(seed: int, layout: str, out_keys: Sequence[str], n_res: int, depth: int = 3,
                  aux_cols: Sequence[str] = (), masks: Sequence[str] = (), params: Sequence[str] = ()) -> Dict[str, sp.Basic]:
    """``n_res`` random residuals over the layout's outputs ``out_keys`` and their derivatives (the layout's multi-indices),
    its inputs, the aux columns ``aux_cols`` and 0 / 1 ``masks`` (conditions of where), learnable ``params`` and
    constants; odd seeds trace torch callables through ad.SymTensor.  The first residual is the layout's anchor."""
    rng = random.Random(seed)
    traced = seed % 2 == 1
    spec = all_layouts()[layout]
    syms = sp.symbols(spec["in_keys"])
    atoms = []
    for k in out_keys:
        f = sp.Function(k)(*syms)
        atoms.append(f)
        for a in layout_alphas(layout):
            atoms.append(f.diff(*[s for s, o in zip(syms, a) for _ in range(o)]))
    atoms += list(syms) + [sp.Symbol(a) for a in aux_cols] + [sp.Symbol(p) for p in params]
    leaves = [ad.SymTensor(a) for a in atoms] if traced else atoms
    g = _Gen(rng, leaves, masks, traced)
    out = {"r0": anchor(layout, out_keys[0])}
    for i in range(1, n_res):
        e = g.expr(depth)
        if isinstance(e, ad.SymTensor):
            e = e.expr
        e = sp.sympify(e)
        if not e.free_symbols and not e.atoms(AppliedUndef):
            e = e + atoms[0]
        out[f"r{i}"] = e
    return out


def ops_of(cr) -> set:
    return {OP_NAMES[o[0]] for o in cr.prog}


# ------------------------------------------------------------------------------------------------------------------
# running one head call
# ------------------------------------------------------------------------------------------------------------------
@dataclass
class Run:
    plan: ResidualPlan
    cr: object
    exprs: List[sp.Basic]
    inputs: Dict[str, torch.Tensor]
    params: torch.Tensor
    labels: List[torch.Tensor]
    weights: List[Optional[torch.Tensor]]
    label_consts: Dict[str, float]
    slots: List[Slot]
    n: int
    n_norm: int
    learn: Dict[str, float]


def setup(layout: str, exprs: Dict[str, sp.Basic], n: int, *, dtype=torch.float32, hidden=(16, 16),
          out_keys: Optional[Sequence[str]] = None, slots: Optional[Sequence[Slot]] = None, n_norm: Optional[int] = None,
          aux_cols: Sequence[str] = (), masks: Sequence[str] = (), learn: Optional[Dict[str, float]] = None,
          tie: bool = False, backend: int = 2, library=None, device="cuda:0", seed: int = 0,
          chunk_points: int = 0, act: str = "tanh") -> Run:
    """A plan for the residuals ``exprs`` on an MLP over the layout's inputs with outputs ``out_keys``, and seeded inputs,
    parameters, aux columns (``masks``: 0 / 1 columns), labels and weights.  ``tie``: the last layer's weight and bias
    columns of output 1 copy output 0's (u and v equal bitwise)."""
    spec = all_layouts()[layout]
    out_keys = tuple(out_keys or spec["out_keys"])
    learn = dict(learn or {})
    torch.manual_seed(seed)
    net = make_net(spec["in_keys"], out_keys, list(hidden), act)
    cr = compile_residuals(net, exprs, param_keys=list(learn))
    learn = {k: v for k, v in learn.items() if k in cr.param_keys}
    names = cr.names
    slots = list(slots or [Slot() for _ in names])
    plan = ResidualPlan(cr, dtype, [s.reduction for s in slots], [s.loss_weight for s in slots], backend=backend,
                        library=library, chunk_points=chunk_points)
    dev = torch.device(device)
    params = O.xavier_uniform_params(net.widths, 1, torch.float64)
    params = params + 0.1 * torch.randn_like(params)
    if tie:
        w_sl, b_sl, (K, N) = param_blocks(net.widths)[-1]
        W = params[w_sl].view(K, N)
        W[:, 1] = W[:, 0]
        params[b_sl.start + 1] = params[b_sl.start]
    params = params.to(dtype).to(dev)
    inputs = {}
    for k in spec["in_keys"]:
        lo, hi = spec.get("ranges", {}).get(k, (0, 1))
        inputs[k] = (torch.rand(n, 1, dtype=torch.float64) * (hi - lo) + lo).to(dtype).to(dev)
    for k in aux_cols:
        inputs[k] = torch.randn(n, 1, dtype=torch.float64).to(dtype).to(dev)
    for k in masks:
        inputs[k] = (torch.rand(n, 1) < 0.5).to(dtype).to(dev)
    for k, v in learn.items():
        inputs[k] = torch.tensor([v], dtype=dtype, device=dev)
    labels, weights, lconst = [], [], {}
    for k, s in zip(names, slots):
        lab = torch.zeros(n, 1, dtype=dtype, device=dev)
        if s.label == "col":
            lab = (0.3 * torch.randn(n, 1, dtype=torch.float64)).to(dtype).to(dev)
        elif s.label == "const":
            lconst[k] = round(0.1 + 0.05 * len(lconst), 3)
            lab = torch.full((n, 1), float(torch.tensor(lconst[k], dtype=dtype)), dtype=dtype, device=dev)
        labels.append(lab)
        weights.append((0.5 + torch.rand(n, 1, dtype=torch.float64)).to(dtype).to(dev) if s.weight else None)
    return Run(plan, cr, [sp.sympify(exprs[k]) for k in names], inputs, params, labels, weights, lconst, slots, n,
               n_norm or n, learn)


def call(run: Run, poison: Optional[int] = None, grads: Optional[torch.Tensor] = None, want_grad: bool = True):
    """One fused loss_fwd_bwd of ``run``: (losses, {slot: residual_out}, grads).  ``poison``: fill the workspace with this
    byte before the call (0xFF: every float a NaN)."""
    plan, n, dev = run.plan, run.n, run.params.device
    ws = plan._workspace(n, dev)
    if poison is not None:
        ws.fill_(poison)
    outs = {k: torch.full((n, 1), math.nan, dtype=plan.dtype, device=dev)
            for i, k in enumerate(run.cr.names) if run.slots[i].out}
    if grads is None and want_grad:
        grads = torch.zeros_like(run.params)
    names = run.cr.names
    loss = plan.loss_fwd_bwd(run.inputs, run.params, grads,
                             labels={k: run.labels[i] for i, k in enumerate(names) if run.slots[i].label == "col"},
                             weights={k: run.weights[i] for i, k in enumerate(names) if run.weights[i] is not None},
                             label_consts=run.label_consts, n_norm=run.n_norm, residual_out=outs)
    return loss.clone(), outs, grads


def reference(run: Run, Y: torch.Tensor, x_off: int = 0) -> HeadRef:
    """``head_reference`` of ``run`` over points x_off .. x_off + Y.shape[1] - 1 from the output jets Y."""
    m = Y.shape[1]
    sl = slice(x_off, x_off + m)
    cr = run.cr
    X = torch.stack([run.inputs[k].view(-1)[sl] for k in cr.net.input_keys]).to(Y.device)
    aux = {k: run.inputs[k].view(-1)[sl].to(Y.device) for k in cr.aux_keys if k not in run.learn}
    learn = {k: float(run.inputs[k]) for k in run.learn}
    labels = [t.view(-1)[sl].to(Y.device) for t in run.labels]
    weights = [t.view(-1)[sl].to(Y.device) if t is not None else None for t in run.weights]
    u = U32 if run.plan.dtype == torch.float32 else U64
    return head_reference(cr, run.exprs, Y, X, aux, learn, labels, weights, run.slots, run.n_norm, u)


def views(run: Run, last: bool = False):
    return stash_views(run.plan, run.n, last=last)


# ------------------------------------------------------------------------------------------------------------------
# the checks of one case
# ------------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    layout: str
    exprs: Callable[[], Dict[str, sp.Basic]]
    n: int
    dtype: torch.dtype = torch.float32
    out_keys: Optional[Tuple[str, ...]] = None
    slots: Optional[List[Slot]] = None
    n_norm: Optional[int] = None
    aux_cols: Tuple[str, ...] = ()
    masks: Tuple[str, ...] = ()
    learn: Optional[Dict[str, float]] = None
    tie: bool = False
    hidden: Tuple[int, ...] = (16, 16)
    chunked: bool = False  # also a call over three workspace chunks
    min_reg: int = 0  # the program must need at least this many registers


def _bitwise(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.shape == b.shape and bool(torch.equal(a.contiguous().view(-1).view(torch.uint8 if a.dtype == torch.uint8 else
                                                                              (torch.int32 if a.element_size() == 4 else torch.int64)),
                                                   b.contiguous().view(-1).view(torch.uint8 if b.dtype == torch.uint8 else
                                                                              (torch.int32 if b.element_size() == 4 else torch.int64))))


def run_case(case: Case, *, library=None, device="cuda:0", backend: int = 2) -> Dict[str, float]:
    """Every check of ``case``: one call on a zeroed workspace (residuals, losses, Ybar, dLoss/dparameter against the
    reference), the same call on a workspace poisoned with NaN bytes (bitwise equal), ``plan.forward`` (residuals
    bitwise equal), the parameter-gradient buffer seeded over two calls, and for ``chunked`` a call over three chunks
    (residual_out and losses over all points, the last chunk's Ybar).  Returns the errors in units of the rounding."""
    n = case.n
    kw = dict(dtype=case.dtype, hidden=case.hidden, out_keys=case.out_keys, slots=case.slots, n_norm=case.n_norm,
              aux_cols=case.aux_cols, masks=case.masks, learn=case.learn, tie=case.tie, backend=backend,
              library=library, device=device)
    run = setup(case.layout, case.exprs(), n, chunk_points=max(n, 1024), **kw)
    cr, plan = run.cr, run.plan
    assert cr.n_reg >= case.min_reg, (cr.n_reg, case.min_reg)
    u = U32 if case.dtype == torch.float32 else U64
    nres = len(cr.names)
    outs_k = [k for k in range(nres) if run.slots[k].out]
    pbuf = plan.param_grad_buffer(run.params.device)
    if pbuf is not None:
        pbuf.zero_()
    run.plan._workspace(n, run.params.device).zero_()
    loss, outs, _ = call(run)
    pg = {k: float(pbuf[cr.aux_keys.index(k)]) for k in run.learn} if pbuf is not None else {}
    V = views(run)
    Y, Ybar = V["Y"].clone(), V["Ybar"].clone()
    assert bool(torch.isfinite(Y).all())
    if case.tie:
        assert _bitwise(Y[:, :, 0], Y[:, :, 1]), "u and v are not equal bitwise"
    ref = reference(run, Y)
    r = torch.stack([outs[cr.names[k]].view(-1) if k in outs_k else torch.zeros(n, dtype=plan.dtype, device=Y.device)
                     for k in range(nres)])
    e = errors(ref, u, r=r, loss=loss, ybar=Ybar, pgrad=pg, slots_out=outs_k)

    # the same call on a workspace of NaN bytes: the head and every kernel after it read only what the call wrote
    loss_p, outs_p, _ = call(run, poison=0xFF)
    Vp = views(run)
    for k in outs_k:
        assert _bitwise(outs_p[cr.names[k]], outs[cr.names[k]]), f"poisoned workspace: residual {cr.names[k]} differs"
    assert _bitwise(Vp["Ybar"], Ybar), "poisoned workspace: Ybar differs"
    # more head blocks add their fp64 partial losses atomically, in any order: within the rounding of that sum
    blocks = (n + 127) // 128
    assert _bitwise(loss_p, loss) if blocks == 1 else \
        torch.allclose(loss_p.double(), loss.double(), rtol=(blocks + 4) * max(u, U64), atol=0), \
        f"poisoned workspace: losses {loss_p.tolist()} != {loss.tolist()}"

    # forward only: the same residuals, bitwise
    _, res_f = plan.forward(run.inputs, run.params)
    for k in outs_k:
        assert _bitwise(res_f[cr.names[k]], outs[cr.names[k]]), f"plan.forward: residual {cr.names[k]} differs"

    # the parameter-gradient buffer accumulates: seed + the gradient of two calls
    if run.learn:
        seed = torch.tensor([0.25 * (i + 1) for i in range(len(cr.aux_keys))], dtype=torch.float64, device=pbuf.device)
        pbuf.copy_(seed)
        call(run)
        call(run)
        for k in run.learn:
            i = cr.aux_keys.index(k)
            want = float(seed[i]) + 2 * pg[k]
            scale = abs(float(seed[i])) + 2 * float(ref.pgrad_abs[k]) + abs(2 * pg[k])
            e["pgrad_acc"] = max(e.get("pgrad_acc", 0.0), abs(float(pbuf[i]) - want) / scale / u)

    if case.chunked:
        ch = (n + 2) // 3
        runc = setup(case.layout, case.exprs(), n, chunk_points=ch, **kw)
        assert runc.plan.chunk_points == ch
        lossc, outsc, _ = call(runc)
        x_off, m = last_chunk(runc.plan, n)
        Vc = views(runc, last=n > ch)
        assert _bitwise(Vc["Y"], Y[:, x_off:x_off + m]), "the chunked call's last chunk read other output jets"
        rc = torch.stack([outsc[cr.names[k]].view(-1) if k in outs_k else
                          torch.zeros(n, dtype=plan.dtype, device=Y.device) for k in range(nres)])
        ec = errors(ref, u, r=rc, loss=lossc, slots_out=outs_k)
        ref_last = reference(runc, Vc["Y"].clone(), x_off)
        ec.update({"ybar": errors(ref_last, u, ybar=Vc["Ybar"])["ybar"]})
        e.update({f"{k}_chunked": v for k, v in ec.items()})
    return e


# ------------------------------------------------------------------------------------------------------------------
# the case matrix (shared by the emulation and the GPU test)
# ------------------------------------------------------------------------------------------------------------------
def _xy():
    x, y = sp.symbols("x y")
    return x, y, sp.Function("u")(x, y), sp.Function("v")(x, y), sp.Function("p")(x, y)


def opcode_exprs() -> Dict[str, sp.Basic]:
    """One residual per opcode (Lay22: u, v, p over x, y; aux column a, 0 / 1 masks m, q).  sign, heaviside, eq, select
    and max as Or also come out of the partials of Abs, Max / Min and Piecewise."""
    x, y, u, v, p = _xy()
    a, m, q = sp.symbols("a m q")
    D = sp.Function(DETACH_FUNC_NAME)
    return {
        "add_sub_mul_fma": u.diff(x) + v.diff(y) - u * v + 0.37 * p.diff(x, 2) - x * y,
        "div_neg": -u / (2 + sp.sin(v)),
        "powi": (2 + sp.sin(u)) ** -3 + v ** 5 + p.diff(y, 2) ** 2,
        "pow": (1 + u ** 2) ** sp.sin(v) + (1 + p ** 2) ** sp.Rational(3, 2),
        "sin_cos_tan": sp.sin(u) * sp.cos(v.diff(x)) + sp.tan(sp.Float(0.5) * sp.tanh(p)),
        "tanh_exp_log_sqrt": sp.tanh(u.diff(y)) + sp.exp(sp.tanh(v)) + sp.log(1 + p ** 2) + sp.sqrt(1 + u ** 2),
        "sinh_cosh": sp.sinh(sp.tanh(u)) * sp.cosh(sp.tanh(v)),
        "abs_sign": sp.Abs(u - 0.1) + sp.sign(v) * p,
        "max_min": sp.Max(u, v) + sp.Min(u.diff(x), p) * a,
        "heaviside": sp.sign(u) * v + sp.Heaviside(u - 0.3) * u + sp.Heaviside(v, 0) * p + sp.Heaviside(p, 1) * u,
        "where": sp.Piecewise((u * v, sp.Eq(m, 1)), (sp.log(1 + p ** 2), True)),
        "where_or": sp.Piecewise((u + 1, sp.Eq(m, 1)), (2 * u, sp.Eq(q, 1)), (v, True)),
        "detach": D(u) * v.diff(x) + D(u * p) ** 2,
    }


def tie_exprs() -> Dict[str, sp.Basic]:
    """u and v equal bitwise (``Case.tie``): Max / Min hand each side half the adjoint, as torch.maximum does."""
    x, y, u, v, p = _xy()
    return {"max": sp.Max(u, v) * (1 + x), "min": sp.Min(u, v) + sp.Min(v, u) * y,
            "where_eq": sp.Piecewise((u * v + p, sp.Eq(u, v)), (sp.log(u - v), True)),
            "max3": sp.Max(u, v, p)}


def select_exprs() -> Dict[str, sp.Basic]:
    """Selects whose untaken branch is the log of a negative number or a division by zero."""
    x, y, u, v, p = _xy()
    m = sp.Symbol("m")
    return {"log_neg": sp.Piecewise((sp.log(m - sp.Rational(1, 2)) * u, sp.Eq(m, 1)), (u * v, True)),
            "div0": sp.Piecewise((u / (m - 1), sp.Eq(m, 0)), (v ** 2 + p, True)),
            "nested": sp.Piecewise((sp.sqrt(-1 - v ** 2), sp.Eq(m, 2)),
                                   (sp.Piecewise((p / (m - 1), sp.Eq(m, 0)), (u * p, True)), True))}


def register_limit_exprs(target: int = 248, seed: int = 11) -> Callable[[], Dict[str, sp.Basic]]:
    """Residuals over 8 outputs of the C = 29 layout (232 output-jet registers) whose program needs between
    ``target`` and 256 registers."""
    keys = tuple("uabcdefg")
    net = make_net(all_layouts()["O4x7"]["in_keys"], keys, [8], "tanh")
    for s in range(seed, seed + 200):
        for n_res in (4, 6, 8, 10, 12):
            ex = gen_residuals(s, "O4x7", keys, n_res, depth=3)
            try:
                cr = compile_residuals(net, ex)
            except NotImplementedError:
                break
            if cr.n_reg >= target:
                return lambda ex=ex: dict(ex)
    raise RuntimeError("no program reached the register target")


def slot_exprs() -> Dict[str, sp.Basic]:
    x, y, u, v, p = _xy()
    a = sp.Symbol("a")
    base = [u.diff(x) + v.diff(y), u * u.diff(x) + p.diff(x), sp.sin(u) - a * v, u.diff(x, 2) + v.diff(y, 2) - p]
    return {f"s{k}": base[k % 4] * (1 + 0.1 * k) + (k % 3) * a * u for k in range(16)}


SLOTS16 = [Slot(label=[None, "col", "const"][k % 3], weight=k % 4 in (1, 2), reduction="sum" if k % 5 == 2 else "mean",
                loss_weight=0.5 + 0.25 * k, out=k % 2 == 0) for k in range(16)]


def param_exprs() -> Dict[str, sp.Basic]:
    """Learnable parameters lam, mu, nu: 16 slots with 2 gradient terms each (32 = PPSCI_MAX_PGRAD), some inside detach."""
    x, y, u, v, p = _xy()
    lam, mu, nu = sp.symbols("lam mu nu")
    D = sp.Function(DETACH_FUNC_NAME)
    out = {}
    for k in range(16):
        pa, pb = [(lam, mu), (mu, nu), (nu, lam)][k % 3]
        t = pa * u.diff(x) + sp.sin(pb) * v * (1 + 0.1 * k) - p.diff(y, 2)
        if k % 4 == 3:
            t = t + D(pa * u) * p - D(pb * v) * u  # detached parameters: no terms of their own
        out[f"q{k}"] = t
    return out


def matrix(dtype: torch.dtype, gpu: bool) -> List[Case]:
    """The directed and random cases of one dtype; ``gpu`` adds the large point counts."""
    dt = "f64" if dtype == torch.float64 else "f32"
    all_out = [Slot(out=True)]
    cs: List[Case] = []
    ops = opcode_exprs()
    cs.append(Case(f"opcodes-{dt}", "Lay22", opcode_exprs, 37, dtype, slots=all_out * len(ops), aux_cols=("a",),
                   masks=("m", "q"), chunked=True))
    cs.append(Case(f"ties-{dt}", "Lay22", tie_exprs, 29, dtype, slots=all_out * 4, tie=True))
    cs.append(Case(f"selects-{dt}", "Lay22", select_exprs, 33, dtype, slots=all_out * 3, masks=("m",)))
    cs.append(Case(f"slots16-{dt}", "Lay22", slot_exprs, 45, dtype, slots=SLOTS16, n_norm=53, aux_cols=("a",),
                   chunked=True))
    cs.append(Case(f"params-{dt}", "Lay22", param_exprs, 3013 if gpu else 200, dtype, slots=all_out * 16,
                   learn={"lam": 0.7, "mu": -1.3, "nu": 0.45}))
    cs.append(Case(f"reglimit-{dt}", "O4x7", register_limit_exprs(), 9 if not gpu else 3013, dtype,
                   out_keys=tuple("uabcdefg"), slots=all_out * 16, hidden=(12, 12), min_reg=248))
    counts = (1, 127, 128, 129, 3013, 70001) if gpu else (1, 127, 128, 129)
    for n in counts:
        cs.append(Case(f"points{n}-{dt}", "Lay22", opcode_exprs, n, dtype, slots=all_out * len(ops), aux_cols=("a",),
                       masks=("m", "q"), chunked=n >= 3))
    for lay, outs, seeds in [("Lay22", ("u", "v", "p"), range(6)), ("Lay12", ("u",), range(6, 10)),
                             ("Lay4444", ("u",), range(10, 12)), ("O1222", ("u",), range(12, 14)),
                             ("LayV", ("u", "v"), range(14, 16))]:
        for s in seeds:
            cs.append(Case(f"random{s}-{lay}-{dt}", lay,
                           lambda s=s, lay=lay, outs=outs: gen_residuals(s, lay, outs, 5, aux_cols=("a",), masks=("m",),
                                                                        params=("lam",)),
                           3013 if gpu else 37, dtype, out_keys=outs, slots=[Slot(label="col", out=True)] * 5,
                           aux_cols=("a",), masks=("m",), learn={"lam": 0.6}, chunked=s % 2 == 0))
    return cs
