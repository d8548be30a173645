"""Residual compiler: sympy expressions -> (jet directions, register program).

This is the H100-native counterpart of ``ppsci.lambdify`` (reference:
ppsci/utils/symbolic.py:681-981).  The reference turns a sympy tree into a list of
``nn.Layer`` nodes whose ``DerivativeNode``s call reverse-mode ``paddle.grad``
(symbolic.py:270-403).  Here the same tree is compiled ONCE into

* the set of univariate Taylor directions (and orders) the forward-jet kernels must
  propagate so that every requested partial derivative is a fixed linear combination of
  propagated coefficients (polarisation; Griewank-Utke-Walther), and
* a straight-line register program evaluating all residuals r_k AND all partials
  d r_k / d (output-jet channel) — so the adjoint needs no autograd graph.  ``detach(...)``
  sub-expressions (ppsci/equation/pde/base.py:91-151) contribute values but no partials.
"""
from __future__ import annotations

import itertools
import math
from dataclasses import dataclass, field
from fractions import Fraction
from typing import Dict, List, Optional, Sequence, Tuple

import sympy as sp
from sympy.core.function import AppliedUndef

from . import binding as B

DETACH_FUNC_NAME = "detach"


def cvt_to_key(expr: sp.Basic) -> str:
    """String key of a sympy node — same naming scheme as the reference's ``_cvt_to_key``
    (ppsci/utils/symbolic.py:111-137): ``Derivative(u(x,y),(x,2))`` -> ``u__x__x``."""
    if isinstance(expr, AppliedUndef) and expr.func.__name__ == DETACH_FUNC_NAME:
        return f"{cvt_to_key(expr.args[0])}_{DETACH_FUNC_NAME}"
    if isinstance(expr, (sp.Symbol, sp.core.function.UndefinedFunction, sp.Function)):
        return expr.name if hasattr(expr, "name") else str(expr)
    if isinstance(expr, sp.Derivative):
        s = expr.args[0].name
        for sym, order in expr.args[1:]:
            s += f"__{sym}" * int(order)
        return s
    return str(expr)


@dataclass
class NetSpec:
    """Static description of an MLP (ppsci/arch/mlp.py:179-315) as the kernels see it."""

    input_keys: Tuple[str, ...]  # raw input columns, in order
    output_keys: Tuple[str, ...]
    feat_src: List[int]  # feature f reads raw input feat_src[f]
    feat_kind: List[int]  # 0 identity, 1 cos(w x), 2 sin(w x)
    feat_omega: List[float]
    widths: List[int]  # [n_feat, hidden..., n_out]
    act: str = "tanh"
    dense_in: bool = False  # the single input key is a row-major [N, n_feat] matrix (DeepONet branch net); values only
    act_first: Optional[str] = None  # activation of the FIRST linear layer's output when it differs (FourierEmbedding: "sin")
    # 1: ModifiedMLP (mlp.py:488-506): U / V embeddings from the features + y <- y U + (1 - y) V after every hidden layer
    # 2: PirateNet (mlp.py:617-624, 800-809): layer 1 is the Fourier embedding, U / V read its output, then blocks of three
    #    layers (gate, gate, x <- alpha h + (1 - alpha) x)
    gated: int = 0

    @property
    def n_params(self) -> int:
        n = sum(self.widths[i] * self.widths[i + 1] + self.widths[i + 1] for i in range(len(self.widths) - 1))
        if self.gated:  # [Wu | bu | Wv | bv] behind the layers (input: the features, or layer 1's output for kind 2)
            emb = 1 if (self.gated == 2 or self.act_first is not None) else 0  # the embeddings read layer 1's output
            n += 2 * (self.widths[emb] * self.widths[-2] + self.widths[-2])
        if self.gated == 2:  # one alpha per block
            n += (len(self.widths) - 3) // 3
        hidden = self.widths[(2 if self.act_first is not None else 1):-1]  # layers whose activation is ``act``
        if self.act == "stan":  # one beta per unit
            n += sum(hidden)
        elif self.act == "swish_b":  # one beta per layer
            n += len(hidden)
        return n


@dataclass
class Direction:
    vec: Tuple[int, ...]  # integer vector over the raw inputs
    order: int = 0


@dataclass
class CompiledResidual:
    net: NetSpec
    names: List[str]  # residual names, in loss order
    dirs: List[Direction]
    aux_keys: List[str]
    n_reg: int
    prog: List[Tuple[int, int, int, int]]
    consts: List[float]
    res_reg: List[int]
    grad_res: List[int]
    grad_in: List[int]
    grad_reg: List[int]
    # learnable equation parameters (ParameterNode, ppsci/utils/symbolic.py:471-485): aux keys that are ONE scalar, and
    # the (residual, aux index, register of d residual / d parameter) terms of their loss gradient
    param_keys: List[str] = field(default_factory=list)
    pgrad_res: List[int] = field(default_factory=list)
    pgrad_aux: List[int] = field(default_factory=list)
    pgrad_reg: List[int] = field(default_factory=list)
    # alpha (multi-index over raw inputs) -> [(dir index, coefficient)]; D^alpha u = sum c * k! * Y[dir,k]
    combos: Dict[Tuple[int, ...], List[Tuple[int, Fraction]]] = field(default_factory=dict)

    @property
    def channels(self) -> int:
        return 1 + sum(d.order for d in self.dirs)

    def channel_of(self, d: int, k: int) -> int:
        return 1 + sum(x.order for x in self.dirs[:d]) + (k - 1)


# ------------------------------------------------------------------------------------------
# direction selection (polarisation)
# ------------------------------------------------------------------------------------------
def _monomials(support: Sequence[int], k: int, n: int) -> List[Tuple[int, ...]]:
    out = []
    for comp in itertools.product(range(k + 1), repeat=len(support)):
        if sum(comp) == k:
            beta = [0] * n
            for s, c in zip(support, comp):
                beta[s] = c
            out.append(tuple(beta))
    return out


def _multinomial(k: int, beta: Sequence[int]) -> int:
    r = math.factorial(k)
    for b in beta:
        r //= math.factorial(b)
    return r


def _candidates(support: Sequence[int], n: int):
    """Integer direction vectors over ``support``: units first, then growing |v|_1."""
    seen = set()
    for s in support:
        v = [0] * n
        v[s] = 1
        seen.add(tuple(v))
        yield tuple(v)
    for bound in (1, 2, 3):
        cands = []
        for comp in itertools.product(range(-bound, bound + 1), repeat=len(support)):
            if all(c == 0 for c in comp):
                continue
            first = next(c for c in comp if c != 0)
            if first < 0:
                continue
            g = 0
            for c in comp:
                g = math.gcd(g, abs(c))
            if g != 1:
                continue
            v = [0] * n
            for s, c in zip(support, comp):
                v[s] = c
            v = tuple(v)
            if v in seen:
                continue
            cands.append(v)
        cands.sort(key=lambda v: (sum(abs(c) for c in v), sum(1 for c in v if c != 0), v))
        for v in cands:
            if v not in seen:
                seen.add(v)
                yield v


def select_directions(alphas: Sequence[Tuple[int, ...]], n: int):
    """Pick directions so that every multi-index in ``alphas`` is a linear combination of
    same-order directional derivatives.  Returns (dirs, combos)."""
    dirs: List[Direction] = []
    index: Dict[Tuple[int, ...], int] = {}
    combos: Dict[Tuple[int, ...], List[Tuple[int, Fraction]]] = {}

    def get_dir(v):
        if v not in index:
            index[v] = len(dirs)
            dirs.append(Direction(v, 0))
        return index[v]

    # axis directions first, in input order, so channel numbering is predictable
    for a in sorted(set(alphas), key=lambda a: (sum(a), tuple(-x for x in a))):
        for i, ai in enumerate(a):
            if ai > 0:
                v = tuple(1 if j == i else 0 for j in range(n))
                get_dir(v)
    # keep axis directions ordered by input index
    order = sorted(range(len(dirs)), key=lambda d: dirs[d].vec, reverse=True)
    dirs[:] = [dirs[d] for d in order]
    index = {d.vec: i for i, d in enumerate(dirs)}

    for a in sorted(set(alphas), key=lambda a: (sum(a), tuple(-x for x in a))):
        k = sum(a)
        support = [i for i, ai in enumerate(a) if ai > 0]
        if len(support) == 1:
            d = get_dir(tuple(1 if j == support[0] else 0 for j in range(n)))
            dirs[d].order = max(dirs[d].order, k)
            combos[a] = [(d, Fraction(1))]
            continue
        mons = _monomials(support, k, n)
        target = sp.Matrix([1 if m == a else 0 for m in mons])
        used: List[Tuple[int, ...]] = [d.vec for d in dirs if all(v == 0 for i, v in enumerate(d.vec) if i not in support)]
        gen = _candidates(support, n)
        solution = None
        while solution is None:
            rows = []
            for v in used:
                row = []
                for m in mons:
                    val = _multinomial(k, m)
                    for vi, mi in zip(v, m):
                        val *= vi**mi if mi > 0 else 1
                    row.append(val)
                rows.append(row)
            A = sp.Matrix(rows).T  # columns = directions
            try:
                sol, params = A.gauss_jordan_solve(target)
                sol = sol.subs({p: 0 for p in params})
                solution = [Fraction(int(sp.numer(x)), int(sp.denom(x))) for x in sol]
            except ValueError:
                nxt = next(gen, None)
                while nxt is not None and nxt in used:
                    nxt = next(gen, None)
                if nxt is None:
                    raise NotImplementedError(f"cannot find Taylor directions for derivative multi-index {a}")
                used.append(nxt)
        combo = []
        for v, c in zip(used, solution):
            if c != 0:
                d = get_dir(v)
                dirs[d].order = max(dirs[d].order, k)
                combo.append((d, c))
        combos[a] = combo
    # drop directions that ended up unused
    keep = [i for i, d in enumerate(dirs) if d.order > 0]
    remap = {old: new for new, old in enumerate(keep)}
    dirs = [dirs[i] for i in keep]
    combos = {a: [(remap[d], c) for d, c in lst] for a, lst in combos.items()}
    return dirs, combos


# ------------------------------------------------------------------------------------------
# program emission
# ------------------------------------------------------------------------------------------
class _Emitter:
    def __init__(self, n_fixed: int):
        self.n_fixed = n_fixed
        self.next = n_fixed
        self.free: List[int] = []
        self.ops: List[Tuple[int, int, int, int]] = []
        self.consts: List[float] = []
        self.const_index: Dict[float, int] = {}
        self.sym_reg: Dict[sp.Symbol, int] = {}
        self.max_reg = n_fixed

    def alloc(self) -> int:
        if self.free:
            return self.free.pop()
        r = self.next
        self.next += 1
        self.max_reg = max(self.max_reg, self.next)
        return r

    def release(self, reg: int, owned: bool):
        if owned:
            self.free.append(reg)

    def const(self, val: float) -> int:
        val = float(val)
        if val not in self.const_index:
            self.const_index[val] = len(self.consts)
            self.consts.append(val)
        r = self.alloc()
        self.ops.append((B.OPS["const"], r, self.const_index[val], 0))
        return r

    def op(self, name: str, dst: int, a: int, b: int = 0):
        self.ops.append((B.OPS[name], dst, a, b))

    def _dst(self, reg: int, owned: bool) -> int:
        return reg if owned else self.alloc()

    def emit(self, e: sp.Basic) -> Tuple[int, bool]:
        """Returns (register, owned)."""
        if isinstance(e, sp.Symbol):
            if e not in self.sym_reg:
                raise NotImplementedError(f"unbound symbol {e} in residual expression")
            return self.sym_reg[e], False
        if e.is_Number or isinstance(e, sp.NumberSymbol):
            return self.const(float(e)), True
        if isinstance(e, sp.Add):
            terms = list(e.args)
            # put a non-negated term first so that a - b patterns become SUB
            acc, own = self.emit(terms[0])
            for t in terms[1:]:
                coeff, rest = t.as_coeff_Mul()
                if coeff == -1 and rest != 1:
                    r, o = self.emit(rest)
                    dst = self._dst(acc, own)
                    self.op("sub", dst, acc, r)
                elif coeff.is_Number and coeff != 1 and rest != 1 and not rest.is_Number:
                    # acc += coeff * rest  (FMA form needs the accumulator in dst)
                    rc = self.const(float(coeff))
                    r, o = self.emit(rest)
                    dst = self._dst(acc, own)
                    if dst != acc:
                        self.op("mov", dst, acc)
                    self.op("fma", dst, rc, r)
                    self.release(rc, True)
                else:
                    r, o = self.emit(t)
                    dst = self._dst(acc, own)
                    self.op("add", dst, acc, r)
                self.release(r, o)
                acc, own = dst, True
            return acc, own
        if isinstance(e, sp.Mul):
            coeff, rest = e.as_coeff_Mul()
            if coeff == -1:
                r, o = self.emit(rest)
                dst = self._dst(r, o)
                self.op("neg", dst, r)
                return dst, True
            acc, own = self.emit(e.args[0])
            for t in e.args[1:]:
                if isinstance(t, sp.Pow) and t.exp == -1:
                    r, o = self.emit(t.base)
                    dst = self._dst(acc, own)
                    self.op("div", dst, acc, r)
                else:
                    r, o = self.emit(t)
                    dst = self._dst(acc, own)
                    self.op("mul", dst, acc, r)
                self.release(r, o)
                acc, own = dst, True
            return acc, own
        if isinstance(e, sp.Pow):
            base, ex = e.args
            if ex.is_Integer and abs(int(ex)) <= 64:
                r, o = self.emit(base)
                dst = self._dst(r, o)
                self.op("powi", dst, r, int(ex))
                return dst, True
            if ex == sp.Rational(1, 2):
                r, o = self.emit(base)
                dst = self._dst(r, o)
                self.op("sqrt", dst, r)
                return dst, True
            rb, ob = self.emit(base)
            re_, oe = self.emit(ex)
            dst = self._dst(rb, ob)
            self.op("pow", dst, rb, re_)
            self.release(re_, oe)
            return dst, True
        unary = {
            sp.sin: "sin", sp.cos: "cos", sp.tanh: "tanh", sp.exp: "exp", sp.log: "log",
            sp.Abs: "abs", sp.sign: "sign", sp.sinh: "sinh", sp.cosh: "cosh", sp.Heaviside: "heaviside",
        }
        for cls, name in unary.items():
            if isinstance(e, cls):
                r, o = self.emit(e.args[0])
                dst = self._dst(r, o)
                self.op(name, dst, r)
                return dst, True
        if isinstance(e, (sp.Max, sp.Min)):
            name = "max" if isinstance(e, sp.Max) else "min"
            acc, own = self.emit(e.args[0])
            for t in e.args[1:]:
                r, o = self.emit(t)
                dst = self._dst(acc, own)
                self.op(name, dst, acc, r)
                self.release(r, o)
                acc, own = dst, True
            return acc, own
        if isinstance(e, sp.tan):
            rs, os_ = self.emit(sp.sin(e.args[0]))
            rc, oc = self.emit(sp.cos(e.args[0]))
            dst = self._dst(rs, os_)
            self.op("div", dst, rs, rc)
            self.release(rc, oc)
            return dst, True
        raise NotImplementedError(
            f"The node {e} (type {type(e).__name__}) is not supported in the residual program."
        )


def _is_detach(e: sp.Basic) -> bool:
    return isinstance(e, AppliedUndef) and e.func.__name__ == DETACH_FUNC_NAME


def compile_residuals(
    net: NetSpec,
    exprs: Dict[str, sp.Basic],
    aux_keys: Optional[Sequence[str]] = None,
    with_grad: bool = True,
    param_keys: Optional[Sequence[str]] = None,
) -> CompiledResidual:
    """Compile residual expressions for ``net``.

    ``exprs`` maps residual name -> sympy expression over
      * ``Symbol`` named like a raw input key        -> that input column
      * ``f(x, y, ...)`` with f in ``net.output_keys``  -> network output value
      * ``Derivative(f(...), ...)``                   -> input derivative of a network output
      * any other ``Symbol`` / applied function       -> auxiliary data column of that name
      * ``detach(sub)``                              -> value of sub, no gradient
    ``param_keys``: names among those auxiliary symbols that are learnable scalar parameters of the equation
    (``PDE.learnable_parameters``): one value for all points, and the program also carries d residual / d parameter.
    """
    n_in = len(net.input_keys)
    n_out = len(net.output_keys)
    in_index = {k: i for i, k in enumerate(net.input_keys)}
    out_index = {k: i for i, k in enumerate(net.output_keys)}
    aux_list: List[str] = list(aux_keys or [])

    names = list(exprs.keys())
    raw = [sp.sympify(exprs[n]) for n in names]

    # ---- 1. collect derivative multi-indices ------------------------------------------------
    alphas = set()
    for e in raw:
        for d in e.atoms(sp.Derivative):
            f = d.args[0]
            if _is_detach(f):
                f = f.args[0]
            if not (isinstance(f, AppliedUndef) and f.func.__name__ in out_index):
                raise NotImplementedError(
                    f"derivative of {f} is not supported: only derivatives of network outputs "
                    f"{net.output_keys} w.r.t. inputs {net.input_keys} can be compiled"
                )
            alpha = [0] * n_in
            for sym, order in d.variable_count:
                if str(sym) not in in_index:
                    raise NotImplementedError(f"derivative w.r.t. {sym}, which is not a network input")
                alpha[in_index[str(sym)]] += int(order)
            if sum(alpha) > B.MAX_ORDER:
                raise NotImplementedError(f"derivative order {sum(alpha)} > {B.MAX_ORDER} is not supported")
            alphas.add(tuple(alpha))
    dirs, combos = select_directions(sorted(alphas), n_in)
    if len(dirs) > B.MAX_DIR:
        raise NotImplementedError(f"{len(dirs)} Taylor directions needed (max {B.MAX_DIR})")
    C = 1 + sum(d.order for d in dirs)
    if C > 32:
        raise NotImplementedError(f"{C} jet channels needed (max 32)")

    def chan(d: int, k: int) -> int:
        return 1 + sum(x.order for x in dirs[:d]) + (k - 1)

    # ---- 2. rewrite expressions over register symbols ----------------------------------------
    ysym = {}  # (channel, out) -> Symbol

    def Y(c: int, j: int) -> sp.Symbol:
        if (c, j) not in ysym:
            ysym[(c, j)] = sp.Symbol(f"Y_{c}_{j}", real=True)
        return ysym[(c, j)]

    xsym = [sp.Symbol(f"X_{i}", real=True) for i in range(n_in)]
    auxsym: Dict[str, sp.Symbol] = {}

    def aux(name: str) -> sp.Symbol:
        if name not in aux_list:
            aux_list.append(name)
        if name not in auxsym:
            auxsym[name] = sp.Symbol(f"A_{name}", real=True)
        return auxsym[name]

    def lower(e: sp.Basic) -> sp.Basic:
        if isinstance(e, sp.Derivative):
            f = e.args[0]
            if _is_detach(f):
                f = f.args[0]
            j = out_index[f.func.__name__]
            alpha = [0] * n_in
            for sym, order in e.variable_count:
                alpha[in_index[str(sym)]] += int(order)
            alpha = tuple(alpha)
            k = sum(alpha)
            return sp.Add(*[sp.Rational(c.numerator, c.denominator) * math.factorial(k) * Y(chan(d, k), j)
                            for d, c in combos[alpha]])
        if isinstance(e, AppliedUndef):
            nm = e.func.__name__
            if nm == DETACH_FUNC_NAME:
                return sp.Function(DETACH_FUNC_NAME)(lower(e.args[0]))
            if nm in out_index:
                return Y(0, out_index[nm])
            if nm in in_index:
                return xsym[in_index[nm]]
            return aux(nm)
        if isinstance(e, sp.Symbol):
            nm = str(e)
            if nm in in_index:
                return xsym[in_index[nm]]
            if nm in out_index:
                return Y(0, out_index[nm])
            return aux(nm)
        if not e.args:
            return e
        return e.func(*[lower(a) for a in e.args])

    lowered = [lower(e) for e in raw]

    # ---- 3. detach handling and symbolic partials ---------------------------------------------
    det_subs: Dict[sp.Symbol, sp.Basic] = {}

    def strip_detach(e: sp.Basic) -> sp.Basic:
        if _is_detach(e):
            inner = strip_detach(e.args[0])
            s = sp.Symbol(f"DET_{len(det_subs)}", real=True)
            det_subs[s] = inner
            return s
        if not e.args:
            return e
        return e.func(*[strip_detach(a) for a in e.args])

    stripped = [strip_detach(e) for e in lowered]

    def restore(e: sp.Basic) -> sp.Basic:
        # detach symbols may be nested; substitute until none is left
        for _ in range(len(det_subs) + 1):
            syms = [s for s in e.free_symbols if s in det_subs]
            if not syms:
                break
            e = e.xreplace({s: det_subs[s] for s in syms})
        return e

    values = [restore(e) for e in stripped]
    grads: List[Tuple[int, int, sp.Basic]] = []  # (res k, input reg idx, expr)
    if with_grad:
        for k, e in enumerate(stripped):
            for (c, j), s in sorted(ysym.items()):
                if s in e.free_symbols:
                    g = sp.diff(e, s)
                    if g != 0:
                        grads.append((k, c * n_out + j, restore(g)))
    grads.sort(key=lambda t: (t[1], t[0]))
    param_set = set(param_keys or [])
    pgrads: List[Tuple[int, int, sp.Basic]] = []  # (res k, aux index, expr)
    if with_grad:
        for k, e in enumerate(stripped):
            for nm, s_ in auxsym.items():
                if nm in param_set and s_ in e.free_symbols:
                    g = sp.diff(e, s_)
                    if g != 0:
                        pgrads.append((k, aux_list.index(nm), restore(g)))
    if len(pgrads) > B.MAX_PGRAD:
        raise NotImplementedError(f"{len(pgrads)} (residual, learnable parameter) gradient terms (max {B.MAX_PGRAD})")

    # ---- 4. CSE + emission -------------------------------------------------------------------
    n_fixed = C * n_out + n_in + len(aux_list)
    all_exprs = values + [g for _, _, g in grads] + [g for _, _, g in pgrads]
    repl, reduced = sp.cse(all_exprs, order="none") if all_exprs else ([], [])
    em = _Emitter(n_fixed)
    for (c, j), s in ysym.items():
        em.sym_reg[s] = c * n_out + j
    for i, s in enumerate(xsym):
        em.sym_reg[s] = C * n_out + i
    for nm, s in auxsym.items():
        em.sym_reg[s] = C * n_out + n_in + aux_list.index(nm)
    # liveness of CSE temporaries
    stmts = [e for _, e in repl] + list(reduced)
    last_use: Dict[sp.Symbol, int] = {}
    for idx, e in enumerate(stmts):
        for s in e.free_symbols:
            last_use[s] = idx
    n_repl = len(repl)
    for idx in range(n_repl, len(stmts)):  # temps referenced directly by outputs live to the end
        for s in stmts[idx].free_symbols:
            last_use[s] = len(stmts)
    temp_owned: Dict[sp.Symbol, int] = {}
    for idx, (s, e) in enumerate(repl):
        r, owned = em.emit(e)
        if not owned:  # alias of an input/temp: copy so lifetime bookkeeping stays simple
            r2 = em.alloc()
            em.op("mov", r2, r)
            r = r2
        em.sym_reg[s] = r
        temp_owned[s] = r
        for t, reg in list(temp_owned.items()):
            if last_use.get(t, -1) <= idx and t is not s:
                em.free.append(reg)
                del temp_owned[t]
    out_regs = []
    for e in reduced:
        r, owned = em.emit(e)
        out_regs.append(r)  # never released: outputs stay live until the program ends
    n_res = len(values)
    cr = CompiledResidual(
        net=net,
        names=names,
        dirs=dirs,
        aux_keys=aux_list,
        n_reg=max(em.max_reg, n_fixed),
        prog=em.ops,
        consts=em.consts,
        res_reg=out_regs[:n_res],
        grad_res=[k for k, _, _ in grads],
        grad_in=[i for _, i, _ in grads],
        grad_reg=out_regs[n_res:n_res + len(grads)],
        combos=combos,
        param_keys=[nm for nm in aux_list if nm in param_set],
        pgrad_res=[k for k, _, _ in pgrads],
        pgrad_aux=[a for _, a, _ in pgrads],
        pgrad_reg=out_regs[n_res + len(grads):],
    )
    if cr.n_reg > B.MAX_REG:
        raise NotImplementedError(f"residual program needs {cr.n_reg} registers (max {B.MAX_REG})")
    return cr
