"""Host logic of the residual compiler: direction selection (polarisation), register programs,
detach handling, naming — checked with a tiny numpy interpreter of the emitted program."""
import itertools
import math
from fractions import Fraction

import numpy as np
import pytest
import sympy as sp

from paddlescience_b200.engine import binding as B
from paddlescience_b200.engine.compiler import (NetSpec, compile_residuals, cvt_to_key, select_directions)


def test_cvt_to_key_matches_reference_naming():
    x, y = sp.symbols("x y")
    u = sp.Function("u")(x, y)
    assert cvt_to_key(u) == "u"
    assert cvt_to_key(u.diff(x, 2).diff(y, 2)) == "u__x__x__y__y"
    assert cvt_to_key(sp.Function("detach")(u.diff(y))) == "u__y_detach"
    assert cvt_to_key(x) == "x"


@pytest.mark.parametrize("alphas,expect_channels", [
    ([(1, 0), (0, 1), (2, 0), (0, 2)], 5),          # Navier-Stokes 2D
    ([(1, 0), (0, 2)], 4),                            # Allen-Cahn (t: 1, x: 2)
    ([(4, 0), (0, 4), (2, 2)], 17),                   # biharmonic: 4 directions x order 4
    ([(2, 0, 0), (0, 2, 0), (0, 0, 2)], 7),           # Laplace 3D
    ([(1, 1)], 7),                                    # mixed second derivative
])
def test_direction_selection_reproduces_every_partial(alphas, expect_channels):
    n = len(alphas[0])
    dirs, combos = select_directions(alphas, n)
    assert 1 + sum(d.order for d in dirs) == expect_channels
    # verify the polarisation identities on a random polynomial of total degree <= 4
    rng = np.random.RandomState(0)
    xs = sp.symbols(f"x0:{n}")
    poly = sum(rng.randn() * sp.prod([xs[i] ** e for i, e in enumerate(ex)])
               for ex in itertools.product(range(5), repeat=n) if sum(ex) <= 4)
    pt = {xs[i]: rng.rand() for i in range(n)}
    t = sp.Symbol("t")
    for a in alphas:
        k = sum(a)
        exact = sp.diff(poly, *[v for i, v in enumerate(xs) for _ in range(a[i])]).subs(pt)
        acc = 0
        for d, c in combos[a]:
            line = poly.subs({xs[i]: xs[i] + t * dirs[d].vec[i] for i in range(n)}, simultaneous=True)
            dk = sp.diff(line, t, k).subs(t, 0).subs(pt)
            acc += sp.Rational(c.numerator, c.denominator) * dk
            assert dirs[d].order >= k
        assert abs(float(acc - exact)) < 1e-8 * max(1.0, abs(float(exact))), (a, float(acc), float(exact))


def _run_program(cr, regs):
    """numpy interpreter of the register program (mirrors vm_run in csrc/kernels_simt.cuh)."""
    ops = {v: k for k, v in B.OPS.items()}
    r = list(regs) + [0.0] * (cr.n_reg - len(regs))
    for op, dst, a, b in cr.prog:
        name = ops[op]
        if name == "const": v = cr.consts[a]
        elif name == "mov": v = r[a]
        elif name == "add": v = r[a] + r[b]
        elif name == "sub": v = r[a] - r[b]
        elif name == "mul": v = r[a] * r[b]
        elif name == "div": v = r[a] / r[b] if r[b] != 0 else math.copysign(math.inf, r[a]) if r[a] else math.nan
        elif name == "neg": v = -r[a]
        elif name == "powi": v = r[a] ** b
        elif name == "pow": v = r[a] ** r[b]
        elif name == "fma": v = r[a] * r[b] + r[dst]
        elif name == "sqrt": v = math.sqrt(r[a]) if r[a] >= 0 else math.nan
        elif name == "log": v = math.log(r[a]) if r[a] > 0 else (-math.inf if r[a] == 0 else math.nan)
        elif name in ("sin", "cos", "tanh", "exp", "sinh", "cosh"): v = getattr(math, name)(r[a])
        elif name == "abs": v = abs(r[a])
        elif name == "max": v = max(r[a], r[b])
        elif name == "min": v = min(r[a], r[b])
        elif name == "sign": v = float(r[a] > 0) - float(r[a] < 0)
        elif name == "heaviside": v = 1.0 if r[a] > 0 else (0.0 if r[a] < 0 else 0.5)
        elif name == "eq": v = 1.0 if r[a] == r[b] else 0.0
        elif name == "select": v = r[a] if r[dst] != 0 else r[b]  # never a blend: the untaken side may be NaN
        else: raise AssertionError(name)
        r[dst] = v
    return r


def test_program_values_and_partials_against_sympy():
    x, y = sp.symbols("x y")
    u = sp.Function("u")(x, y)
    v = sp.Function("v")(x, y)
    nu = 0.01
    exprs = {
        "r1": u * u.diff(x) + v * u.diff(y) - nu * (u.diff(x, 2) + u.diff(y, 2)) + sp.sin(x) * v ** 3 / (1 + y ** 2),
        "r2": sp.Function("detach")(u) * v.diff(y) + sp.exp(-u) * sp.sqrt(1 + v ** 2),
    }
    net = NetSpec(("x", "y"), ("u", "v"), [0, 1], [0, 0], [0.0, 0.0], [2, 8, 2], "tanh")
    cr = compile_residuals(net, exprs)
    C, m = cr.channels, 2
    rng = np.random.RandomState(1)
    Y = rng.randn(C, m)
    X = rng.rand(2)
    regs = list(Y.reshape(-1)) + list(X)
    r = _run_program(cr, regs)
    # independent evaluation with sympy
    chan = {(0, 0): 0}
    def val(name_idx, alpha):
        k = sum(alpha)
        if k == 0:
            return Y[0, name_idx]
        return sum(float(c) * math.factorial(k) * Y[cr.channel_of(d, k), name_idx] for d, c in cr.combos[alpha])
    subs = {u: val(0, (0, 0)), v: val(1, (0, 0)), x: X[0], y: X[1]}
    for a in [(1, 0), (0, 1), (2, 0), (0, 2)]:
        for j, f in enumerate((u, v)):
            d = sp.Derivative(f, *[s for i, s in enumerate((x, y)) for _ in range(a[i])])
            subs[d] = val(j, a)
    for k, name in enumerate(cr.names):
        e = exprs[name].replace(lambda z: getattr(z.func, "__name__", "") == "detach", lambda z: z.args[0])
        want = float(e.subs(subs))
        assert r[cr.res_reg[k]] == pytest.approx(want, rel=1e-12), name
    # partials by finite differences of the program itself; detached factor must contribute none
    eps = 1e-6
    dense = np.zeros((len(cr.names), C * m))
    for g_res, g_in, g_reg in zip(cr.grad_res, cr.grad_in, cr.grad_reg):
        dense[g_res, g_in] += r[g_reg]
    for idx in range(C * m):
        rp = _run_program(cr, [regs[i] + (eps if i == idx else 0) for i in range(len(regs))])
        rm = _run_program(cr, [regs[i] - (eps if i == idx else 0) for i in range(len(regs))])
        for k in range(len(cr.names)):
            fd = (rp[cr.res_reg[k]] - rm[cr.res_reg[k]]) / (2 * eps)
            if k == 1 and idx == 0:  # d r2 / d u has a detached part: analytic = only the exp(-u) term
                want = float((-sp.exp(-u) * sp.sqrt(1 + v ** 2)).subs(subs))
                assert dense[k, idx] == pytest.approx(want, rel=1e-9)
            else:
                assert dense[k, idx] == pytest.approx(fd, rel=2e-5, abs=2e-7), (k, idx)
    assert list(cr.grad_in) == sorted(cr.grad_in)


def test_unsupported_nodes_raise():
    x, y = sp.symbols("x y")
    u = sp.Function("u")(x, y)
    net = NetSpec(("x", "y"), ("u",), [0, 1], [0, 0], [0.0, 0.0], [2, 8, 1], "tanh")
    with pytest.raises(NotImplementedError):
        compile_residuals(net, {"r": u.diff(x, 5)})
    q = sp.Function("q")(x, y)
    with pytest.raises(NotImplementedError):
        compile_residuals(net, {"r": q.diff(x)})  # derivative of a data field
    cr = compile_residuals(net, {"r": u.diff(x) + q})  # a data field itself becomes an aux column
    assert cr.aux_keys == ["q"]


def _net1():
    return NetSpec(("x", "y"), ("u", "v"), [0, 1], [0, 0], [0.0, 0.0], [2, 8, 2], "tanh")


def _partials(cr, regs, k=0):
    """{input register: d residual k / d register} of the program at ``regs``."""
    r = _run_program(cr, regs)
    out = {}
    for g_res, g_in, g_reg in zip(cr.grad_res, cr.grad_in, cr.grad_reg):
        if g_res == k:
            out[g_in] = out.get(g_in, 0.0) + r[g_reg]
    return r[cr.res_reg[k]], out


def test_sign_and_heaviside_partials_drop_dirac_delta():
    """d sign(u) / du and d Heaviside(u - c) / du are DiracDelta terms: zero almost everywhere (as autograd has them),
    so the program compiles and only the other factors contribute."""
    x, y = sp.symbols("x y")
    u, v = sp.Function("u")(x, y), sp.Function("v")(x, y)
    cr = compile_residuals(_net1(), {"r": sp.sign(u) * v + sp.Heaviside(u - 0.3) * u})
    names = {B.OPS[o]: o for o in B.OPS}
    assert {"sign", "heaviside"} <= {names[op] for op, *_ in cr.prog}
    for uu, vv in [(0.7, -1.2), (-0.4, 2.0), (0.1, 0.5)]:
        regs = [uu, vv] + [0.0] * (2 * cr.channels - 2) + [0.2, 0.3]
        val, d = _partials(cr, regs)
        assert val == pytest.approx(np.sign(uu) * vv + (uu > 0.3) * uu)
        assert d.get(0, 0.0) == pytest.approx(float(uu > 0.3))  # d / du: the step, no delta
        assert d.get(1, 0.0) == pytest.approx(np.sign(uu))  # d / dv
    # a learnable parameter inside a step has no gradient term at all
    lam = sp.Symbol("lam")
    cr = compile_residuals(_net1(), {"r": sp.Heaviside(lam - u) * v}, param_keys=["lam"])
    assert cr.pgrad_reg == []


@pytest.mark.parametrize("h0", [0, 1, sp.Rational(1, 2), 0.25])
def test_heaviside_value_at_zero_is_honoured(h0):
    """Heaviside(a, H0) is H0 at a == 0 (sympy's default 1/2 is the HEAVISIDE op), 0 below and 1 above."""
    x, y = sp.symbols("x y")
    u, v = sp.Function("u")(x, y), sp.Function("v")(x, y)
    cr = compile_residuals(_net1(), {"r": sp.Heaviside(u - v, h0) + 2 * sp.Heaviside(u, h0)})
    for uu, vv, want in [(0.0, 0.0, 3 * float(h0)), (0.5, 0.5, float(h0) + 2), (0.0, -1.0, 1 + 2 * float(h0)),
                         (-0.5, 1.0, 0.0), (0.5, -1.0, 3.0)]:
        regs = [uu, vv] + [0.0] * (2 * cr.channels - 2) + [0.2, 0.3]
        assert _run_program(cr, regs)[cr.res_reg[0]] == want, (h0, uu, vv)


def test_heaviside_with_a_non_constant_value_at_zero_raises():
    x, y = sp.symbols("x y")
    u = sp.Function("u")(x, y)
    with pytest.raises(NotImplementedError, match="H0"):
        compile_residuals(_net1(), {"r": sp.Heaviside(u, x)})


def test_every_opcode_against_sympy_values_and_autograd_partials():
    """A program that runs all 25 opcodes (sign / heaviside / eq / select / max-as-Or through the partials of
    Abs, Max / Min, Heaviside and where): values against sympy, partials against torch autograd of the same expression."""
    import torch

    from oracle.ppsci_oracle import eval_expr

    x, y = sp.symbols("x y")
    u, v = sp.Function("u")(x, y), sp.Function("v")(x, y)
    m, q = sp.symbols("m q")
    exprs = {
        "a": u.diff(x) + v * u - 0.37 * u.diff(y, 2) - x / (2 + sp.sin(v)) + (2 + sp.cos(u)) ** -3,
        "b": (1 + u ** 2) ** sp.sin(v) + sp.sqrt(1 + v ** 2) + sp.log(1 + u ** 2) + sp.exp(sp.tanh(v)),
        "c": sp.sinh(sp.tanh(u)) * sp.cosh(v) + sp.tan(sp.Float(0.5) * sp.tanh(u)) - sp.Abs(u - v) * v ** 5,
        "d": sp.Max(u, v) - sp.Min(u, y) + sp.sign(v) * u + sp.Heaviside(u, 0) * v,
        "e": sp.Piecewise((u + 1, sp.Eq(m, 1)), (2 * u * v, sp.Eq(q, 1)), (sp.log(1 + v ** 2), True)),
    }
    cr = compile_residuals(_net1(), exprs)
    names = {B.OPS[o]: o for o in B.OPS}
    assert {names[op] for op, *_ in cr.prog} == set(B.OPS)
    rng = np.random.RandomState(3)
    for mm, qq in [(1.0, 0.0), (0.0, 1.0), (0.0, 0.0)]:
        Y = rng.randn(cr.channels, 2)
        X = rng.rand(2)
        regs = [float(t) for t in Y.reshape(-1)] + [float(t) for t in X] + [{"m": mm, "q": qq}[k] for k in cr.aux_keys]
        r = _run_program(cr, regs)
        Yt = torch.tensor(Y, requires_grad=True)
        data = {"u": Yt[0, 0:1], "v": Yt[0, 1:2], "x": torch.tensor([X[0]]), "y": torch.tensor([X[1]]),
                "m": torch.tensor([mm]), "q": torch.tensor([qq])}
        for a in [(1, 0), (0, 2)]:
            k = sum(a)
            key = f"_D{a}"
            data[key] = sum(float(c) * math.factorial(k) * Yt[cr.channel_of(d, k), 0:1] for d, c in cr.combos[a])
        subs = {u.diff(x): sp.Symbol("_D(1, 0)"), u.diff(y, 2): sp.Symbol("_D(0, 2)")}
        for k, name in enumerate(cr.names):
            e = exprs[name].xreplace(subs)
            if isinstance(e, sp.Piecewise):  # the branch the mask selects
                e = {(1.0, 0.0): e.args[0][0], (0.0, 1.0): e.args[1][0], (0.0, 0.0): e.args[2][0]}[(mm, qq)]
            ref = eval_expr(e, data)
            (g,) = torch.autograd.grad(ref.sum(), Yt)
            assert r[cr.res_reg[k]] == pytest.approx(float(ref.detach()), rel=1e-12, abs=1e-12), name
            _, d = _partials(cr, regs, k)
            got = np.zeros(Y.size)
            for i, val in d.items():
                got[i] = val
            np.testing.assert_allclose(got, g.numpy().reshape(-1), rtol=1e-11, atol=1e-12, err_msg=name)
