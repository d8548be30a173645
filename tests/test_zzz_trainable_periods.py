"""Trainable PeriodEmbedding frequencies (reference: ppsci/arch/mlp.py:95-114, ``periods={key: (period, True)}``): one
scalar w = 2 pi / period per trainable key at the end of ``model.flat``, read by the seed kernels from the parameter
buffer at every call, its gradient reduced in the first-layer adjoint kernels (fp64 per call).  Loss and gradient
against the oracle with the frequencies as inputs of its autograd graph (``_TrainablePeriods``) — the frequency entries
checked on their own as well as the whole vector — through the CPU emulation build of the real kernel sources and on
the GPU."""
import math

import numpy as np
import pytest
import sympy as sp
import torch

import ppsci
from oracle import ppsci_oracle as O
from paddlescience_b200.engine import binding as B
from tests.reparam_ref import oracle_flat

TOL = {torch.float64: (1e-11, 1e-12, 1e-11), torch.float32: (5e-6, 2e-6, 1e-5)}  # residual, loss, gradient


def _allen_cahn():
    t, x = sp.symbols("t x")
    u = sp.Function("u")(t, x)
    return {"ac": u.diff(t) - 1e-2 * u.diff(x, 2) + 5 * u ** 3 - 5 * u}


def _two_outputs():
    x, y = sp.symbols("x y")
    u, v = sp.Function("u")(x, y), sp.Function("v")(x, y)
    return {"r1": u.diff(x, 2) + u.diff(y, 2) - v * u.diff(x), "r2": u.diff(x) + v.diff(y) + sp.sin(x) * v}


def _biharmonic():
    x, y = sp.symbols("x y")
    u = sp.Function("u")(x, y)
    return {"bh": u.diff(x, 4) + 2 * u.diff(x, 2, y, 2) + u.diff(y, 4) - sp.sin(x)}


def _many_features():
    x, y, z, s, t = sp.symbols("x y z s t")
    u = sp.Function("u")(x, y, z, s, t)
    return {"r": u.diff(x, 2) + u.diff(y) + u.diff(t) * u - z}


FOURIER = {"dim": 12, "scale": 1.0}
# name -> (architecture, input keys, output keys, periods, residuals, extra constructor arguments)
CASES = {
    "allen_cahn": ("MLP", ("t", "x"), ("u",), {"x": (2.0, True)}, _allen_cahn, dict(num_layers=3, hidden_size=16)),
    "many_features": ("MLP", ("x", "y", "z", "s", "t"), ("u",), {"x": (2.0, True), "y": (1.5, False), "z": (3.0, True),
                                                                   "s": (2.5, False)}, _many_features,
                      dict(num_layers=2, hidden_size=12)),
    "fourier": ("MLP", ("x", "y"), ("u", "v"), {"x": (1.5, True)}, _two_outputs,
                dict(num_layers=2, hidden_size=12, fourier=FOURIER)),
    "modified_mlp": ("ModifiedMLP", ("x", "y"), ("u", "v"), {"x": (1.5, True)}, _two_outputs,
                     dict(num_layers=3, hidden_size=12)),
    "piratenet": ("PirateNet", ("x", "y"), ("u", "v"), {"y": (1.25, True)}, _two_outputs,
                  dict(num_blocks=1, hidden_size=12, fourier=FOURIER)),
    "biharmonic": ("MLP", ("x", "y"), ("u",), {"x": (2.0, True), "y": (3.0, True)}, _biharmonic,
                   dict(num_layers=2, hidden_size=12)),
    "mixed": ("MLP", ("x", "y"), ("u", "v"), {"x": (2.0, False), "y": (3.0, True)}, _two_outputs,
              dict(num_layers=3, hidden_size=12, weight_norm=True)),
}


def _model(name, dtype, dev):
    arch, ins, outs, periods, _, kw = CASES[name]
    ppsci.utils.misc.set_random_seed(3)
    m = getattr(ppsci.arch, arch)(ins, outs, activation="tanh", periods=periods, dtype=dtype, **kw)
    with torch.no_grad():
        m.flat.data[: m._n_eff] += 0.1 * torch.randn(m._n_eff, dtype=dtype)  # biases off zero
        m.period_freqs.mul_(1.1)  # off the initial value
    return m.to(dev)


class _TrainablePeriods:
    """The oracle network with the frequencies of the trainable keys taken from its flat vector
    ``[the oracle's own parameters | w of the trainable keys, in the order of periods]`` (the layout of ``model.flat``).

    ``OracleMLP`` embeds key k as cos(w0 x), sin(w0 x) with the fixed w0 = 2 pi / period and uses x[k] nowhere else, so
    handing it (w / w0) x[k] gives cos(w x), sin(w x); autograd then carries d/dw, and the input derivatives through x."""

    def __init__(self, om: O.OracleMLP, periods):
        self.om = om
        self.input_keys, self.output_keys = om.input_keys, om.output_keys
        self.keys = [k for k, (_, trainable) in periods.items() if trainable]
        self.n_params = om.n_params + len(self.keys)

    def __call__(self, flat, x):
        n = self.om.n_params
        xs = dict(x)
        for j, k in enumerate(self.keys):
            xs[k] = x[k] * (flat[n + j] / (2 * math.pi / float(self.om.periods[k][0])))
        return self.om(flat[:n], xs)


def _oracle_model(name):
    arch, ins, outs, periods, _, kw = CASES[name]
    hidden = [kw["hidden_size"]] * kw.get("num_layers", kw.get("num_blocks"))
    om = O.OracleMLP(ins, outs, hidden, "tanh", periods, fourier=kw.get("fourier"), modified=arch == "ModifiedMLP",
                     pirate=arch == "PirateNet")
    return _TrainablePeriods(om, periods)


def _oracle(m, om, exprs, inp, lab):
    """Oracle losses, residuals and gradient w.r.t. ``m.flat`` (the frequencies are the last entries of both vectors)."""
    flat = m.flat.data.detach().cpu().double().clone().requires_grad_(True)
    of = torch.cat([oracle_flat(m, flat), flat[m._omega_off:]])
    assert om.n_params == of.numel(), (om.n_params, of.numel())
    lo, res, go = O.train_forward_backward(om, of.detach(), exprs, {k: inp[k].cpu().double() for k in om.input_keys},
                                           {k: v.cpu().double() for k, v in lab.items()}, None, "mean")
    (g,) = torch.autograd.grad(of, flat, grad_outputs=go)
    return lo, res, g


def _batch(m, exprs, n, dev, dtype, seed=7):
    g = torch.Generator().manual_seed(seed)
    inp = {k: (torch.rand(n, 1, generator=g, dtype=torch.float64) * 2 - 1).to(dev, dtype) for k in m.input_keys}
    lab = {k: torch.zeros(n, 1, dtype=dtype, device=dev) for k in exprs}
    return inp, lab


def _train_forward(m, exprs, inp, lab):
    rect = ppsci.geometry.Rectangle((0, 0), (1, 1))  # unused by train_forward; the constraint carries the expressions
    cst = ppsci.constraint.InteriorConstraint(exprs, {k: 0 for k in exprs}, rect,
                                              {"dataset": "IterableNamedArrayDataset", "iters_per_epoch": 1, "batch_size": 4},
                                              ppsci.loss.MSELoss("mean"), name="EQ")
    m.flat.grad = None
    losses_all, _ = ppsci.utils.ExpressionSolver().train_forward((cst.output_expr,), [inp], m, {"EQ": cst}, [lab], [None])
    return {k: float(losses_all[k]) for k in exprs}


def _check_case(name, dtype, n, dev):
    exprs = CASES[name][4]()
    m = _model(name, dtype, dev)
    inp, lab = _batch(m, exprs, n, dev, dtype)
    got = _train_forward(m, exprs, inp, lab)
    lo, res, g = _oracle(m, _oracle_model(name), exprs, inp, lab)
    _, tl, tg = TOL[dtype]
    for k in exprs:
        assert abs(got[k] - float(lo[k])) <= tl * abs(float(lo[k])), (name, k, got[k], float(lo[k]))
    gg = m.flat.grad.detach().cpu().double()
    err = float((gg - g).norm() / g.norm())
    assert err <= tg, (name, err)
    om = slice(m._omega_off, m._omega_off + m._n_omega)
    assert float(g[om].abs().min()) > 0
    oerr = float((gg[om] - g[om]).norm() / g[om].norm())  # on their own: a whole-vector bar can hide a wrong scalar
    assert oerr <= tg, (name, oerr, gg[om], g[om])
    return m, oerr


def _emul(monkeypatch):
    from tests.emul.build_emul import build

    monkeypatch.setattr(B, "_default", B.Library(build()))


# ---- CPU -------------------------------------------------------------------------------------------------------------
_SEED_DCOEF_SRC = r"""
#include "jet_math.h"
extern "C" void seed_dcoef_f64(int kind, double omega, double x, double v, double* out) {
  double o[5];
  ppsci::seed_dcoef<double, 4>(kind, omega, x, v, o);
  for (int k = 0; k < 5; ++k) out[k] = o[k];
}
"""


def test_seed_dcoef_matches_sympy(tmp_path):
    """seed_dcoef (csrc/jet_math.h): d/d omega of (1/k!) d^k/dt^k g(omega (x + t v)) at t = 0, k <= 4, g = cos, sin."""
    import ctypes as C
    import os
    import subprocess

    src, so = tmp_path / "seed_dcoef.cpp", tmp_path / "libseed_dcoef.so"
    src.write_text(_SEED_DCOEF_SRC)
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "paddlescience_b200", "csrc")
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", str(src), "-I" + csrc, "-shared", "-fPIC", "-o", str(so)],
                   check=True)
    fn = C.CDLL(str(so)).seed_dcoef_f64
    fn.argtypes = [C.c_int, C.c_double, C.c_double, C.c_double, C.POINTER(C.c_double)]
    w, x, v, t = sp.symbols("w x v t")
    rng = np.random.default_rng(0)
    for kind, g in ((1, sp.cos), (2, sp.sin)):
        f = g(w * (x + t * v))
        exact = [sp.lambdify((w, x, v), sp.diff(sp.diff(f, t, k).subs(t, 0) / math.factorial(k), w)) for k in range(5)]
        for _ in range(8):
            om, xv, vv = rng.uniform(0.3, 4.0), rng.uniform(-2, 2), rng.uniform(-1.5, 1.5)
            out = (C.c_double * 5)()
            fn(kind, om, xv, vv, out)
            for k in range(5):
                ref = float(exact[k](om, xv, vv))
                assert abs(out[k] - ref) <= 1e-13 * max(1.0, abs(ref)), (kind, k, out[k], ref)
    out = (C.c_double * 5)()
    fn(0, 1.3, 0.4, 0.7, out)
    assert list(out) == [0.0] * 5  # identity features have no frequency


@pytest.mark.parametrize("name,dtype", [("allen_cahn", torch.float64), ("allen_cahn", torch.float32),
                                        ("many_features", torch.float64), ("fourier", torch.float64),
                                        ("modified_mlp", torch.float64), ("piratenet", torch.float64),
                                        ("biharmonic", torch.float64), ("biharmonic", torch.float32),
                                        ("mixed", torch.float64)])
def test_loss_and_gradient_through_emulated_kernels_match_oracle(monkeypatch, name, dtype):
    _emul(monkeypatch)
    _check_case(name, dtype, 40, "cpu")


def test_allen_cahn_f32_runs_on_the_vectorised_thin_layout():
    """The f32 Allen-Cahn case above exercises thin::k_first_dw_v: one first-order t and one second-order x direction is
    the compile-time layout Lay12 (jet_layout.cuh, ThinLays), and the features fit the thin first layer."""
    from paddlescience_b200.engine.compiler import compile_residuals

    m = _model("allen_cahn", torch.float32, "cpu")
    cr = compile_residuals(m.net_spec(), _allen_cahn(), with_grad=True)
    assert [d.order for d in cr.dirs] == [1, 2] and m.net_spec().widths[0] == 3 <= 8


def test_finite_difference_of_the_engine_loss_in_omega(monkeypatch):
    _emul(monkeypatch)
    exprs = _allen_cahn()
    m = _model("allen_cahn", torch.float64, "cpu")
    inp, lab = _batch(m, exprs, 40, "cpu", torch.float64)
    _train_forward(m, exprs, inp, lab)
    dl = float(m.flat.grad[m._omega_off])
    h = 1e-5
    w0 = float(m.period_freqs[0])
    ls = []
    for s in (1, -1):
        m.period_freqs[0] = w0 + s * h
        ls.append(_train_forward(m, exprs, inp, lab)["ac"])
    m.period_freqs[0] = w0
    fd = (ls[0] - ls[1]) / (2 * h)
    assert abs(fd - dl) <= 1e-6 * abs(dl), (fd, dl)


def test_adam_moves_omega_and_every_consumer_reads_it(monkeypatch):
    """Two Adam steps move w; the values-only plan (MLP.forward's) and the residual-only plan (lambdify's) then agree with
    the oracle at the UPDATED w: the kernels read it from the parameter buffer, not from the plan."""
    _emul(monkeypatch)
    exprs = _two_outputs()
    m = _model("fourier", torch.float64, "cpu")
    inp, lab = _batch(m, exprs, 24, "cpu", torch.float64)
    opt = torch.optim.Adam([m.flat], lr=1e-2)  # the fused Adam kernel runs on the GPU only; the GPU test below uses it
    w0 = m.period_freqs.clone()
    for _ in range(2):
        _train_forward(m, exprs, inp, lab)
        opt.step()
    assert float((m.period_freqs - w0).abs().min()) > 1e-3
    om = _oracle_model("fourier")
    of = torch.cat([oracle_flat(m, m.flat.data.double()), m.flat.data[m._omega_off:].double()])
    ref = om(of, {k: inp[k] for k in om.input_keys})
    jets, _ = m._plan_values().forward({k: inp[k] for k in m.input_keys}, m.engine_params(), want_jets=True,
                                       want_residuals=False)
    for j, k in enumerate(m.output_keys):
        np.testing.assert_allclose(jets[0][:, j].numpy(), ref[k].reshape(-1).numpy(), rtol=1e-12, atol=1e-12)
    from paddlescience_b200.engine.compiler import compile_residuals
    from paddlescience_b200.engine.plan import ResidualPlan

    plan = ResidualPlan(compile_residuals(m.net_spec(), exprs, with_grad=False), torch.float64)
    _, res = plan.forward({k: inp[k] for k in m.input_keys}, m.engine_params())
    _, ores, _ = O.train_forward_backward(om, of, exprs, inp, lab, want_grad=False)
    for k in exprs:
        np.testing.assert_allclose(res[k].reshape(-1).numpy(), ores[k].reshape(-1).numpy(), rtol=1e-10, atol=1e-11)


def test_state_dict_keys_and_round_trip():
    periods = {"t": (4.0, False), "x": (2.0, True), "y": (3.0, True)}
    m = ppsci.arch.MLP(("t", "x", "y"), ("u",), 2, 8, "tanh", periods=periods, dtype=torch.float64)
    n_lin = 6 * 8 + 8 + 8 * 8 + 8 + 8 + 1
    assert m.flat.numel() == n_lin + 2 and m._omega_off == n_lin
    assert torch.equal(m.period_freqs, torch.tensor([2 * math.pi / 2.0, 2 * math.pi / 3.0], dtype=torch.float64))
    assert m.net_spec().feat_omega_param == [-1, -1, 0, 0, 1, 1] and m.net_spec().n_params == m.flat.numel()
    sd = m.state_dict()
    assert [k for k in sd if k.startswith("period_emb")] == ["period_emb.freqs.1", "period_emb.freqs.2"]
    assert tuple(sd["period_emb.freqs.2"].shape) == ()
    with torch.no_grad():
        m.flat.data += 0.25
    m2 = ppsci.arch.MLP(("t", "x", "y"), ("u",), 2, 8, "tanh", periods=periods, dtype=torch.float64)
    m2.set_state_dict(m.state_dict())
    assert torch.equal(m2.flat.data, m.flat.data)
    bad = dict(m.state_dict())
    bad["period_emb.freqs.0"] = torch.tensor(1.0)  # a fixed key takes no parameter
    with pytest.raises(KeyError):
        m2.load_state_dict(bad)
    fixed = ppsci.arch.MLP(("t", "x", "y"), ("u",), 2, 8, "tanh", periods={k: (p, False) for k, (p, _) in periods.items()})
    plain = ppsci.arch.MLP(("t", "x", "y"), ("u",), 2, 8, "tanh", periods={"t": (4.0, False), "x": (2.0, False),
                                                                             "y": (3.0, False)})
    assert list(fixed.state_dict()) == list(plain.state_dict()) and not any("period" in k for k in fixed.state_dict())
    assert fixed.flat.numel() == n_lin and fixed.net_spec().n_omega == 0


def test_plan_create_validates_trainable_frequencies(monkeypatch):
    _emul(monkeypatch)
    from paddlescience_b200.engine.compiler import compile_residuals
    from paddlescience_b200.engine.plan import ResidualPlan

    m = ppsci.arch.MLP(("x", "y"), ("u",), 2, 8, "tanh", periods={"x": (2.0, True)}, dtype=torch.float64)
    net = m.net_spec()
    ok = ResidualPlan(compile_residuals(net, {}, with_grad=False), torch.float64)
    assert ok.n_params == m.flat.numel()
    for param, n_omega in (([0, 0, 1], 1), ([0, 0, -2], 1), ([0, 0, 0], 1)):  # out of range x2, identity feature
        net.feat_omega_param, net.n_omega = param, n_omega
        with pytest.raises(B.EngineError, match="feat_omega_param|cos / sin"):
            ResidualPlan(compile_residuals(net, {}, with_grad=False), torch.float64)
    net.feat_omega_param, net.n_omega = [0, 0, 0], 0  # n_omega = 0: the fixed frequencies, whatever the indices say
    assert ResidualPlan(compile_residuals(net, {}, with_grad=False), torch.float64).n_params == m.flat.numel() - 1


# ---- GPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,dtype", [("allen_cahn", torch.float64), ("allen_cahn", torch.float32),
                                        ("many_features", torch.float64), ("many_features", torch.float32),
                                        ("fourier", torch.float64), ("modified_mlp", torch.float64),
                                        ("modified_mlp", torch.float32), ("piratenet", torch.float64),
                                        ("biharmonic", torch.float64), ("biharmonic", torch.float32),
                                        ("mixed", torch.float64), ("mixed", torch.float32)])
def test_loss_and_gradient_on_gpu_match_oracle(name, dtype):
    _check_case(name, dtype, 3000, "cuda")


@pytest.mark.gpu
def test_forward_and_lambdify_read_the_updated_omega_on_gpu():
    exprs = _two_outputs()
    m = _model("modified_mlp", torch.float64, "cuda")
    inp, lab = _batch(m, exprs, 512, "cuda", torch.float64)
    opt = ppsci.optimizer.Adam(1e-2)(m)
    w0 = m.period_freqs.clone()
    for _ in range(2):
        _train_forward(m, exprs, inp, lab)
        opt.step()
        opt.clear_grad()
    assert float((m.period_freqs - w0).abs().min()) > 1e-3
    om = _oracle_model("modified_mlp")
    flat = m.flat.data.double().cpu()
    of = torch.cat([oracle_flat(m, flat), flat[m._omega_off:]])
    cpu_in = {k: v.cpu() for k, v in inp.items()}
    ref = om(of, {k: cpu_in[k] for k in om.input_keys})
    out = m({k: inp[k] for k in m.input_keys})
    for k in m.output_keys:
        np.testing.assert_allclose(out[k].cpu().reshape(-1).numpy(), ref[k].reshape(-1).numpy(), rtol=1e-11, atol=1e-12)
    _, ores, _ = O.train_forward_backward(om, of, exprs, cpu_in, {k: v.cpu() for k, v in lab.items()}, want_grad=False)
    for k, e in exprs.items():
        r = ppsci.lambdify(e, m)(inp)
        np.testing.assert_allclose(r.cpu().reshape(-1).numpy(), ores[k].reshape(-1).numpy(), rtol=1e-9, atol=1e-10)


def _solver_run(to_static, iters):
    ppsci.utils.misc.set_random_seed(11)
    model = ppsci.arch.MLP(("x", "y"), ("u",), 3, 32, "tanh", periods={"x": (2.0, True)})
    rect = ppsci.geometry.Rectangle((-1, 0), (1, 1))
    x, y = sp.symbols("x y")
    u = sp.Function("u")(x, y)
    ac = {"ac": u.diff(y) - 1e-2 * u.diff(x, 2) + 5 * u ** 3 - 5 * u}  # Allen-Cahn with y as the time axis
    pde = ppsci.constraint.InteriorConstraint(ac, {"ac": 0}, rect,
                                              {"dataset": "IterableNamedArrayDataset", "iters_per_epoch": iters, "batch_size": 1024},
                                              ppsci.loss.MSELoss("mean"), name="EQ")
    opt = ppsci.optimizer.Adam(1e-2)(model)
    p0 = model.flat.detach().cpu().double().clone()
    solver = ppsci.solver.Solver(model, {"EQ": pde}, None, opt, None, epochs=1, iters_per_epoch=iters, to_static=to_static,
                                 log_freq=5)
    solver.train()
    return model.flat.detach().cpu().double(), p0, solver


@pytest.mark.gpu
def test_to_static_graph_replay_trains_omega_like_the_eager_loop():
    iters = 5  # two eager warm-up iterations, then three replays of the captured graph
    pe, p0, _ = _solver_run(False, iters)
    pg, _, sg = _solver_run(True, iters)
    assert sg._graph_step is not None and sg._graph_step.replays == iters - 2
    dw = abs(float(pe[-1] - p0[-1]))  # w is the last entry of flat
    assert dw > 1e-3
    assert abs(float(pg[-1] - pe[-1])) <= 1e-4 * dw
    assert float((pg - pe).norm()) <= 1e-4 * float((pe - p0).norm())
