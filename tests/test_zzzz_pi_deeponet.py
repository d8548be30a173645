"""Physics-informed DeepONet: constraints whose residuals differentiate G(u)(y) with respect to the trunk coordinate y,
trained through the trunk's Taylor jets and ``k_deeponet_jet_head``.

Oracle: ``O.train_forward_backward`` over a wrapper that presents ``O.OracleDeepONet`` as an ``OracleMLP``-style callable
(autograd supplies dG/dy, d2G/dy2, ...).  CPU: the emulation build of the same kernel sources, fp64.  GPU: the cfg5 shapes
in fp32 and small shapes in fp64, and a few Solver steps on the example."""
import os
import sys
import types

import numpy as np
import pytest
import sympy as sp
import torch

import ppsci
from oracle import ppsci_oracle as O
from paddlescience_b200.engine import binding as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _effective(model, raw, r):
    """The sub-network reparametrisation restated (weight norm on the hidden layers, doubled even hidden layers >= 2)."""
    sub = raw[r.lo: r.lo + r.n]
    parts = []
    for i, (a, b) in enumerate(r.shapes):
        w = sub[r.w_off[i]: r.w_off[i] + a * b].view(a, b)
        bias = sub[r.b_off[i]: r.b_off[i] + b]
        if r.weight_norm and i < len(r.shapes) - 1:
            g = raw[r.g_off[i]: r.g_off[i] + b]
            w = g * w / torch.sqrt((w * w).sum(dim=0, keepdim=True))
        if i in r.skip_layers:
            w, bias = 2 * w, 2 * bias
        parts += [w.reshape(-1), bias]
    return torch.cat(parts)


class _OracleOperator:
    """``O.OracleDeepONet`` as an OracleMLP-style callable ``(flat, inputs) -> {"G": [N, 1]}`` over the model's flat buffer."""

    def __init__(self, model, hidden, act):
        self.model = model
        self.od = O.OracleDeepONet(model.num_loc, model.num_features, hidden, hidden, trunk_activation=act)
        self.input_keys = ("u", "y")
        self.output_keys = ("G",)

    def __call__(self, raw, x):
        m = self.model
        pb, pt = _effective(m, raw, m._rb), _effective(m, raw, m._rt)
        return {"G": self.od(pb, pt, raw[m._bias_off: m._bias_off + 1], x["u"], x["y"])}


def _jac_ppsci(f, x):
    return ppsci.autodiff.jacobian(f, x)


# residuals written once over a jacobian function: the model side traces them, the oracle runs them under autograd
def _antiderivative(d, jac):
    return jac(d["G"], d["y"]) - d["u_y"]


def _nonlinear2(d, jac):
    g_y = jac(d["G"], d["y"])
    return d["G"] * g_y + jac(g_y, d["y"]) - d["f"]


def _order4(d, jac):
    g1 = jac(d["G"], d["y"])
    g4 = jac(jac(jac(g1, d["y"]), d["y"]), d["y"])
    return g4 + 0.5 * g1 * d["G"] - d["y"] * d["f"]


def _model(dtype, num_loc, feats, hidden, act="tanh", seed=3, **options):
    ppsci.utils.misc.set_random_seed(seed)
    model = ppsci.arch.DeepONet("u", "y", "G", num_loc, feats, None, None, tuple(hidden), tuple(hidden), trunk_activation=act,
                                dtype=dtype, **options)
    with torch.no_grad():
        model.flat.data += 0.05 * torch.randn_like(model.flat.data)
    return model


def _data(n, num_loc, seed=7):
    rng = np.random.RandomState(seed)
    return {"u": rng.randn(n, num_loc), "y": rng.rand(n, 1), "u_y": rng.randn(n, 1), "f": rng.randn(n, 1),
            "lab": rng.randn(n, 1), "w": rng.rand(n, 1) + 0.5, "area": rng.rand(n, 1) + 0.5}


def _run(model, hidden, fns, data, device, dtype, labels, weights=None, reduction="mean", loss_weight=None, area=False, calls=1):
    """Our fused call through ExpressionSolver.train_forward and the oracle on the same inputs; returns both."""
    t = lambda a: torch.as_tensor(a, dtype=dtype, device=device)  # noqa: E731
    inputs = {k: t(data[k]) for k in ("u", "y", "u_y", "f")}
    if area:
        inputs["area"] = t(data["area"])
    lab = {k: (t(data[v]) if isinstance(v, str) else t(np.full((len(data["y"]), 1), v))) for k, v in labels.items()}
    wts = {k: t(data[v]) for k, v in (weights or {}).items()}
    loss = ppsci.loss.MSELoss(reduction, loss_weight)
    cst = types.SimpleNamespace(loss=loss, output_expr={k: (lambda d, f=f: f(d, _jac_ppsci)) for k, f in fns.items()})
    fh = ppsci.utils.ExpressionSolver()
    for _ in range(calls):
        losses_all, losses_cst = fh.train_forward((cst.output_expr,), [inputs], model, {"PI": cst}, [lab], [wts or None])
    od = _OracleOperator(model, hidden, model.trunk_activation)
    cpu = {k: v.detach().cpu().double() for k, v in inputs.items()}
    ow = {k: v.detach().cpu().double() for k, v in wts.items()}
    if area:
        ow = {k: (ow[k] if k in ow else 1.0) * cpu["area"] for k in labels}
    o_losses, o_res, o_grad = O.train_forward_backward(
        od, model.flat.detach().cpu().double(), {k: (lambda d, f=f: f(d, O.jacobian)) for k, f in fns.items()},
        {k: v for k, v in cpu.items() if k != "area"}, {k: v.cpu().double() for k, v in lab.items()}, ow or None,
        reduction, loss_weight)
    return losses_all, losses_cst, o_losses, o_res, o_grad


def _emul(monkeypatch):
    from tests.emul.build_emul import build

    monkeypatch.setattr(B, "_default", B.Library(build()))


def _check(model, losses_all, o_losses, o_grad, calls=1, rtol=1e-9):
    for k, v in o_losses.items():
        assert abs(float(losses_all[k]) - float(v)) <= 1e-12 * abs(float(v)), (k, float(losses_all[k]), float(v))
    got = model.flat.grad.detach().cpu().double()
    np.testing.assert_allclose(got.numpy(), calls * o_grad.numpy(), rtol=rtol, atol=1e-13 * float(o_grad.abs().max()))


CASES = {
    "order1": dict(fns={"res": _antiderivative}, labels={"res": 0.0}),
    "order2_nonlinear": dict(fns={"res": _nonlinear2}, labels={"res": 0.0}, weights={"res": "w"}),
    "order4": dict(fns={"res": _order4}, labels={"res": "lab"}),
    "sin_sum": dict(fns={"res": _nonlinear2}, labels={"res": 0.0}, act="sin", reduction="sum"),
    "identity_and_residual": dict(fns={"G": lambda d, jac: d["G"], "res": _antiderivative}, labels={"G": "lab", "res": 0.0},
                                  weights={"G": "w"}, loss_weight={"G": 2.5, "res": 0.75}, area=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_pi_losses_and_gradients_through_emulated_kernels_match_oracle(monkeypatch, case):
    _emul(monkeypatch)
    c = dict(CASES[case])
    hidden = [12, 12]
    model = _model(torch.float64, 6, 9, hidden, act=c.pop("act", "tanh"))
    losses_all, losses_cst, o_losses, _, o_grad = _run(model, hidden, c.pop("fns"), _data(37, 6), "cpu", torch.float64, **c)
    _check(model, losses_all, o_losses, o_grad)
    total = sum(float(v) for v in o_losses.values())
    assert abs(float(losses_cst["PI"]) - total) <= 1e-12 * abs(total)


def test_weight_norm_skip_multi_chunk_and_accumulation_through_emulated_kernels(monkeypatch):
    """A weight-norm branch and a skip-connection trunk, 2,500 pairs over 1,024-point chunks, two calls accumulating."""
    _emul(monkeypatch)
    monkeypatch.setenv("PPSCI_B200_CHUNK_POINTS", "1024")  # read when the plans are created below
    hidden = [8, 8, 8]
    model = _model(torch.float64, 5, 7, hidden, branch_weight_norm=True, trunk_skip_connection=True)
    losses_all, _, o_losses, _, o_grad = _run(model, hidden, {"res": _nonlinear2}, _data(2500, 5), "cpu", torch.float64,
                                              labels={"res": 0.0}, weights={"res": "w"}, calls=2)
    assert model._get_plans()[0].chunk_points == 1024
    _check(model, losses_all, o_losses, o_grad, calls=2, rtol=1e-8)


def test_eval_forward_residuals_through_emulated_kernels_match_oracle(monkeypatch):
    _emul(monkeypatch)
    hidden = [10, 10]
    model = _model(torch.float64, 4, 6, hidden)
    data = _data(29, 4)
    inputs = {k: torch.as_tensor(data[k]) for k in ("u", "y", "u_y", "f")}
    monkeypatch.setattr(model, "forward", lambda x: {"G": torch.zeros(29, 1, dtype=torch.float64)})  # values: no CPU path
    fns = {"res1": _antiderivative, "res2": _nonlinear2}
    out, _ = ppsci.utils.ExpressionSolver().eval_forward({k: (lambda d, f=f: f(d, _jac_ppsci)) for k, f in fns.items()},
                                                         inputs, model, None, None, None)
    _, o_res, _ = O.train_forward_backward(_OracleOperator(model, hidden, "tanh"), model.flat.detach().double(),
                                           {k: (lambda d, f=f: f(d, O.jacobian)) for k, f in fns.items()}, inputs,
                                           {k: torch.zeros(29, 1, dtype=torch.float64) for k in fns}, want_grad=False)
    for k in fns:
        np.testing.assert_allclose(out[k].numpy(), o_res[k].numpy(), rtol=1e-11, atol=1e-13)


def test_refusals(monkeypatch):
    _emul(monkeypatch)
    model = _model(torch.float64, 4, 6, [8])
    data = _data(11, 4)
    fh = ppsci.utils.ExpressionSolver()
    inputs = {k: torch.as_tensor(data[k]) for k in ("u", "y", "u_y", "f")}

    def call(expr, loss=None):
        cst = types.SimpleNamespace(loss=loss or ppsci.loss.MSELoss(), output_expr={"res": expr})
        return fh.train_forward((cst.output_expr,), [inputs], model, {"c": cst}, [{"res": torch.zeros(11, 1, dtype=torch.float64)}],
                                [None])

    with pytest.raises(NotImplementedError, match="branch input"):
        call(lambda d: ppsci.autodiff.jacobian(d["G"], d["u"]))
    with pytest.raises(NotImplementedError, match="branch input"):
        call(lambda d: d["G"] * d["u"])
    class L1Loss(ppsci.loss.MSELoss):  # any loss other than MSELoss
        pass

    with pytest.raises(NotImplementedError, match="only MSELoss"):
        call(lambda d: ppsci.autodiff.jacobian(d["G"], d["y"]), L1Loss())
    nu = ppsci.equation.PDE().create_parameter(1.0)
    with pytest.raises(NotImplementedError, match="learnable"):
        call(sp.Derivative(sp.Function("G")(sp.Symbol("u"), sp.Symbol("y")), sp.Symbol("y")) - sp.Symbol(nu.name))
    with pytest.raises(NotImplementedError, match="per-term"):
        cst = types.SimpleNamespace(loss=ppsci.loss.MSELoss(), output_expr={"res": lambda d: d["G"]})
        fh.train_forward((cst.output_expr,), [inputs], model, {"c": cst}, [{"res": torch.zeros(11, 1)}], [None], per_key_grads=True)
    model.register_output_transform(lambda x, y: y)
    with pytest.raises(NotImplementedError, match="transform"):
        call(lambda d: ppsci.autodiff.jacobian(d["G"], d["y"]))


def test_example_small_trains_two_iterations(monkeypatch):
    _emul(monkeypatch)
    sys.path.insert(0, os.path.join(ROOT, "examples", "operator_learning"))
    try:
        import pi_deeponet_antiderivative as ex
    finally:
        sys.path.pop(0)
    from paddlescience_b200.optimizer.optimizer import FlatAdam

    def sgd_step(self):  # FlatAdam.step runs its fused kernel on the device only: a plain step stands in on the CPU
        with torch.no_grad():
            self.model.flat.data -= 1e-3 * self.model.flat.grad

    monkeypatch.setattr(FlatAdam, "step", sgd_step)
    res = ex.main(["--small", "--iters", "2", "--device", "cpu"])
    assert len(res["loss"]) == 2 and all(np.isfinite(res["loss"]))
    assert np.isfinite(res["l2_rel"])


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fns", [{"res": _antiderivative}, {"res": _nonlinear2}])
def test_cfg5_shapes_fp32_on_gpu_match_oracle(fns):
    hidden = [128, 128, 128]
    model = _model(torch.float32, 100, 128, hidden).to("cuda")
    data = _data(4096, 100)
    losses_all, _, o_losses, o_res, o_grad = _run(model, hidden, fns, data, "cuda", torch.float32, labels={"res": 0.0},
                                                  weights={"res": "w"})
    inputs = {k: torch.as_tensor(data[k], dtype=torch.float32, device="cuda") for k in ("u", "y", "u_y", "f")}
    res = model.evaluate_expressions({"res": lambda d: fns["res"](d, _jac_ppsci)}, inputs, ["u_y", "f"])["res"]
    assert float((res.cpu().double() - o_res["res"]).norm() / o_res["res"].norm()) <= 1e-5
    assert abs(float(losses_all["res"]) - float(o_losses["res"])) <= 2e-5 * abs(float(o_losses["res"]))
    got = model.flat.grad.detach().cpu().double()
    assert float((got - o_grad).norm() / o_grad.norm()) <= 5e-5


@pytest.mark.gpu
@pytest.mark.parametrize("fn", [_antiderivative, _order4])
def test_small_shapes_fp64_on_gpu_match_oracle(fn):
    hidden = [16, 16]
    model = _model(torch.float64, 8, 10, hidden).to("cuda")
    data = _data(777, 8)
    _, _, o_losses, o_res, o_grad = _run(model, hidden, {"res": fn}, data, "cuda", torch.float64, labels={"res": 0.0})
    inputs = {k: torch.as_tensor(data[k], device="cuda") for k in ("u", "y", "u_y", "f")}
    res = model.evaluate_expressions({"res": lambda d: fn(d, _jac_ppsci)}, inputs, ["u_y", "f"])["res"]
    assert float((res.cpu() - o_res["res"]).norm() / o_res["res"].norm()) <= 1e-11
    got = model.flat.grad.detach().cpu()
    assert float((got - o_grad).norm() / o_grad.norm()) <= 1e-11


@pytest.mark.gpu
def test_example_solver_steps_on_gpu(tmp_path):
    """A few Adam steps of ppsci.solver.Solver on the example's constraints: the loss stays finite and goes down."""
    sys.path.insert(0, os.path.join(ROOT, "examples", "operator_learning"))
    try:
        import pi_deeponet_antiderivative as ex
    finally:
        sys.path.pop(0)
    cfg = {**ex.CFG, **ex.SMALL}
    model, constraint, validator, _ = ex.build(cfg, "cuda")
    data = ex.batches(constraint, "cuda")
    fh = ppsci.utils.ExpressionSolver()

    def loss():
        losses, _ = fh.train_forward(tuple(c.output_expr for c in constraint.values()), [d[0] for d in data], model, constraint,
                                     [d[1] for d in data], [d[2] for d in data])
        model.flat.grad.zero_()
        return float(sum(losses.values()))

    before = loss()
    solver = ppsci.solver.Solver(model, constraint, str(tmp_path), ppsci.optimizer.Adam(learning_rate=3e-3)(model), epochs=20,
                                 iters_per_epoch=1, validator={validator.name: validator}, log_freq=5)
    solver.train()
    after = loss()
    assert np.isfinite(before) and np.isfinite(after) and after < before, (before, after)
    metric, _ = solver.eval()
    assert np.isfinite(float(metric))
