"""HEDeepONets: two branch nets, three outputs and an (x, t) trunk trained through the operator jet head
(``k_deeponet_jet_head`` with a second branch factor and n_out = 3), with the HeatExchanger equations.

Oracle: ``O.train_forward_backward`` over ``OracleHEDeepONets`` (tests/he_deeponet_ref.py) (autograd supplies the x and t derivatives).  CPU: the
emulation build of the same kernel sources, fp64.  GPU: the example's shapes in fp32, small shapes in fp64, and Solver
steps on the example's small configuration."""
import os
import sys
import types

import numpy as np
import pytest
import sympy as sp
import torch

import ppsci
from oracle import ppsci_oracle as O
from tests.he_deeponet_ref import OracleHEDeepONets
from tests.test_zzzz_pi_deeponet import _check, _effective, _emul

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = (("qm_h",), ("qm_c",), ("x", "t"), ("T_h", "T_c", "T_w"))
T_HIN, T_CIN, T_WIN = 10.0, 1.0, 5.5


def _model(dtype, feats, hb, ht, act="tanh", seed=5, heat_num_loc=1, **options):
    ppsci.utils.misc.set_random_seed(seed)
    model = ppsci.arch.HEDeepONets(*KEYS, heat_num_loc, 1, feats, None, None, tuple(hb), tuple(ht), branch_activation=act,
                                   trunk_activation=act, dtype=dtype, **options)
    with torch.no_grad():
        model.flat.data += 0.05 * torch.randn_like(model.flat.data)
    return model


def _oracle(model, hb, ht, act):
    m = model
    return OracleHEDeepONets(*KEYS, m._branch_locs[0], m._branch_locs[1], m.num_features, hb, ht, act, act,
                               effective=lambda flat, j, p: _effective(m, flat, m._subnets[j]))


def _data(n, seed=11, heat_num_loc=1):
    rng = np.random.RandomState(seed)
    return {"x": rng.rand(n, 1), "t": 2 * rng.rand(n, 1), "qm_h": 0.2 + 1.8 * rng.rand(n, heat_num_loc),
            "qm_c": 0.2 + 1.8 * rng.rand(n, 1), "w": rng.rand(n, 1) + 0.5, "lab": rng.randn(n, 1)}


def _equation():
    return ppsci.equation.HeatExchanger(1.0, 0.7, 1.0, 1.3, 2.0, 1.5)


def _mixed(d, jac):  # second order with a mixed partial: directions x:2, t:2 and x + t:2 (C = 7)
    return jac(jac(d["T_h"], d["x"]), d["t"]) + jac(jac(d["T_w"], d["x"]), d["x"]) - d["qm_c"] * d["T_c"]


def _run(model, hb, ht, exprs, oracle_exprs, data, device, dtype, labels, weights=None, calls=1):
    """Our fused call through ExpressionSolver.train_forward and the oracle on the same inputs."""
    t = lambda a: torch.as_tensor(a, dtype=dtype, device=device)  # noqa: E731
    n = len(data["x"])
    inputs = {k: t(data[k]) for k in ("x", "t", "qm_h", "qm_c")}
    lab = {k: (t(data[v]) if isinstance(v, str) else t(np.full((n, 1), v))) for k, v in labels.items()}
    wts = {k: t(data[v]) for k, v in (weights or {}).items()}
    cst = types.SimpleNamespace(loss=ppsci.loss.MSELoss("mean"), output_expr=exprs)
    fh = ppsci.utils.ExpressionSolver()
    for _ in range(calls):
        losses_all, losses_cst = fh.train_forward((exprs,), [inputs], model, {"c": cst}, [lab], [wts or None])
    cpu = {k: v.detach().cpu().double() for k, v in inputs.items()}
    o_losses, o_res, o_grad = O.train_forward_backward(
        _oracle(model, hb, ht, model.trunk_activation), model.flat.detach().cpu().double(), oracle_exprs, cpu,
        {k: v.cpu().double() for k, v in lab.items()}, {k: v.cpu().double() for k, v in wts.items()} or None)
    return losses_all, losses_cst, o_losses, o_res, o_grad


def _boundary_exprs():
    """The example's supervised constraints as it writes them: left, right (label key T_h, expression on T_c), initial."""
    return [{"T_h": lambda out: out["T_h"] - T_HIN}, {"T_h": lambda out: out["T_c"] - T_CIN},
            {"T_h": lambda out: out["T_h"] - T_HIN, "T_c": lambda out: out["T_c"] - T_CIN,
             "T_w": lambda out: out["T_w"] - T_WIN}]


def _jac_both(fn):
    return (lambda d: fn(d, ppsci.autodiff.jacobian)), (lambda d: fn(d, O.jacobian))


# ---------------------------------------------------------------------------------------------------------------------
def test_heat_exchanger_residuals_through_emulated_kernels_match_oracle(monkeypatch):
    """The three HeatExchanger residuals (qm_h / qm_c read as aux columns), per-slot weights."""
    _emul(monkeypatch)
    hb, ht = [10, 10], [9, 9]
    model = _model(torch.float64, 6, hb, ht)
    eqs = _equation().equations
    labels = {k: 0.0 for k in eqs}
    labels["wall"] = "lab"
    losses_all, losses_cst, o_losses, _, o_grad = _run(model, hb, ht, eqs, eqs, _data(41), "cpu", torch.float64, labels,
                                                       weights={"heat_boundary": "w", "wall": "w"})
    _check(model, losses_all, o_losses, o_grad)
    total = sum(float(v) for v in o_losses.values())
    assert abs(float(losses_cst["c"]) - total) <= 1e-12 * abs(total)


@pytest.mark.parametrize("which", [0, 1, 2])
def test_supervised_constraints_as_the_example_writes_them(monkeypatch, which):
    """No derivatives: a values-only head (n_dir = 0); the right boundary trains T_c - T_cin under the label key T_h."""
    _emul(monkeypatch)
    hb, ht = [8, 8], [8]
    model = _model(torch.float64, 5, hb, ht, act="sin")
    exprs = _boundary_exprs()[which]
    losses_all, _, o_losses, _, o_grad = _run(model, hb, ht, exprs, exprs, _data(23), "cpu", torch.float64,
                                              {k: 0.0 for k in exprs}, weights={k: "w" for k in exprs})
    _check(model, losses_all, o_losses, o_grad)


def test_second_order_mixed_partial_through_emulated_kernels(monkeypatch):
    _emul(monkeypatch)
    hb, ht = [8, 8], [10, 10]
    model = _model(torch.float64, 4, hb, ht)
    ours, theirs = _jac_both(_mixed)
    losses_all, _, o_losses, _, o_grad = _run(model, hb, ht, {"res": ours}, {"res": theirs}, _data(31), "cpu",
                                              torch.float64, {"res": "lab"})
    _check(model, losses_all, o_losses, o_grad)


def test_weight_norm_skip_multi_chunk_and_accumulation_through_emulated_kernels(monkeypatch):
    """A weight-norm branch pair and a skip-connection trunk, 2,300 pairs over 1,024-point chunks, two calls."""
    _emul(monkeypatch)
    monkeypatch.setenv("PPSCI_B200_CHUNK_POINTS", "1024")  # read when the plans are created below
    hb, ht = [8, 8, 8], [8, 8, 8]
    model = _model(torch.float64, 4, hb, ht, branch_weight_norm=True, trunk_skip_connection=True)
    eqs = _equation().equations
    losses_all, _, o_losses, _, o_grad = _run(model, hb, ht, eqs, eqs, _data(2300), "cpu", torch.float64,
                                              {k: 0.0 for k in eqs}, calls=2)
    assert model._get_plans()[0].chunk_points == 1024
    _check(model, losses_all, o_losses, o_grad, calls=2, rtol=1e-8)


def test_state_dict_round_trip_with_reference_keys():
    hb, ht = [6, 6], [5]
    model = _model(torch.float64, 3, hb, ht, trunk_weight_norm=True)
    sd = model.state_dict()
    expect = set()
    for net, n_hidden in (("heat_net", 2), ("cold_net", 2)):
        expect |= {f"{net}.linears.{i}.{p}" for i in range(n_hidden) for p in ("weight", "bias")}
        expect |= {f"{net}.last_fc.weight", f"{net}.last_fc.bias"}
    expect |= {"trunk_net.linears.0.weight_v", "trunk_net.linears.0.weight_g", "trunk_net.linears.0.bias",
               "trunk_net.last_fc.weight", "trunk_net.last_fc.bias", "b"}
    assert set(sd) == expect
    assert tuple(sd["b"].shape) == (3,) and tuple(sd["heat_net.linears.0.weight"].shape) == (1, 6)
    assert tuple(sd["trunk_net.linears.0.weight_v"].shape) == (2, 5) and tuple(sd["cold_net.last_fc.weight"].shape) == (6, 9)
    other = _model(torch.float64, 3, hb, ht, seed=9, trunk_weight_norm=True)
    assert not torch.equal(other.state_dict()["b"], sd["b"])
    other.load_state_dict(sd)
    back = other.state_dict()
    assert all(torch.equal(back[k], v) for k, v in sd.items())


def test_eval_forward_residuals_and_validator_metrics_match_oracle(monkeypatch):
    """Residuals and the example's validators through eval_forward, including the right boundary's
    ``"T_h": out["T_c"] - T_cin``, which must not be taken for the output T_h."""
    _emul(monkeypatch)
    hb, ht = [8, 8], [8, 8]
    model = _model(torch.float64, 5, hb, ht)
    n = 27
    data = _data(n)
    inputs = {k: torch.as_tensor(data[k]) for k in ("x", "t", "qm_h", "qm_c")}
    oracle = _oracle(model, hb, ht, "tanh")
    monkeypatch.setattr(model, "forward", lambda x: oracle(model.flat.detach(), x))  # values: no CPU path for forward
    fh = ppsci.utils.ExpressionSolver()
    eqs = _equation().equations
    cases = [eqs] + _boundary_exprs() + [{"T_w": lambda out: out["T_w"]}]
    for exprs in cases:
        labels = {k: torch.zeros(n, 1, dtype=torch.float64) for k in exprs}
        validator = types.SimpleNamespace(loss=ppsci.loss.MSELoss("mean"))
        out, losses = fh.eval_forward(exprs, inputs, model, validator, labels, None)
        _, o_res, _ = O.train_forward_backward(oracle, model.flat.detach().double(), exprs, inputs, labels, want_grad=False)
        for k in exprs:
            np.testing.assert_allclose(out[k].numpy(), o_res[k].numpy(), rtol=1e-11, atol=1e-12)
            mse = float((o_res[k] ** 2).mean())
            assert abs(float(losses[k]) - mse) <= 1e-11 * mse, (k, float(losses[k]), mse)
    right = fh.eval_forward(cases[2], inputs, model, None, None, None)[0]["T_h"]
    np.testing.assert_allclose(right.numpy(), (oracle(model.flat.detach(), inputs)["T_c"] - T_CIN).numpy(), rtol=1e-11)


def test_deeponet_eval_forward_computes_an_expression_named_like_its_output(monkeypatch):
    """DeepONet: ``"G": out["G"] - 1`` used to come back as G itself (skipped by its name); ``"G": out["G"]`` still
    passes the output through."""
    from tests.test_zzzz_pi_deeponet import _OracleOperator, _data as don_data, _model as don_model

    _emul(monkeypatch)
    hidden = [8, 8]
    model = don_model(torch.float64, 4, 6, hidden)
    data = don_data(19, 4)
    inputs = {k: torch.as_tensor(data[k]) for k in ("u", "y")}
    g = _OracleOperator(model, hidden, "tanh")(model.flat.detach(), inputs)["G"]
    monkeypatch.setattr(model, "forward", lambda x: {"G": g.clone()})
    fh = ppsci.utils.ExpressionSolver()
    out, _ = fh.eval_forward({"G": lambda d: d["G"] - 1.0}, inputs, model, None, None, None)
    np.testing.assert_allclose(out["G"].numpy(), (g - 1.0).numpy(), rtol=1e-11, atol=1e-13)
    out, _ = fh.eval_forward({"G": lambda d: d["G"]}, inputs, model, None, None, None)
    assert torch.equal(out["G"], g)


def test_refusals(monkeypatch):
    _emul(monkeypatch)
    model = _model(torch.float64, 3, [6], [6])
    data = _data(9)
    fh = ppsci.utils.ExpressionSolver()
    inputs = {k: torch.as_tensor(data[k]) for k in ("x", "t", "qm_h", "qm_c")}

    def call(expr, loss=None, m=None, inp=None):
        cst = types.SimpleNamespace(loss=loss or ppsci.loss.MSELoss(), output_expr={"res": expr})
        return fh.train_forward((cst.output_expr,), [inp or inputs], m or model, {"c": cst},
                                [{"res": torch.zeros(9, 1, dtype=torch.float64)}], [None])

    with pytest.raises(NotImplementedError, match="branch input 'qm_h'"):
        call(lambda d: ppsci.autodiff.jacobian(d["T_h"], d["qm_h"]))
    wide = _model(torch.float64, 3, [6], [6], heat_num_loc=2)
    wide_inputs = dict(inputs, qm_h=torch.as_tensor(_data(9, heat_num_loc=2)["qm_h"]))
    with pytest.raises(NotImplementedError, match="branch input 'qm_h'"):
        call(lambda d: d["T_h"] / d["qm_h"], m=wide, inp=wide_inputs)

    class L1Loss(ppsci.loss.MSELoss):  # any loss other than MSELoss
        pass

    with pytest.raises(NotImplementedError, match="only MSELoss"):
        call(lambda d: d["T_h"], L1Loss())
    with pytest.raises(NotImplementedError, match="per-term"):
        cst = types.SimpleNamespace(loss=ppsci.loss.MSELoss(), output_expr={"res": lambda d: d["T_h"]})
        fh.train_forward((cst.output_expr,), [inputs], model, {"c": cst}, [{"res": torch.zeros(9, 1)}], [None], per_key_grads=True)
    nu = ppsci.equation.PDE().create_parameter(1.0)
    with pytest.raises(NotImplementedError, match="learnable"):
        call(sp.Function("T_w")(sp.Symbol("x"), sp.Symbol("t")) - sp.Symbol(nu.name))
    model.register_output_transform(lambda x, y: y)
    with pytest.raises(NotImplementedError, match="transform"):
        call(lambda d: d["T_h"])
    with pytest.raises(NotImplementedError, match="stan"):
        _model(torch.float64, 3, [6], [6], act="stan")
    with pytest.raises(ValueError, match="three outputs"):
        ppsci.arch.HEDeepONets(("qm_h",), ("qm_c",), ("x", "t"), ("T_h", "T_c"), 1, 1, 3, 1, 1, 4, 4)


def _example():
    sys.path.insert(0, os.path.join(ROOT, "examples", "heat_exchanger"))
    try:
        import heat_exchanger as ex
    finally:
        sys.path.pop(0)
    return ex


def test_example_small_trains_two_iterations(monkeypatch):
    _emul(monkeypatch)
    from paddlescience_b200.optimizer.optimizer import FlatAdam

    def sgd_step(self):  # FlatAdam.step runs its fused kernel on the device only: a plain step stands in on the CPU
        with torch.no_grad():
            self.model.flat.data -= 1e-3 * self.model.flat.grad

    monkeypatch.setattr(FlatAdam, "step", sgd_step)
    res = _example().main(["--small", "--iters", "2", "--device", "cpu", "--no-reference"])
    assert len(res["loss"]) == 2 and all(np.isfinite(res["loss"]))


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_example_shapes_fp32_on_gpu_match_oracle():
    """9 x 256 swish branches, a 6 x 128 swish trunk, F = 100, 4,096 pairs: the HeatExchanger residuals."""
    hb, ht = [256] * 9, [128] * 6
    model = _model(torch.float32, 100, hb, ht, act="swish").to("cuda")
    eqs = _equation().equations
    data = _data(4096)
    losses_all, _, o_losses, o_res, o_grad = _run(model, hb, ht, eqs, eqs, data, "cuda", torch.float32,
                                                  {k: 0.0 for k in eqs}, weights={"wall": "w"})
    inputs = {k: torch.as_tensor(data[k], dtype=torch.float32, device="cuda") for k in ("x", "t", "qm_h", "qm_c")}
    res = model.evaluate_expressions(eqs, inputs)
    for k in eqs:
        assert float((res[k].cpu().double() - o_res[k]).norm() / o_res[k].norm()) <= 1e-5, k
        assert abs(float(losses_all[k]) - float(o_losses[k])) <= 2e-5 * abs(float(o_losses[k])), k
    got = model.flat.grad.detach().cpu().double()
    assert float((got - o_grad).norm() / o_grad.norm()) <= 5e-5


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["equation", "mixed"])
def test_small_shapes_fp64_on_gpu_match_oracle(case):
    hb, ht = [16, 16], [12, 12]
    model = _model(torch.float64, 8, hb, ht).to("cuda")
    if case == "equation":
        ours = theirs = _equation().equations
    else:
        o, t_ = _jac_both(_mixed)
        ours, theirs = {"res": o}, {"res": t_}
    data = _data(777)
    _, _, o_losses, o_res, o_grad = _run(model, hb, ht, ours, theirs, data, "cuda", torch.float64, {k: 0.0 for k in ours})
    inputs = {k: torch.as_tensor(data[k], device="cuda") for k in ("x", "t", "qm_h", "qm_c")}
    res = model.evaluate_expressions(ours, inputs)
    for k in ours:
        assert float((res[k].cpu() - o_res[k]).norm() / o_res[k].norm()) <= 1e-11, k
    got = model.flat.grad.detach().cpu()
    assert float((got - o_grad).norm() / o_grad.norm()) <= 1e-11


@pytest.mark.gpu
def test_example_solver_steps_on_gpu(tmp_path):
    """20 Adam steps of ppsci.solver.Solver on the example's small configuration: the loss goes down and the
    validators return finite metrics."""
    ex = _example()
    cfg = {**ex.CFG, **ex.SMALL}
    model, constraint, validator = ex.build(cfg, "cuda")
    fh = ppsci.utils.ExpressionSolver()
    data = ex.full_batches(constraint, "cuda")

    def loss():
        losses, _ = fh.train_forward(tuple(c.output_expr for c in constraint.values()), [d[0] for d in data], model,
                                     constraint, [d[1] for d in data], [d[2] for d in data])
        model.flat.grad.zero_()
        return float(sum(losses.values()))

    before = loss()
    solver = ppsci.solver.Solver(model, constraint, str(tmp_path), ppsci.optimizer.Adam(cfg["lr"])(model), epochs=20,
                                 iters_per_epoch=1, validator=validator, log_freq=5)
    solver.train()
    after = loss()
    assert np.isfinite(before) and np.isfinite(after) and after < before, (before, after)
    _, metrics = solver.eval()
    assert metrics and all(np.isfinite(float(v)) for m in metrics.values() for v in m.values()), metrics
