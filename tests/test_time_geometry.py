"""CPU tests of the time-dependent problem set-up: TimeDomain / TimeXGeometry sampling (seeded counts, time-major order,
t0 left out of the interior and boundary and given by sample_initial_interior, criteria(t, x, y)), InitialConstraint,
GeometryValidator(..., with_initial=True), the unsteady Navier-Stokes plan through the emulated kernels against the
fp64 oracle, the batched call of the unsteady cavity's six constraints against the loop over them, and the example's
small configuration.  The docstring answers of the reference's timedomain.py are pinned in tests/golden/."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

import ppsci
from oracle import ppsci_oracle as O
from paddlescience_b200.engine import binding as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "time_geometry_known_answers.json")))


def _cavity(ntime_all=4):
    ts = np.linspace(0.0, 1.5, ntime_all, endpoint=True)
    return ppsci.geometry.TimeXGeometry(ppsci.geometry.TimeDomain(0.0, 1.5, timestamps=ts),
                                        ppsci.geometry.Rectangle((-0.05, -0.05), (0.05, 0.05)))


def _unit(**kw):
    return ppsci.geometry.TimeXGeometry(ppsci.geometry.TimeDomain(0, 1, **kw), ppsci.geometry.Rectangle((0, 0), (1, 1)))


def test_docstring_known_answers():
    on = ppsci.geometry.TimeDomain(0, 1).on_initial([0, 0.01, 0.126, 0.2, 0.3])
    assert on.tolist() == GOLDEN["TimeDomain(0, 1).on_initial([0, 0.01, 0.126, 0.2, 0.3])"]
    g = _unit(time_step=0.001)
    np.random.seed(0)
    for name, fn in (("uniform_points", g.uniform_points), ("random_points", g.random_points),
                     ("random_boundary_points", g.random_boundary_points)):
        assert list(fn(1000).shape) == GOLDEN[f"TimeXGeometry(TimeDomain(0, 1, 0.001), Rectangle((0, 0), (1, 1))).{name}(1000).shape"]
    g = _unit()
    for name in ("uniform_boundary_points", "uniform_initial_points"):
        assert list(getattr(g, name)(1000).shape) == GOLDEN[f"TimeXGeometry(TimeDomain(0, 1), Rectangle((0, 0), (1, 1))).{name}(1000).shape"]
    d = g.sample_initial_interior(1000)
    assert {k: list(v.shape) for k, v in d.items()} == \
        GOLDEN["TimeXGeometry(TimeDomain(0, 1), Rectangle((0, 0), (1, 1))).sample_initial_interior(1000)"]
    assert g.dim_keys == ("t", "x", "y") and g.ndim == 3


def test_interior_even_time_major_without_t0():
    g = _cavity()
    d = g.sample_interior(81 * 3, evenly=True)
    assert {k: v.shape for k, v in d.items()} == {k: (243, 1) for k in ("t", "x", "y")}
    ts = np.linspace(0.0, 1.5, 4).astype("float32")
    assert np.array_equal(d["t"].ravel(), np.repeat(ts[1:], 81))  # time-major, t0 left out
    grid = ppsci.geometry.Rectangle((-0.05, -0.05), (0.05, 0.05)).uniform_points(81)
    for i in range(3):
        assert np.array_equal(np.hstack((d["x"], d["y"]))[81 * i: 81 * (i + 1)], grid)


def test_heat_exchanger_grid_is_the_time_geometry():
    """examples/heat_exchanger builds TimeXGeometry(...).sample_interior(NPOINT * NTIME, evenly=True) with numpy."""
    spec = importlib.util.spec_from_file_location("hx", os.path.join(ROOT, "examples", "heat_exchanger", "heat_exchanger.py"))
    hx = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(hx)
    cfg = {**hx.CFG, "NTIME": 5, "NPOINT": 11}
    g = ppsci.geometry.TimeXGeometry(
        ppsci.geometry.TimeDomain(0.0, 2, timestamps=np.linspace(0.0, 2, cfg["NTIME"] + 1, endpoint=True)),
        ppsci.geometry.Interval(0, cfg["DL"]))
    d, ref = g.sample_interior(cfg["NPOINT"] * cfg["NTIME"], evenly=True), hx.grid(cfg)
    assert np.array_equal(d["t"], ref["t"]) and np.array_equal(d["x"], ref["x"])


def test_random_interior_seeded_order():
    """Space points drawn once (numpy's global stream, the reference's order) and repeated for each t after t0."""
    g = _cavity()
    np.random.seed(42)
    d = g.sample_interior(30)
    np.random.seed(42)
    x = np.random.random((10, 2)).astype("float32") * np.float32(0.1) + np.float32(-0.05)
    assert np.array_equal(d["t"].ravel(), np.repeat(np.linspace(0, 1.5, 4).astype("float32")[1:], 10))
    for i in range(3):
        assert np.allclose(np.hstack((d["x"], d["y"]))[10 * i: 10 * (i + 1)], x, atol=1e-7)


def test_boundary_criteria_takes_t_first():
    g = _cavity()
    seen = []

    def top(t, x, y):
        seen.append(t is None)
        return np.isclose(y, 0.05)

    np.random.seed(1)
    b = g.sample_boundary(11 * 3, criteria=top)
    assert b["t"].shape == (33, 1) and np.allclose(b["y"], 0.05)
    assert np.array_equal(b["t"].ravel(), np.repeat(np.linspace(0, 1.5, 4).astype("float32")[1:], 11))
    assert np.array_equal(b["normal_y"], np.ones_like(b["y"])) and np.array_equal(b["normal_t"], b["t"])
    assert True in seen and False in seen  # space points filtered with t = None, then (t, x, y) filtered again


def test_initial_points_and_on_initial():
    g = _cavity()
    i = g.sample_initial_interior(81, evenly=True)
    assert set(i) == {"t", "x", "y", "sdf"} and np.all(i["t"] == 0)
    pts = np.hstack((i["t"], i["x"], i["y"]))
    assert g.on_initial(pts).all()
    assert not g.on_initial(np.hstack((np.full_like(i["t"], 0.5), i["x"], i["y"]))).any()
    left = g.sample_initial_interior(9, criteria=lambda t, x, y: np.isclose(t, 0) & (x < 0))
    assert np.all(left["x"] < 0)
    with pytest.raises(ValueError):
        ppsci.geometry.TimeXGeometry(ppsci.geometry.TimeDomain(0, 1), ppsci.geometry.Rectangle((0, 0), (1, 1))).random_points(10)


def test_time_step_domain():
    g = _unit(time_step=0.25)
    assert g.timedomain.num_timestamps == 5
    assert np.allclose(np.unique(g.random_points(100)[:, 0]), [0.25, 0.5, 0.75, 1.0])
    assert np.allclose(np.unique(g.uniform_points(100, boundary=False)[:, 0]), [0.25, 0.5, 0.75, 1.0])


def _cfg(batch):
    return {"dataset": "IterableNamedArrayDataset", "iters_per_epoch": 1, "batch_size": batch}


def test_initial_constraint_and_validator_shapes():
    g = _cavity()
    ic = ppsci.constraint.InitialConstraint({"u": lambda out: out["u"]}, {"u": lambda d: d["x"] * 2}, g, _cfg(81),
                                            ppsci.loss.MSELoss("sum"), evenly=True, name="IC")
    ld = ic.data_loader.loader
    assert ld.input["t"].shape == (81, 1) and float(ld.input["t"].abs().max()) == 0
    assert torch.equal(ld.label["u"], 2 * ld.input["x"]) and ic.input_keys == ("t", "x", "y")
    eq = ppsci.equation.NavierStokes(0.01, 1.0, 2, True)
    cfg = {"dataset": "NamedArrayDataset", "total_size": 81 * 4, "batch_size": 64, "sampler": {"name": "BatchSampler"}}
    for with_initial, nts in ((True, 4), (False, 3)):
        v = ppsci.validate.GeometryValidator(eq.equations, {"momentum_x": 0, "continuity": 0, "momentum_y": 0}, g, cfg,
                                             ppsci.loss.MSELoss("sum"), evenly=True, metric={"MSE": ppsci.metric.MSE()},
                                             with_initial=with_initial, name="Residual")
        t = v.data_loader.loader.ds.input["t"].ravel()
        assert v.num_timestamps == nts and len(t) == 81 * 4 // nts * 3 + (81 if with_initial else 0)
        assert (t == 0).sum() == (81 if with_initial else 0) and np.all(np.diff(t) >= 0)
    with pytest.raises(NotImplementedError):
        ppsci.validate.GeometryValidator(eq.equations, {"continuity": 0}, _unit(), {**cfg, "total_size": 64},
                                         ppsci.loss.MSELoss("sum"), with_initial=True)


def test_unsteady_ns_layout_is_in_both_kernel_families():
    """NavierStokes(time=True) on (t, x, y) compiles to t:1, x:2, y:2; ThinLays and WgLays both list that layout."""
    from paddlescience_b200.engine.compiler import compile_residuals
    from tests.cases import make_net
    from tests.test_jet_layouts import FAMILIES, _family

    cr = compile_residuals(make_net(("t", "x", "y"), ("u", "v", "p"), [50] * 9, "tanh"),
                           O.navier_stokes_expr(0.01, 1.0, 2, True))
    assert [d.order for d in cr.dirs] == [1, 2, 2] and [d.vec for d in cr.dirs] == [(1, 0, 0), (0, 1, 0), (0, 0, 1)]
    for fam in FAMILIES.values():
        assert ((1, 2, 2), (1, 2, 4)) in [(o, b) for _, o, b in _family(fam)]


@pytest.fixture(scope="module")
def emul_lib():
    from tests.emul.build_emul import build

    return B.Library(build())


def test_unsteady_ns_plan_matches_oracle_fp64(emul_lib):
    from tests.cases import run_case

    case = dict(in_keys=("t", "x", "y"), out_keys=("u", "v", "p"), hidden=[16, 16], act="tanh",
                exprs=lambda: O.navier_stokes_expr(0.01, 1.0, 2, True), dtype=torch.float64)
    r = run_case(case, 60, library=emul_lib, device="cpu")
    assert r["loss"] <= 1e-12 and r["res"] <= 1e-11 and r["grad"] <= 1e-11, r


def _load_example():
    spec = importlib.util.spec_from_file_location("ldc_unsteady", os.path.join(ROOT, "examples", "ldc", "ldc2d_unsteady_Re10.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    return ex


def _example_losses(batched, emul_lib):
    ex = _load_example()
    cfg = ex.merged(ex.CFG, ex.SMALL)
    cfg["MODEL"]["dtype"] = torch.float64
    solver, model, equation, geom, csts = ex.build(cfg)
    fh = ppsci.utils.ExpressionSolver()
    fh.batch_constraints = batched
    loaders = [c.data_loader.loader for c in csts.values()]
    f64 = lambda d: {k: v.double() for k, v in d.items()}  # noqa: E731
    ins, labs = [f64(ld.input) for ld in loaders], [f64(ld.label) for ld in loaders]
    ws = [f64(ld.weight) if getattr(ld, "weight", None) else None for ld in loaders]
    la, lc = fh.train_forward(tuple(c.output_expr for c in csts.values()), ins, model, csts, labs, ws)
    return {k: float(v) for k, v in la.items()}, {k: float(v) for k, v in lc.items()}, model.flat.grad.clone(), fh


def test_example_constraints_batched_equal_the_loop(monkeypatch, emul_lib):
    monkeypatch.setattr(B, "_default", emul_lib)
    la_b, lc_b, g_b, fh = _example_losses(True, emul_lib)
    la_l, lc_l, g_l, _ = _example_losses(False, emul_lib)
    assert len(fh._batched) == 1
    assert set(lc_b) == {"EQ", "BC_top", "BC_down", "BC_left", "BC_right", "IC"}
    for k in la_l:
        assert la_b[k] == pytest.approx(la_l[k], rel=1e-12)
    for k in lc_l:
        assert lc_b[k] == pytest.approx(lc_l[k], rel=1e-12)
    assert float((g_b - g_l).norm() / g_l.norm()) <= 1e-12


def test_example_small_trains_two_iterations(monkeypatch, emul_lib):
    from paddlescience_b200.optimizer import optimizer as opt_mod
    from paddlescience_b200.solver import train as train_mod

    monkeypatch.setattr(B, "_default", emul_lib)

    def cpu_step(self):  # FlatAdam.step without the device guard, on the emulated library
        p = self.model.flat
        self._ensure_state()
        self.t += 1
        rc = emul_lib.lib.ppsci_b200_adam_step(B.F64 if p.dtype == torch.float64 else B.F32, p.data.data_ptr(),
                                               p.grad.data_ptr(), self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(),
                                               p.numel(), self.get_lr(), self.beta1, self.beta2, self.epsilon,
                                               self.weight_decay, self.t, self.grad_scale, None)
        assert rc == 0

    monkeypatch.setattr(opt_mod.FlatAdam, "step", cpu_step)
    ex = _load_example()
    cfg = ex.merged(ex.CFG, ex.SMALL)
    solver, model, equation, geom, csts = ex.build(cfg)
    assert list(csts) == ["EQ", "BC_top", "BC_down", "BC_left", "BC_right", "IC"]
    assert len(csts["EQ"].data_loader.loader.input["t"]) == 81 * 3 and len(csts["IC"].data_loader.loader.input["t"]) == 81
    p0 = model.flat.data.clone()
    for epoch in (1, 2):
        train_mod.train_epoch_func(solver, epoch, solver.log_freq)
    assert solver.global_step == 2 and np.isfinite(solver.last_loss)
    assert torch.isfinite(model.flat.data).all() and float((model.flat.data - p0).abs().max()) > 0
