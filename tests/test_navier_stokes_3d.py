"""CPU tests of unsteady 3-D Navier-Stokes: PointCloud (the reference's docstring answers, pinned in tests/golden/,
boundary points, translate / scale, seeded sampling and InteriorConstraint), L2RelLoss (docstring answers, and the
raise of a training constraint given it), the compiled jet layouts of NavierStokes(nu, rho, 3, True) in both key
orders and the kernel families that list them, the emulated fp64 plans against the oracle, the batched call of the
Beltrami example's three constraints against the loop over them, and the example's small configuration."""
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
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "ns3d_known_answers.json")))


def _line(n=5):
    return np.linspace(0, 2, n, dtype="float32").reshape((-1, 1))


def test_pointcloud_docstring_known_answers():
    G = ppsci.geometry.PointCloud
    got = {
        "PointCloud({x: linspace(0, 2, 5)}, (x,)).translate([1.0]).interior":
            G({"x": _line()}, ("x",)).translate(np.array([1.0])).interior,
        "PointCloud({x, y: linspace(0, 2, 5)}, (x, y)).translate([1.0, 3.0]).interior":
            G({"x": _line(), "y": _line()}, ("x", "y")).translate(np.array([1.0, 3.0])).interior,
        "PointCloud({x: linspace(0, 2, 5)}, (x,)).scale([2.0]).interior":
            G({"x": _line()}, ("x",)).scale(np.array([2.0])).interior,
        "PointCloud({x, y: linspace(0, 2, 5)}, (x, y)).scale([2.0, 0.5]).interior":
            G({"x": _line(), "y": _line()}, ("x", "y")).scale(np.array([2.0, 0.5])).interior,
        "PointCloud({x: linspace(0, 2, 5)}, (x,)).uniform_points(2)": G({"x": _line()}, ("x",)).uniform_points(2),
    }
    np.random.seed(0)
    got["seed(0); PointCloud({x: linspace(0, 2, 5)}, (x,), {x: [0, 2]}).random_boundary_points(1)"] = G(
        {"x": _line()}, ("x",), {"x": np.array([[0.0], [2.0]], dtype="float32")}).random_boundary_points(1)
    np.random.seed(0)
    got["seed(0); PointCloud({x: linspace(0, 2, 5)}, (x,)).random_points(2)"] = G({"x": _line()}, ("x",)).random_points(2)
    for k, v in got.items():
        assert v.dtype == np.float32 and v.tolist() == GOLDEN[k], k


def test_pointcloud_geometry():
    g = ppsci.geometry.PointCloud({"x": _line(), "y": 2 * _line()}, ("x", "y"))
    assert g.dim_keys == ("x", "y") and g.ndim == 2 and g.len == 5
    assert np.array_equal(g.bbox[0], [0, 0]) and np.array_equal(g.bbox[1], [2, 4])
    assert g.is_inside(np.array([[0.5, 1.0], [0.5, 1.0 + 5e-7], [0.5, 1.1]], dtype="float32")).tolist() == [True, True, False]
    with pytest.raises(ValueError):  # no boundary points given
        g.on_boundary(np.zeros((1, 2), dtype="float32"))
    with pytest.raises(ValueError):
        g.random_points(6)
    with pytest.raises(NotImplementedError):
        g.uniform_boundary_points(1)
    for op in (lambda: g | g, lambda: g - g, lambda: g & g, lambda: g.union(g), lambda: g.difference(g),
               lambda: g.intersection(g)):
        with pytest.raises(NotImplementedError):
            op()


def test_pointcloud_with_boundary_and_normals():
    """The reference tests ``if self.boundary:`` on the array, which raises for more than one boundary point."""
    bnd = {"x": np.array([[0.0], [2.0]], dtype="float32"), "y": np.array([[0.0], [4.0]], dtype="float32")}
    nrm = {"x_normal": np.array([[-1.0], [1.0]], dtype="float32"), "y_normal": np.array([[-1.0], [1.0]], dtype="float32")}
    g = ppsci.geometry.PointCloud({"x": _line(), "y": 2 * _line()}, ("x", "y"), bnd, nrm)
    assert g.on_boundary(np.array([[0, 0], [2, 4], [1, 2]], dtype="float32")).tolist() == [True, True, False]
    np.random.seed(3)
    b = g.random_boundary_points(2)
    np.random.seed(3)
    assert np.array_equal(b, g.boundary[np.random.choice(2, size=2, replace=False)])
    with pytest.raises(ValueError):
        g.random_boundary_points(3)
    g.translate(np.array([1.0, -1.0]))
    assert g.boundary.tolist() == [[1, -1], [3, 3]] and g.interior[:, 1].tolist() == [-1, 0, 1, 2, 3]
    g.scale(np.array([2.0, 0.5]))
    assert g.boundary.tolist() == [[2, -0.5], [6, 1.5]] and g.normal.tolist() == [[-2, -0.5], [2, 0.5]]
    assert g.interior[:, 0].tolist() == [2, 3, 4, 5, 6]
    with pytest.raises(ValueError):  # normals without boundary points, or of another shape
        ppsci.geometry.PointCloud({"x": _line()}, ("x",), None, {"x_normal": _line()})
    with pytest.raises(ValueError):
        ppsci.geometry.PointCloud({"x": _line()}, ("x",), {"x": _line()}, {"x_normal": _line(3)})


def test_pointcloud_interior_constraint():
    """sample_interior draws n of the points without replacement (numpy's global stream) and adds no sdf column."""
    rng = np.random.RandomState(7)
    pts = {k: rng.rand(40, 1).astype("float32") for k in ("x", "y", "z", "t")}
    g = ppsci.geometry.PointCloud(pts, ("x", "y", "z", "t"))
    np.random.seed(11)
    d = g.sample_interior(25)
    np.random.seed(11)
    idx = np.random.choice(40, size=25, replace=False)
    assert set(d) == {"x", "y", "z", "t"}
    for k in d:
        assert np.array_equal(d[k], pts[k][idx])
    eq = ppsci.equation.NavierStokes(1.0, 1.0, 3, True)
    np.random.seed(11)
    c = ppsci.constraint.InteriorConstraint(
        eq.equations, {"continuity": 0, "momentum_x": 0, "momentum_y": 0, "momentum_z": 0}, g,
        {"dataset": {"name": "IterableNamedArrayDataset"}, "batch_size": 25, "iters_per_epoch": 1},
        ppsci.loss.MSELoss("mean"), name="EQ")
    inp = c.data_loader.loader.input
    assert c.input_keys == ("x", "y", "z", "t") and set(inp) == {"x", "y", "z", "t"}
    assert np.array_equal(np.asarray(inp["t"]), pts["t"][idx])
    assert np.array_equal(g.uniform_points(3), np.hstack([pts[k][:3] for k in ("x", "y", "z", "t")]))


def test_l2rel_loss_docstring_known_answers():
    out = {"u": torch.tensor([[0.5, 0.9], [1.1, -1.3]]), "v": torch.tensor([[0.5, 0.9], [1.1, -1.3]])}
    lab = {"u": torch.tensor([[-1.8, 1.0], [-0.2, 2.5]]), "v": torch.tensor([[0.1, 0.1], [0.1, 0.1]])}
    w = {"u": 0.8, "v": 0.2}
    for key, loss in (("L2RelLoss(weight={u: 0.8, v: 0.2})", ppsci.loss.L2RelLoss(weight=w)),
                      ("L2RelLoss(reduction=sum, weight={u: 0.8, v: 0.2})", ppsci.loss.L2RelLoss("sum", w))):
        got = loss(out, lab)
        for k, v in GOLDEN[key].items():
            assert float(got[k]) == pytest.approx(v, rel=1e-6), (key, k)
    # [N, 1] columns: one relative error per point; a per-point weight column and a float weight
    x, y = torch.tensor([[1.0], [3.0]]), torch.tensor([[2.0], [4.0]])
    got = ppsci.loss.L2RelLoss(weight=2.0)({"u": x}, {"u": y}, {"u": torch.tensor([[1.0], [4.0]])})
    assert float(got["u"]) == pytest.approx(2.0 * (0.5 + 4 * 0.25) / 2)
    with pytest.raises(ValueError):
        ppsci.loss.L2RelLoss("none")


def _cfg(batch):
    return {"dataset": "IterableNamedArrayDataset", "iters_per_epoch": 1, "batch_size": batch}


def test_l2rel_loss_in_a_training_constraint_raises():
    model = ppsci.arch.MLP(("x", "y", "z", "t"), ("u", "v", "w", "p"), 2, 8, "tanh")
    rng = np.random.RandomState(0)
    g = ppsci.geometry.PointCloud({k: rng.rand(16, 1).astype("float32") for k in ("x", "y", "z", "t")},
                                  ("x", "y", "z", "t"))
    eq = ppsci.equation.NavierStokes(1.0, 1.0, 3, True)
    c = ppsci.constraint.InteriorConstraint(eq.equations, {"continuity": 0}, g, _cfg(16), ppsci.loss.L2RelLoss(),
                                            name="EQ")
    inp, lab, _ = next(iter(c.data_loader.loader))
    for batched in (True, False):
        fh = ppsci.utils.ExpressionSolver()
        fh.batch_constraints = batched
        with pytest.raises(NotImplementedError, match="L2RelLoss"):
            fh.train_forward((c.output_expr,), [inp], model, {"EQ": c}, [lab], [None])


@pytest.mark.parametrize("keys,orders,bases,families", [
    (("x", "y", "z", "t"), [2, 2, 2, 1], (1, 3, 5, 7), {"ThinLays", "WgLays"}),
    (("t", "x", "y", "z"), [1, 2, 2, 2], (1, 2, 4, 6), {"WgLays"})])
def test_ns3d_layouts_kernel_families(keys, orders, bases, families):
    """NavierStokes(nu, rho, 3, True) compiles to its four directions in input order, C = 8.  The (x, y, z, t) layout is
    in ThinLays and WgLays; the (t, x, y, z) one in WgLays only (its plans keep the generic thin kernels)."""
    from paddlescience_b200.engine.compiler import compile_residuals
    from tests.cases import make_net
    from tests.test_jet_layouts import FAMILIES, _family

    cr = compile_residuals(make_net(keys, ("u", "v", "w", "p"), [100] * 10, "tanh"),
                           O.navier_stokes_expr(1.0, 1.0, 3, True))
    assert [d.order for d in cr.dirs] == orders and cr.channels == 8
    assert [d.vec for d in cr.dirs] == [tuple(int(i == j) for i in range(4)) for j in range(4)]
    for name, fam in FAMILIES.items():
        listed = (tuple(orders), bases) in [(o, b) for _, o, b in _family(fam)]
        assert listed == (name in families), name


@pytest.fixture(scope="module")
def emul_lib():
    from tests.emul.build_emul import build

    return B.Library(build())


@pytest.mark.parametrize("keys", [("x", "y", "z", "t"), ("t", "x", "y", "z")])
def test_beltrami_shaped_plan_matches_oracle_fp64(emul_lib, keys):
    from tests.cases import run_case

    case = dict(in_keys=keys, out_keys=("u", "v", "w", "p"), hidden=[12, 12, 12], act="tanh",
                exprs=lambda: O.navier_stokes_expr(1.0, 1.0, 3, True), dtype=torch.float64,
                ranges={k: (0, 1) if k == "t" else (-1, 1) for k in keys})
    r = run_case(case, 40, library=emul_lib, device="cpu")
    assert r["loss"] <= 1e-12 and r["res"] <= 1e-11 and r["grad"] <= 1e-11, r


def _load_example():
    spec = importlib.util.spec_from_file_location("beltrami3d", os.path.join(ROOT, "examples", "nsfnet", "beltrami3d.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    return ex


def test_example_data_follow_the_reference():
    """Point counts of the full configuration, the exact solution on the data, and the schedule's bounds."""
    ex = _load_example()
    np.random.seed(1234)
    bound, init, interior, test = ex.generate_data(70000)
    assert len(bound["x"]) == 59400 and len(init["x"]) == 29791 and len(interior["x"]) == 70000 and len(test["x"]) == 1000
    assert all(v.dtype == np.float32 for d in (bound, init, interior) for v in d.values())
    assert set(np.unique(interior["t"]).round(6)) == set(np.linspace(0, 1, 11).astype("float32").round(6))
    on_face = np.isclose(np.abs(np.hstack([bound[k] for k in "xyz"])), 1).any(axis=1)
    assert on_face.all() and np.all(init["t"] == 0)
    u, v, w, p = ex.analytic_solution(test["x"], test["y"], test["z"], test["t"])
    assert np.array_equal(u, test["u"]) and np.array_equal(p, test["p"])
    assert ex.schedule(ex.CFG["TRAIN"]) == ([5000, 10000, 60000, 110000], [1e-3, 1e-4, 1e-5, 1e-6, 1e-7])
    assert ex.schedule({**ex.CFG["TRAIN"], "epochs": 11000})[0] == [500, 1000, 6000, 11000]
    # Beltrami flow: divergence free (central differences on the exact solution)
    h, X = 1e-4, np.array([0.3, -0.2, 0.5, 0.4])
    div = sum((ex.analytic_solution(*(X + h * e))[i] - ex.analytic_solution(*(X - h * e))[i]) / (2 * h)
              for i, e in enumerate(np.eye(4)[:3]))
    assert abs(div) < 1e-6


def _batches(csts, f64=True):
    ins, labs, ws = [], [], []
    cast = (lambda t: torch.as_tensor(t).double()) if f64 else torch.as_tensor  # noqa: E731
    for c in csts.values():
        inp, lab, w = next(iter(c.data_loader.loader))
        ins.append({k: cast(v) for k, v in inp.items()})
        labs.append({k: cast(v) for k, v in lab.items()})
        ws.append({k: cast(v) for k, v in w.items()} if w else None)
    return ins, labs, ws


def _example_losses(batched):
    ex = _load_example()
    cfg = ex.merged(ex.CFG, ex.SMALL)
    cfg["MODEL"]["dtype"] = torch.float64
    solver, model, equation, geom, csts, test = ex.build(cfg)
    fh = ppsci.utils.ExpressionSolver()
    fh.batch_constraints = batched
    ins, labs, ws = _batches(csts)
    la, lc = fh.train_forward(tuple(c.output_expr for c in csts.values()), ins, model, csts, labs, ws)
    return {k: float(v) for k, v in la.items()}, {k: float(v) for k, v in lc.items()}, model.flat.grad.clone(), fh


def test_example_constraints_batched_equal_the_loop(monkeypatch, emul_lib):
    monkeypatch.setattr(B, "_default", emul_lib)
    la_b, lc_b, g_b, fh = _example_losses(True)
    la_l, lc_l, g_l, _ = _example_losses(False)
    assert len(fh._batched) == 1
    assert set(lc_b) == {"EQ", "Sup_b", "Sup_0"}
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
    solver, model, equation, geom, csts, test = ex.build(cfg)
    assert list(csts) == ["EQ", "Sup_b", "Sup_0"]
    assert isinstance(geom["points"], ppsci.geometry.PointCloud) and geom["points"].len == 300
    assert [type(c.loss).__name__ for c in csts.values()] == ["MSELoss"] * 3
    assert csts["Sup_b"].loss.weight == 100.0 and csts["Sup_0"].loss.weight == 100.0
    assert type(solver.validator["Residual"].loss).__name__ == "L2RelLoss"
    p0 = model.flat.data.clone()
    for epoch in (1, 2):
        train_mod.train_epoch_func(solver, epoch, solver.log_freq)
    assert solver.global_step == 2 and np.isfinite(solver.last_loss)
    assert torch.isfinite(model.flat.data).all() and float((model.flat.data - p0).abs().max()) > 0
