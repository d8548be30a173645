"""End-to-end training steps through the public API on an H100 (Solver.train: fused loss + weight-gradient call per
constraint -> optimizer) against the same optimizer driven by the oracle's loss / gradient in fp64.

Reference loops: ppsci/solver/train.py:58-213 (Adam), :216-319 (L-BFGS closure)."""
import numpy as np
import pytest
import sympy as sp
import torch

import ppsci
from oracle import ppsci_oracle as O

pytestmark = pytest.mark.gpu


def _problem(opt_factory, iters):
    ppsci.utils.misc.set_random_seed(11)
    model = ppsci.arch.MLP(("x", "y"), ("u",), 3, 20, "tanh")
    eq = ppsci.equation.Laplace(2)
    rect = ppsci.geometry.Rectangle((0, 0), (1, 1))
    cfg = {"dataset": "IterableNamedArrayDataset", "iters_per_epoch": 1}
    pde = ppsci.constraint.InteriorConstraint(eq.equations, {"laplace": 0}, rect, {**cfg, "batch_size": 512},
                                              ppsci.loss.MSELoss("mean"), name="EQ")
    bc = ppsci.constraint.BoundaryConstraint({"u": lambda out: out["u"]}, {"u": lambda d: d["x"] ** 2 - d["y"] ** 2}, rect,
                                             {**cfg, "batch_size": 128}, ppsci.loss.MSELoss("mean"), name="BC")
    params0 = model.flat.detach().cpu().double().clone()
    solver = ppsci.solver.Solver(model, {"EQ": pde, "BC": bc}, None, opt_factory(model), epochs=1, iters_per_epoch=iters,
                                 equation={"lap": eq})
    return model, solver, pde, bc, params0


def _oracle_loss_grad(om, p, pde, bc):
    x, y = sp.symbols("x y")
    tot, grad = 0.0, torch.zeros_like(p)
    for cst, exprs in ((pde, O.laplace_expr(2)), (bc, {"u": sp.Function("u")(x, y)})):
        ds = cst.data_loader.loader
        inp = {k: v.detach().cpu().double() for k, v in ds.input.items() if k in ("x", "y")}
        lab = {k: v.detach().cpu().double() for k, v in ds.label.items()}
        losses, _, g = O.train_forward_backward(om, p, exprs, inp, lab, None, "mean", None)
        tot = tot + sum(float(v) for v in losses.values())
        grad = grad + g
    return tot, grad


def test_solver_train_adam_matches_oracle_adam():
    model, solver, pde, bc, params0 = _problem(lambda m: ppsci.optimizer.Adam(1e-3)(m), 5)
    solver.train()
    om = O.OracleMLP(("x", "y"), ("u",), [20, 20, 20], "tanh")
    p = params0.clone().requires_grad_(True)
    opt = torch.optim.Adam([p], lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
    for _ in range(5):
        _, g = _oracle_loss_grad(om, p.detach(), pde, bc)
        p.grad = g
        opt.step()
    got = model.flat.detach().cpu().double()
    step = (p.detach() - params0).norm()
    assert float((got - p.detach()).norm() / step) <= 2e-3  # fp32 engine vs fp64 oracle over 5 Adam steps
    assert float(step) > 0


def test_solver_train_lbfgs_decreases_loss_like_oracle_lbfgs():
    kw = dict(learning_rate=1.0, max_iter=4, history_size=10, line_search_fn="strong_wolfe")
    model, solver, pde, bc, params0 = _problem(lambda m: ppsci.optimizer.LBFGS(**kw)(m), 3)
    om = O.OracleMLP(("x", "y"), ("u",), [20, 20, 20], "tanh")
    loss0, _ = _oracle_loss_grad(om, params0, pde, bc)
    solver.train()
    p = params0.clone().requires_grad_(True)
    opt = torch.optim.LBFGS([p], lr=1.0, max_iter=4, history_size=10, line_search_fn="strong_wolfe")

    def closure():
        loss, g = _oracle_loss_grad(om, p.detach(), pde, bc)
        p.grad = g
        return torch.tensor(loss, dtype=torch.float64)

    for _ in range(3):
        opt.step(closure)
    loss_engine, _ = _oracle_loss_grad(om, model.flat.detach().cpu().double(), pde, bc)
    loss_oracle, _ = _oracle_loss_grad(om, p.detach(), pde, bc)
    assert loss_engine < 0.5 * loss0, (loss0, loss_engine)
    # same algorithm, fp32 vs fp64 loss / gradient: the two trajectories reach the same loss level
    assert abs(np.log10(loss_engine) - np.log10(loss_oracle)) < 0.5, (loss_engine, loss_oracle)


def test_batched_constraints_equal_the_loop_on_gpu():
    """Three constraints sharing the MLP through ONE native call (BatchedConstraints) == the reference's loop over
    constraints (expression.py:89-129), on the real kernels."""
    import ppsci as _p
    from tests.test_batching import _problem

    outs = []
    for batched in (True, False):
        model, csts = _problem(torch.float32)
        model = model.to("cuda")
        fh = _p.utils.ExpressionSolver()
        fh.batch_constraints = batched
        loaders = [c.data_loader.loader for c in csts.values()]
        dev = lambda d: None if d is None else {k: v.to("cuda", torch.float32) for k, v in d.items()}  # noqa: E731
        ins, labs = [dev(ld.input) for ld in loaders], [dev(ld.label) for ld in loaders]
        ws = [dev(ld.weight) if getattr(ld, "weight", None) else None for ld in loaders]
        la, lc = fh.train_forward(tuple(c.output_expr for c in csts.values()), ins, model, csts, labs, ws)
        outs.append(({k: float(v) for k, v in la.items()}, {k: float(v) for k, v in lc.items()}, model.flat.grad.detach().cpu().double()))
    for k in outs[1][0]:
        assert outs[0][0][k] == pytest.approx(outs[1][0][k], rel=2e-6)
    for k in outs[1][1]:
        assert outs[0][1][k] == pytest.approx(outs[1][1][k], rel=2e-6)
    assert float((outs[0][2] - outs[1][2]).norm() / outs[1][2].norm()) <= 1e-5


def test_run_check_trains_and_evaluates():
    """ppsci.utils.run_check (reference ppsci/utils/checker.py:34-117): two epochs of N-S + one evaluation."""
    assert ppsci.utils.run_check() is True


def _train_params(to_static, iters, sched=True, dataset="IterableNamedArrayDataset"):
    ppsci.utils.misc.set_random_seed(11)
    model = ppsci.arch.MLP(("x", "y"), ("u",), 3, 20, "tanh")
    eq = ppsci.equation.Laplace(2)
    rect = ppsci.geometry.Rectangle((0, 0), (1, 1))
    cfg = {"dataset": dataset, "iters_per_epoch": iters}
    if dataset == "NamedArrayDataset":
        cfg["sampler"] = {"name": "BatchSampler", "shuffle": True, "drop_last": True}
    pde = ppsci.constraint.InteriorConstraint(eq.equations, {"laplace": 0}, rect, {**cfg, "batch_size": 512},
                                              ppsci.loss.MSELoss("mean"), name="EQ")
    bc = ppsci.constraint.BoundaryConstraint({"u": lambda out: out["u"]}, {"u": lambda d: d["x"] ** 2 - d["y"] ** 2}, rect,
                                             {**cfg, "batch_size": 128}, ppsci.loss.MSELoss("mean"), name="BC")
    lr = ppsci.optimizer.lr_scheduler.ExponentialDecay(1, iters, 1e-3, 0.5, 4, by_epoch=False)() if sched else 1e-3
    opt = ppsci.optimizer.Adam(lr)(model)
    p0 = model.flat.detach().cpu().double().clone()
    solver = ppsci.solver.Solver(model, {"EQ": pde, "BC": bc}, None, opt, lr if sched else None, epochs=1, iters_per_epoch=iters,
                                 equation={"lap": eq}, to_static=to_static, log_freq=5)
    solver.train()
    return model.flat.detach().cpu().double(), p0, solver


def test_to_static_replays_the_iteration_as_a_cuda_graph():
    """Solver(to_static=True): two eager iterations, one capture, then one graph launch per iteration (scheduler-driven
    learning rate and Adam bias corrections read from device memory) == the eager loop."""
    iters = 14
    pe, p0, _ = _train_params(False, iters)
    pg, _, sg = _train_params(True, iters)
    assert sg._graph_step is not None and sg._graph_step.replays == iters - 2
    step = float((pe - p0).norm())
    assert step > 0
    assert float((pg - pe).norm()) / step <= 1e-4  # same kernels; float atomics order differs between runs
    assert sg.optimizer.t == iters
    assert np.isfinite(sg.last_loss)


def test_to_static_copies_fresh_batches_into_the_graph():
    """Batches that change every iteration (a shuffled epoch over a fixed point set) reach the replayed graph."""
    iters = 4
    pe, p0, _ = _train_params(False, iters, sched=False, dataset="NamedArrayDataset")
    pg, _, sg = _train_params(True, iters, sched=False, dataset="NamedArrayDataset")
    assert sg._graph_step is not None and sg._graph_step.replays == iters - 2
    step = float((pe - p0).norm())
    assert float((pg - pe).norm()) / step <= 1e-4
