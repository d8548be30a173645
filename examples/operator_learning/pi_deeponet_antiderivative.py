"""Physics-informed DeepONet for the antiderivative operator G(u)(y) = int_0^y u(s) ds (Wang, Wang & Perdikaris 2021),
trained without solution data: the residual dG/dy - u(y) = 0 on (function, y) pairs and the initial condition
G(u, 0) = 0.  dG/dy comes from the trunk net's Taylor jets along y (``arch.DeepONet`` with a derivative in the
constraint's expression), not from autograd.

The input functions are seeded random sums of sines  u(x) = sum_k a_k sin(k pi x + phi_k)  on [0, 1], sampled at the
``num_loc`` sensors, so their antiderivatives are closed-form; an L2-relative validator compares G with them on held-out
functions.  Default shapes: the reference's examples/operator_learning/conf/deeponet.yaml (100 sensors, 40 features,
one hidden layer of 40 in both sub-networks, relu branch, relu trunk replaced by tanh: relu has no second derivative to
train through).  ``--small`` is a seconds-long configuration for tests.

    python examples/operator_learning/pi_deeponet_antiderivative.py [--iters 10000] [--small] [--device cuda]

It prints the final loss and the L2-relative error reached; ``build`` also serves ``ppsci.solver.Solver``.
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import ppsci  # noqa: E402

CFG = {
    "seed": 42, "num_loc": 100, "n_modes": 4, "n_funcs": 1000, "n_y": 100, "n_val_funcs": 100, "lr": 1e-3, "iters": 10000,
    "MODEL": dict(num_features=40, branch_num_layers=1, trunk_num_layers=1, branch_hidden_size=40, trunk_hidden_size=40,
                  branch_activation="relu", trunk_activation="tanh"),
}
SMALL = {"num_loc": 12, "n_funcs": 16, "n_y": 8, "n_val_funcs": 8,
         "MODEL": dict(num_features=8, branch_num_layers=1, trunk_num_layers=1, branch_hidden_size=8, trunk_hidden_size=8,
                       branch_activation="relu", trunk_activation="tanh")}


def functions(rng, n, n_modes):
    """Amplitudes / phases of n random sums of sines, u(x) = sum_k a_k sin(k pi x + phi_k), k = 1..n_modes."""
    return rng.randn(n, n_modes) / np.arange(1, n_modes + 1), rng.rand(n, n_modes) * 2 * math.pi


def u_of(a, phi, x):
    k = np.arange(1, a.shape[1] + 1) * math.pi
    return (a[:, None, :] * np.sin(k * x[..., None] + phi[:, None, :])).sum(-1)


def antiderivative(a, phi, y):
    k = np.arange(1, a.shape[1] + 1) * math.pi
    return (a[:, None, :] / k * (np.cos(phi[:, None, :]) - np.cos(k * y[..., None] + phi[:, None, :]))).sum(-1)


def pairs(rng, cfg, n_funcs):
    """(sensor values u, coordinate y, u(y), G(u)(y)) of n_funcs functions at n_y random coordinates each."""
    a, phi = functions(rng, n_funcs, cfg["n_modes"])
    sensors = np.linspace(0.0, 1.0, cfg["num_loc"])
    u = u_of(a, phi, sensors[None, :])                                  # [F, num_loc]
    y = rng.rand(n_funcs, cfg["n_y"])                                   # [F, n_y]
    u_y = u_of(a, phi, y)
    g = antiderivative(a, phi, y)
    rep = lambda m: np.repeat(m, cfg["n_y"], axis=0).astype(np.float32)  # noqa: E731
    col = lambda m: m.reshape(-1, 1).astype(np.float32)  # noqa: E731
    return {"u": rep(u), "y": col(y), "u_y": col(u_y)}, col(g), u.astype(np.float32)


def build(cfg, device):
    """Model, the two constraints, the L2-relative validator and its held-out (inputs, G) arrays."""
    ppsci.utils.misc.set_random_seed(cfg["seed"])
    rng = np.random.RandomState(cfg["seed"])
    model = ppsci.arch.DeepONet("u", "y", "G", cfg["num_loc"], **cfg["MODEL"]).to(device)
    inp, _, u_sens = pairs(rng, cfg, cfg["n_funcs"])
    n = len(inp["y"])
    res = ppsci.constraint.SupervisedConstraint(
        {"dataset": {"name": "IterableNamedArrayDataset", "input": inp, "label": {"res": np.zeros((n, 1), np.float32)}},
         "batch_size": n},
        ppsci.loss.MSELoss("mean"), {"res": lambda out: ppsci.autodiff.jacobian(out["G"], out["y"]) - out["u_y"]},
        name="residual")
    ic_in = {"u": u_sens, "y": np.zeros((len(u_sens), 1), np.float32)}
    ic = ppsci.constraint.SupervisedConstraint(
        {"dataset": {"name": "IterableNamedArrayDataset", "input": ic_in, "label": {"G": np.zeros((len(u_sens), 1), np.float32)}},
         "batch_size": len(u_sens)}, ppsci.loss.MSELoss("mean"), {"G": lambda out: out["G"]}, name="initial")
    val_in, val_g, _ = pairs(np.random.RandomState(cfg["seed"] + 1), cfg, cfg["n_val_funcs"])
    validator = ppsci.validate.SupervisedValidator(
        {"dataset": {"name": "NamedArrayDataset", "input": {k: val_in[k] for k in ("u", "y")}, "label": {"G": val_g}},
         "batch_size": len(val_g)},
        ppsci.loss.MSELoss("mean"), {"G": lambda out: out["G"]}, metric={"L2Rel": ppsci.metric.L2Rel()}, name="G_L2Rel")
    return model, {res.name: res, ic.name: ic}, validator, ({k: val_in[k] for k in ("u", "y")}, val_g)


def batches(constraint, device):
    """(inputs, labels, weights) of every constraint: each one's full point set as one batch, on the device."""
    to = lambda d: None if d is None else {k: torch.as_tensor(v).to(device) for k, v in d.items()}  # noqa: E731
    out = []
    for cst in constraint.values():
        ds = cst.data_loader.loader
        out.append((to(ds.input), to(ds.label), to(getattr(ds, "weight", None))))
    return out


def l2_rel(model, held_out, device):
    """L2-relative error of G on the held-out functions (read through the jet head's forward)."""
    inp, ref = held_out
    pred = model.evaluate_expressions({"G": lambda out: out["G"]}, {k: torch.as_tensor(v).to(device) for k, v in inp.items()})
    pred = pred["G"].cpu().numpy()
    return float(np.linalg.norm(pred - ref) / np.linalg.norm(ref))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=CFG["iters"])
    ap.add_argument("--small", action="store_true")
    ap.add_argument("--device", default="cuda")
    a = ap.parse_args(argv)
    cfg = {**CFG, **(SMALL if a.small else {})}
    model, constraint, _, held_out = build(cfg, a.device)
    data = batches(constraint, a.device)
    optimizer = ppsci.optimizer.Adam(learning_rate=cfg["lr"])(model)
    fh = ppsci.utils.ExpressionSolver()
    history = []
    t0 = time.perf_counter()
    for it in range(a.iters):  # Solver.train's step (solver/train.py) spelled out: one fused call per constraint
        losses, _ = fh.train_forward(tuple(c.output_expr for c in constraint.values()), [d[0] for d in data], model, constraint,
                                     [d[1] for d in data], [d[2] for d in data])
        optimizer.step()
        optimizer.clear_grad()
        if it % max(1, a.iters // 100) == 0 or it == a.iters - 1:
            history.append(float(sum(losses.values())))
    wall = time.perf_counter() - t0
    return {"iters": a.iters, "train_wall_s": wall, "loss": history, "l2_rel": l2_rel(model, held_out, a.device)}


if __name__ == "__main__":
    out = main()
    print(json.dumps({k: (v[-1] if k == "loss" else v) for k, v in out.items()}))
