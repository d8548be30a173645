"""Unsteady 2-D lid-driven cavity at Re = 10 (the reference's examples/ldc/ldc2d_unsteady_Re10.py and
conf/ldc2d_unsteady_Re10.yaml) on the H100-native engine.

An MLP on (t, x, y) -> (u, v, p), 9 x 50 tanh, trained on NavierStokes(nu=0.01, rho=1, dim=2, time=True) over the
square [-0.05, 0.05]^2 and the 16 timestamps linspace(0, 1.5, 16).  Six constraints, as in the reference, all with
MSELoss("sum"): the residuals on 99^2 evenly spaced points at each of the 15 times after t0 (weights 1e-4), the four
walls at those times (lid u = 1, the others u = v = 0), and the initial condition u = v = 0 on 99^2 points at t0.
Cosine learning rate 1e-3 with 5 % linear warm-up, 20,000 iterations, and the residual validator on every timestamp,
t0 included (``with_initial=True``).  The reference's VTU visualiser is left out.

The time derivative of the residuals makes the jet layout (t: 1, x: 2, y: 2); the thin first and last layers run on
its compile-time kernels, the 50-wide hidden layers on the CUDA-core tiles.

    python examples/ldc/ldc2d_unsteady_Re10.py [--epochs 20000] [--small] [--output_dir ./output_ldc2d_unsteady_Re10]
"""
import argparse
import copy
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import ppsci  # noqa: E402

CFG = {
    "seed": 42, "NU": 0.01, "RHO": 1.0, "NTIME_ALL": 16,
    "NPOINT_PDE": 99**2, "NPOINT_TOP": 101, "NPOINT_DOWN": 101, "NPOINT_LEFT": 99, "NPOINT_RIGHT": 99,
    "NPOINT_IC": 99**2,
    "MODEL": {"input_keys": ("t", "x", "y"), "output_keys": ("u", "v", "p"), "num_layers": 9, "hidden_size": 50,
              "activation": "tanh"},
    "TRAIN": {"epochs": 20000, "iters_per_epoch": 1, "eval_during_train": True, "eval_freq": 200, "learning_rate": 1e-3,
              "weight": {"pde": {"continuity": 1e-4, "momentum_x": 1e-4, "momentum_y": 1e-4}}},
    "EVAL": {"batch_size": 8192},
}
# wiring check: 4 timestamps, a 9 x 9 grid, a 2 x 16 network, two iterations
SMALL = {"NTIME_ALL": 4, "NPOINT_PDE": 81, "NPOINT_TOP": 11, "NPOINT_DOWN": 11, "NPOINT_LEFT": 9, "NPOINT_RIGHT": 9,
         "NPOINT_IC": 81, "MODEL": {"num_layers": 2, "hidden_size": 16},
         "TRAIN": {"epochs": 2, "eval_during_train": False}, "EVAL": {"batch_size": 128}}


def merged(base, over):
    out = copy.deepcopy(base)
    for k, v in over.items():
        out[k] = merged(out[k], v) if isinstance(v, dict) and isinstance(out.get(k), dict) else v
    return out


def build(cfg, output_dir=None):
    """Model, equation, geometry, the six constraints, the residual validator and the Solver."""
    ppsci.utils.misc.set_random_seed(cfg["seed"])
    model = ppsci.arch.MLP(**cfg["MODEL"])
    equation = {"NavierStokes": ppsci.equation.NavierStokes(cfg["NU"], cfg["RHO"], 2, True)}
    timestamps = np.linspace(0.0, 1.5, cfg["NTIME_ALL"], endpoint=True)  # t0 included
    geom = {"time_rect": ppsci.geometry.TimeXGeometry(ppsci.geometry.TimeDomain(0.0, 1.5, timestamps=timestamps),
                                                      ppsci.geometry.Rectangle((-0.05, -0.05), (0.05, 0.05)))}
    tr = cfg["TRAIN"]
    loader = {"dataset": "IterableNamedArrayDataset", "iters_per_epoch": tr["iters_per_epoch"]}
    ntime = cfg["NTIME_ALL"] - 1  # the PDE and the walls use t1..tn, the initial condition t0
    uv = {"u": lambda out: out["u"], "v": lambda out: out["v"]}
    pde = ppsci.constraint.InteriorConstraint(
        equation["NavierStokes"].equations, {"continuity": 0, "momentum_x": 0, "momentum_y": 0}, geom["time_rect"],
        {**loader, "batch_size": cfg["NPOINT_PDE"] * ntime}, ppsci.loss.MSELoss("sum"), evenly=True,
        weight_dict=tr["weight"]["pde"], name="EQ")
    walls = {  # name: (points per time, label of u, criteria)
        "BC_top": (cfg["NPOINT_TOP"], 1, lambda t, x, y: np.isclose(y, 0.05)),
        "BC_down": (cfg["NPOINT_DOWN"], 0, lambda t, x, y: np.isclose(y, -0.05)),
        "BC_left": (cfg["NPOINT_LEFT"], 0, lambda t, x, y: np.isclose(x, -0.05)),
        "BC_right": (cfg["NPOINT_RIGHT"], 0, lambda t, x, y: np.isclose(x, 0.05)),
    }
    constraint = {pde.name: pde}
    for name, (npoint, u_label, criteria) in walls.items():
        constraint[name] = ppsci.constraint.BoundaryConstraint(
            uv, {"u": u_label, "v": 0}, geom["time_rect"], {**loader, "batch_size": npoint * ntime},
            ppsci.loss.MSELoss("sum"), criteria=criteria, name=name)
    ic = ppsci.constraint.InitialConstraint(
        uv, {"u": 0, "v": 0}, geom["time_rect"], {**loader, "batch_size": cfg["NPOINT_IC"]}, ppsci.loss.MSELoss("sum"),
        evenly=True, name="IC")
    constraint[ic.name] = ic
    lr_scheduler = ppsci.optimizer.lr_scheduler.Cosine(
        tr["epochs"], tr["iters_per_epoch"], tr["learning_rate"], warmup_epoch=int(0.05 * tr["epochs"]))()
    optimizer = ppsci.optimizer.Adam(lr_scheduler)(model)
    residual_validator = ppsci.validate.GeometryValidator(
        equation["NavierStokes"].equations, {"momentum_x": 0, "continuity": 0, "momentum_y": 0}, geom["time_rect"],
        {"dataset": "NamedArrayDataset", "total_size": cfg["NPOINT_PDE"] * cfg["NTIME_ALL"],
         "batch_size": cfg["EVAL"]["batch_size"], "sampler": {"name": "BatchSampler"}},
        ppsci.loss.MSELoss("sum"), evenly=True, metric={"MSE": ppsci.metric.MSE()}, with_initial=True, name="Residual")
    validator = {residual_validator.name: residual_validator}
    solver = ppsci.solver.Solver(
        model, constraint, output_dir, optimizer, lr_scheduler, tr["epochs"], tr["iters_per_epoch"],
        eval_during_train=tr["eval_during_train"], eval_freq=tr["eval_freq"], equation=equation, geom=geom,
        validator=validator, log_freq=1000)
    return solver, model, equation, geom, constraint


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=None)
    ap.add_argument("--small", action="store_true", help="tiny configuration, two iterations (wiring check)")
    ap.add_argument("--output_dir", default="./output_ldc2d_unsteady_Re10")
    args = ap.parse_args()
    cfg = merged(CFG, SMALL) if args.small else CFG
    if args.epochs is not None:
        cfg = merged(cfg, {"TRAIN": {"epochs": args.epochs}})
    solver, model, equation, geom, constraint = build(cfg, args.output_dir)
    tic = time.perf_counter()
    solver.train()
    train_s = time.perf_counter() - tic
    metric, metric_dict = solver.eval()
    result = {"epochs": cfg["TRAIN"]["epochs"], "train_wall_s": train_s, "final_loss": solver.last_loss,
              "residual_mse": metric_dict["MSE"],
              "points_per_step": sum(len(c.data_loader.loader.input["t"]) for c in constraint.values())}
    os.makedirs(args.output_dir, exist_ok=True)
    with open(os.path.join(args.output_dir, "result.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
