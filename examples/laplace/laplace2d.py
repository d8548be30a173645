"""Laplace2D PINN — the reference's acceptance example (examples/laplace/laplace2d.py:20-140, BASELINE configs[0]) on the
H100-native engine.  Same script structure and the same ``ppsci`` calls; the hydra / yaml layer is replaced by the
plain dict below (the values of examples/laplace/conf/laplace2d.yaml).  Published result to reproduce
(docs/zh/examples/laplace2d.md:31): MSE.u(MSE_Metric) = 0.00002.

    python examples/laplace/laplace2d.py [--epochs 20000] [--output_dir ./output_laplace2d]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import ppsci  # noqa: E402

CFG = {
    "seed": 2024,
    "NPOINT_INTERIOR": 9801,
    "NPOINT_BC": 400,
    "DIAGONAL_COORD": {"xmin": (0.0, 0.0), "xmax": (1.0, 1.0)},
    "MODEL": {"input_keys": ("x", "y"), "output_keys": ("u",), "num_layers": 5, "hidden_size": 20},
    "TRAIN": {"epochs": 20000, "iters_per_epoch": 1, "eval_during_train": True, "eval_freq": 200, "learning_rate": 0.001},
}


def train(cfg, output_dir):
    ppsci.utils.misc.set_random_seed(cfg["seed"])
    model = ppsci.arch.MLP(**cfg["MODEL"])
    equation = {"laplace": ppsci.equation.Laplace(dim=2)}
    geom = {"rect": ppsci.geometry.Rectangle(cfg["DIAGONAL_COORD"]["xmin"], cfg["DIAGONAL_COORD"]["xmax"])}

    def u_solution_func(out):
        """ground truth for u as label data"""
        x, y = out["x"], out["y"]
        return np.cos(x) * np.cosh(y)

    train_dataloader_cfg = {"dataset": "IterableNamedArrayDataset", "iters_per_epoch": cfg["TRAIN"]["iters_per_epoch"]}
    npoint_total = cfg["NPOINT_INTERIOR"] + cfg["NPOINT_BC"]
    pde_constraint = ppsci.constraint.InteriorConstraint(
        equation["laplace"].equations, {"laplace": 0}, geom["rect"], {**train_dataloader_cfg, "batch_size": npoint_total},
        ppsci.loss.MSELoss("sum"), evenly=True, name="EQ")
    bc = ppsci.constraint.BoundaryConstraint(
        {"u": lambda out: out["u"]}, {"u": u_solution_func}, geom["rect"], {**train_dataloader_cfg, "batch_size": cfg["NPOINT_BC"]},
        ppsci.loss.MSELoss("sum"), name="BC")
    constraint = {pde_constraint.name: pde_constraint, bc.name: bc}
    optimizer = ppsci.optimizer.Adam(learning_rate=cfg["TRAIN"]["learning_rate"])(model)
    mse_metric = ppsci.validate.GeometryValidator(
        {"u": lambda out: out["u"]}, {"u": u_solution_func}, geom["rect"],
        {"dataset": "IterableNamedArrayDataset", "total_size": npoint_total}, ppsci.loss.MSELoss(), evenly=True,
        metric={"MSE": ppsci.metric.MSE()}, with_initial=True, name="MSE_Metric")
    validator = {mse_metric.name: mse_metric}
    solver = ppsci.solver.Solver(
        model, constraint, output_dir, optimizer, epochs=cfg["TRAIN"]["epochs"], iters_per_epoch=cfg["TRAIN"]["iters_per_epoch"],
        eval_during_train=cfg["TRAIN"]["eval_during_train"], eval_freq=cfg["TRAIN"]["eval_freq"], equation=equation, geom=geom,
        validator=validator, log_freq=1000, to_static=bool(cfg.get("to_static", False)))
    t0 = time.perf_counter()
    solver.train()
    train_s = time.perf_counter() - t0
    metric, metric_dict = solver.eval()
    return {"epochs": cfg["TRAIN"]["epochs"], "train_wall_s": train_s, "MSE.u(MSE_Metric)": float(metric),
            "published": 2e-5, "points_per_step": npoint_total + cfg["NPOINT_BC"],
            "steps_per_s": cfg["TRAIN"]["epochs"] * cfg["TRAIN"]["iters_per_epoch"] / train_s}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=CFG["TRAIN"]["epochs"])
    ap.add_argument("--output_dir", default="./output_laplace2d")
    ap.add_argument("--result_json", default=None)
    ap.add_argument("--to_static", action="store_true", help="replay the training iteration as a CUDA graph (the reference's to_static flag)")
    a = ap.parse_args()
    CFG["TRAIN"]["epochs"] = a.epochs
    CFG["to_static"] = a.to_static
    res = train(CFG, a.output_dir)
    print(json.dumps(res))
    if a.result_json:
        with open(a.result_json, "w") as f:
            json.dump(res, f)
