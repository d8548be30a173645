"""3-D unsteady Beltrami flow (the reference's examples/nsfnet/VP_NSFNet3.py and conf/VP_NSFNet3.yaml; NSFNet, Jin
et al. 2021, section 3.3) on the H100-native engine.

An MLP on (x, y, z, t) -> (u, v, w, p), 10 x 100 tanh, trained on NavierStokes(nu=1/Re, rho=1, dim=3, time=True) with
Re = 1 over [-1, 1]^3 x [0, 1], where the Beltrami flow (a = d = 1) is the exact solution.  Three constraints, as in the
reference, each with MSELoss("mean"): the four residuals on 70,000 interior points drawn from the 31^3 x 11 grid (a
``PointCloud``), the velocity on the 59,400 boundary points of the six faces (weight alpha = 100) and at t = 0 on the
29,791 points of the grid (weight beta = 100).  The data are generated exactly as the reference does, in the same
numpy RNG order after seeding 1234.  Adam with piecewise-constant LR 1e-3 / 1e-4 / 1e-5 / 1e-6 over 5,000 + 5,000 +
50,000 + 50,000 = 110,000 iterations; ``--epochs`` shortens the schedule, scaling each piece in proportion.

Evaluation: the L2Rel validator (``loss.L2RelLoss``, metric ``L2Rel``) of u, v and w on the reference's 1,000 random
test points.  The reference also validates ``p - p.min() + p_star.min()``; that shift is a reduction over the batch,
which the engine's per-point expressions cannot express, so ``errors`` applies it in numpy to the predicted p of the
same 1,000 points after prediction and reports the L2-relative errors of u, v, w and the shifted p.

Kernels: C = 8 jet channels per point (x: 2, y: 2, z: 2, t: 1, ``Lay2221``).  The first (4 -> 100) and last (100 -> 4)
layers run on the vectorised thin kernels of that layout (100 is a multiple of 4, M = 4); the 100-wide hidden layers
stay on the CUDA-core tiles, because 100 is not a multiple of 32 (the wgmma kernels take widths that are).

    python examples/nsfnet/beltrami3d.py [--epochs 110000] [--small] [--output_dir ./output_NSFNet3]
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
    "seed": 1234, "RE": 1.0, "NTRAIN": 70000, "ALPHA": 100.0, "BETA": 100.0, "NTEST": 1000,
    "MODEL": {"input_keys": ("x", "y", "z", "t"), "output_keys": ("u", "v", "w", "p"), "num_layers": 10,
              "hidden_size": 100, "activation": "tanh"},
    "TRAIN": {"epochs": 110000, "iters_per_epoch": 1, "epoch_list": (5000, 5000, 50000, 50000),
              "lr_list": (1e-3, 1e-4, 1e-5, 1e-6, 1e-7), "eval_during_train": True, "eval_freq": 5000,
              "log_freq": 5000},
}
# wiring check: 300 interior points, every 90th boundary and initial point, a 2 x 16 network, two iterations
SMALL = {"NTRAIN": 300, "SUBSAMPLE": 90, "NTEST": 50, "MODEL": {"num_layers": 2, "hidden_size": 16},
         "TRAIN": {"epochs": 2, "eval_during_train": False, "log_freq": 1}}


def merged(base, over):
    out = copy.deepcopy(base)
    for k, v in over.items():
        out[k] = merged(out[k], v) if isinstance(v, dict) and isinstance(out.get(k), dict) else v
    return out


def analytic_solution(x, y, z, t, a=1.0, d=1.0):
    """The Beltrami flow of Ethier and Steinman (1994): (u, v, w, p) at (x, y, z, t)."""
    u = -a * (np.exp(a * x) * np.sin(a * y + d * z) + np.exp(a * z) * np.cos(a * x + d * y)) * np.exp(-d * d * t)
    v = -a * (np.exp(a * y) * np.sin(a * z + d * x) + np.exp(a * x) * np.cos(a * y + d * z)) * np.exp(-d * d * t)
    w = -a * (np.exp(a * z) * np.sin(a * x + d * y) + np.exp(a * y) * np.cos(a * z + d * x)) * np.exp(-d * d * t)
    p = -0.5 * a * a * (np.exp(2 * a * x) + np.exp(2 * a * y) + np.exp(2 * a * z)
                        + 2 * np.sin(a * x + d * y) * np.cos(a * z + d * x) * np.exp(a * (y + z))
                        + 2 * np.sin(a * y + d * z) * np.cos(a * x + d * y) * np.exp(a * (z + x))
                        + 2 * np.sin(a * z + d * x) * np.cos(a * y + d * z) * np.exp(a * (x + y))) * np.exp(-2 * d * d * t)
    return u, v, w, p


def _col(a):
    return np.asarray(a).reshape(-1, 1).astype("float32")


def generate_data(n_train, n_test=1000):
    """Boundary, initial, interior and test data, in the reference's order of numpy draws (VP_NSFNet3.py:54-151).

    Returns dicts ``bound`` / ``init`` / ``test`` of (x, y, z, t, u, v, w[, p]) columns and ``interior`` of (x, y, z, t)."""
    x1 = np.linspace(-1, 1, 31)
    y1 = np.linspace(-1, 1, 31)
    z1 = np.linspace(-1, 1, 31)
    t1 = np.linspace(0, 1, 11)
    b0 = np.array([-1] * 900)
    b1 = np.array([1] * 900)
    xt, yt = np.tile(x1[0:30], 30), np.tile(y1[0:30], 30)
    xt1, yt1 = np.tile(x1[1:31], 30), np.tile(y1[1:31], 30)
    yr, zr = y1[0:30].repeat(30), z1[0:30].repeat(30)
    yr1, zr1 = y1[1:31].repeat(30), z1[1:31].repeat(30)
    bx = np.concatenate([b1, b0, xt1, xt, xt1, xt], 0).repeat(t1.shape[0])
    by = np.concatenate([yt, yt1, b1, b0, yr1, yr], 0).repeat(t1.shape[0])
    bz = np.concatenate([zr, zr1, zr, zr1, b1, b0], 0).repeat(t1.shape[0])
    bt = np.tile(t1, 5400)
    bu, bv, bw, _ = analytic_solution(bx, by, bz, bt)
    bound = {k: _col(v) for k, v in zip("xyztuvw", (bx, by, bz, bt, bu, bv, bw))}

    x0 = np.tile(x1, 31 * 31)
    y0 = np.tile(y1.repeat(31), 31)
    z0 = z1.repeat(31 * 31)
    t0 = np.array([0] * x0.shape[0])
    u0, v0, w0, _ = analytic_solution(x0, y0, z0, t0)
    init = {k: _col(v) for k, v in zip("xyztuvw", (x0, y0, z0, t0, u0, v0, w0))}

    xx = np.random.randint(31, size=n_train) / 15 - 1
    yy = np.random.randint(31, size=n_train) / 15 - 1
    zz = np.random.randint(31, size=n_train) / 15 - 1
    tt = np.random.randint(11, size=n_train) / 10
    interior = {k: _col(v) for k, v in zip("xyzt", (xx, yy, zz, tt))}

    xs = ((np.random.rand(n_test, 1) - 1 / 2) * 2).astype("float32")
    ys = ((np.random.rand(n_test, 1) - 1 / 2) * 2).astype("float32")
    zs = ((np.random.rand(n_test, 1) - 1 / 2) * 2).astype("float32")
    ts = (np.random.randint(11, size=(n_test, 1)) / 10).astype("float32")
    us, vs, ws, ps = analytic_solution(xs, ys, zs, ts)
    test = dict(x=xs, y=ys, z=zs, t=ts, u=us, v=vs, w=ws, p=ps)
    return bound, init, interior, test


def _array_loader(inp, lab, batch_size, iters_per_epoch):
    return {"dataset": {"name": "NamedArrayDataset", "input": inp, "label": lab}, "batch_size": batch_size,
            "iters_per_epoch": iters_per_epoch, "sampler": {"name": "BatchSampler", "drop_last": False, "shuffle": False}}


def schedule(tr):
    """Piecewise bounds (cumulative) and values; a shortened run scales each piece in proportion."""
    pieces = np.array(tr["epoch_list"], dtype=float) * tr["epochs"] / sum(tr["epoch_list"])
    bounds = [max(1, int(round(b))) for b in np.cumsum(pieces)]
    return bounds, list(tr["lr_list"])


def build(cfg, output_dir=None):
    """Model, equation, geometry, the three constraints, the L2Rel validator and the Solver; also the test data."""
    ppsci.utils.misc.set_random_seed(cfg["seed"])
    model = ppsci.arch.MLP(**cfg["MODEL"])
    bound, init, interior, test = generate_data(cfg["NTRAIN"], cfg["NTEST"])
    if cfg.get("SUBSAMPLE"):
        bound = {k: v[:: cfg["SUBSAMPLE"]] for k, v in bound.items()}
        init = {k: v[:: cfg["SUBSAMPLE"]] for k, v in init.items()}
    tr = cfg["TRAIN"]
    ipe = tr["iters_per_epoch"]
    xyzt, uvw = ("x", "y", "z", "t"), ("u", "v", "w")
    nb, n0 = len(bound["x"]), len(init["x"])  # one batch each: 59,400 and 29,791 points
    sup_b = ppsci.constraint.SupervisedConstraint(
        _array_loader({k: bound[k] for k in xyzt}, {k: bound[k] for k in uvw}, nb, ipe),
        ppsci.loss.MSELoss("mean", cfg["ALPHA"]), name="Sup_b")
    sup_0 = ppsci.constraint.SupervisedConstraint(
        _array_loader({k: init[k] for k in xyzt}, {k: init[k] for k in uvw}, n0, ipe),
        ppsci.loss.MSELoss("mean", cfg["BETA"]), name="Sup_0")
    geom = {"points": ppsci.geometry.PointCloud(interior, xyzt)}
    equation = {"NavierStokes": ppsci.equation.NavierStokes(nu=1.0 / cfg["RE"], rho=1.0, dim=3, time=True)}
    pde = ppsci.constraint.InteriorConstraint(
        equation["NavierStokes"].equations, {"continuity": 0, "momentum_x": 0, "momentum_y": 0, "momentum_z": 0},
        geom["points"], {"dataset": {"name": "IterableNamedArrayDataset"}, "batch_size": cfg["NTRAIN"],
                         "iters_per_epoch": ipe}, ppsci.loss.MSELoss("mean"), name="EQ")
    constraint = {pde.name: pde, sup_b.name: sup_b, sup_0.name: sup_0}
    n_test = len(test["x"])
    validator = ppsci.validate.SupervisedValidator(
        _array_loader({k: test[k] for k in xyzt}, {k: test[k] for k in uvw}, n_test, 1) | {"total_size": n_test},
        ppsci.loss.L2RelLoss(), output_expr={k: (lambda out, k=k: out[k]) for k in uvw},
        metric={"L2R": ppsci.metric.L2Rel()}, name="Residual")
    bounds, values = schedule(tr)
    lr_scheduler = ppsci.optimizer.lr_scheduler.Piecewise(tr["epochs"], ipe, bounds, values)()
    optimizer = ppsci.optimizer.Adam(lr_scheduler)(model)
    solver = ppsci.solver.Solver(
        model, constraint, output_dir, optimizer, lr_scheduler, tr["epochs"], ipe,
        eval_during_train=tr["eval_during_train"], eval_freq=tr["eval_freq"], equation=equation, geom=geom,
        validator={validator.name: validator}, log_freq=tr["log_freq"])
    return solver, model, equation, geom, constraint, test


def errors(solver, test):
    """L2-relative errors of u, v, w and of p shifted by ``- p.min() + p_star.min()`` on the test points (numpy)."""
    pred = solver.predict({k: test[k] for k in ("x", "y", "z", "t")}, batch_size=None, return_numpy=True)
    pred["p"] = pred["p"] - pred["p"].min() + test["p"].min()
    return {k: float(np.linalg.norm(test[k] - pred[k]) / np.linalg.norm(test[k])) for k in ("u", "v", "w", "p")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=None, help="iterations (the schedule's pieces scale with it)")
    ap.add_argument("--small", action="store_true", help="tiny configuration, two iterations (wiring check)")
    ap.add_argument("--output_dir", default="./output_NSFNet3")
    args = ap.parse_args()
    cfg = merged(CFG, SMALL) if args.small else CFG
    if args.epochs is not None:
        cfg = merged(cfg, {"TRAIN": {"epochs": args.epochs}})
    solver, model, equation, geom, constraint, test = build(cfg, args.output_dir)
    tic = time.perf_counter()
    solver.train()
    train_s = time.perf_counter() - tic
    metric, metric_dict = solver.eval()
    result = {"epochs": cfg["TRAIN"]["epochs"], "train_wall_s": train_s, "final_loss": solver.last_loss,
              "validator_l2rel": metric_dict["L2R"], "l2rel_with_shifted_p": errors(solver, test)}
    os.makedirs(args.output_dir, exist_ok=True)
    with open(os.path.join(args.output_dir, "result.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
