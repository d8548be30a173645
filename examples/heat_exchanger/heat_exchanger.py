"""Heat exchanger operator learning with HEDeepONets (the reference's examples/heat_exchanger/heat_exchanger.py and
conf/heat_exchanger.yaml), trained physics-informed without solution data.

Two branch nets read the hot and the cold side's mass flow rates qm_h, qm_c, the trunk net (x, t); the outputs are the
hot fluid, cold fluid and wall temperatures T_h, T_c, T_w.  Four constraints, as in the reference: the hot inlet
T_h(0, t) = T_hin, the cold inlet T_c(DL, t) = T_cin (written, like the reference, under the label key "T_h"), the
HeatExchanger equations on every point, and the initial temperatures.  Every constraint runs through the operator jet
head; x and t derivatives come from the trunk's Taylor jets.

The grid is the one ``TimeXGeometry(TimeDomain(0, 1, timestamps=linspace(0, 2, NTIME + 1)), Interval(0, DL))
.sample_interior(NPOINT * NTIME, evenly=True)`` gives (ppsci/geometry/timedomain.py:156-201), built here with numpy:
time-major, t = timestamps[1:], and for each t, x = linspace(0, DL, NPOINT) (``geometry.TimeXGeometry`` gives the same
points, tests/test_time_geometry.py).  The grid is replicated over NQM x NQM random (qm_h, qm_c) pairs the way the reference does.

Besides the reference's validators (MSE of the boundary conditions and the residuals on a held-out (qm_h, qm_c)),
``main`` checks the trained operator against an independent solution the reference does not have: an upwind
method-of-lines discretisation of the same three equations on a fine x grid (scipy ``solve_ivp``), and prints the
L2-relative error of each field on the NPOINT x NTIME grid.

    python examples/heat_exchanger/heat_exchanger.py [--iters 10000] [--small] [--device cuda]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import ppsci  # noqa: E402

CFG = {
    "seed": 42, "DL": 1.0, "cp_c": 1.0, "cp_h": 1.0, "cp_w": 1.0, "v_h": 1.0, "v_c": 1.0, "alpha_h": 1.0, "alpha_c": 1.0,
    "L": 1.0, "M": 1.0, "T_hin": 10.0, "T_cin": 1.0, "T_win": 5.5, "NTIME": 20, "NPOINT": 101, "NQM": 60,
    "lr": 1e-3, "iters": 10000, "batch_size": 1000,
    "weight": {"left": {"T_h": 20.0}, "right": {"T_h": 20.0},
               "interior": {"heat_boundary": 1.0, "cold_boundary": 1.0, "wall": 20.0},
               "initial": {"T_h": 1.0, "T_c": 1.0, "T_w": 20.0}},
    "MODEL": dict(heat_input_keys=("qm_h",), cold_input_keys=("qm_c",), trunk_input_keys=("x", "t"),
                  output_keys=("T_h", "T_c", "T_w"), heat_num_loc=1, cold_num_loc=1, num_features=100, branch_num_layers=9,
                  trunk_num_layers=6, branch_hidden_size=256, trunk_hidden_size=128, branch_activation="swish",
                  trunk_activation="swish", use_bias=True),
}
SMALL = {"NQM": 3, "MODEL": {**CFG["MODEL"], "num_features": 8, "branch_num_layers": 2, "trunk_num_layers": 2,
                             "branch_hidden_size": 16, "trunk_hidden_size": 16}}


def grid(cfg):
    """TimeXGeometry(...).sample_interior(NPOINT * NTIME, evenly=True): time-major, t = timestamps[1:]."""
    timestamps = np.linspace(0.0, 2, cfg["NTIME"] + 1, endpoint=True)
    x = np.linspace(0.0, cfg["DL"], cfg["NPOINT"])
    return {"t": np.repeat(timestamps[1:], len(x)).reshape(-1, 1).astype("float32"),
            "x": np.tile(x, cfg["NTIME"]).reshape(-1, 1).astype("float32")}


def _equation(cfg):
    return ppsci.equation.HeatExchanger(cfg["alpha_h"] / (cfg["L"] * cfg["cp_h"]), cfg["alpha_c"] / (cfg["L"] * cfg["cp_c"]),
                                        cfg["v_h"], cfg["v_c"], cfg["alpha_h"] / (cfg["M"] * cfg["cp_w"]),
                                        cfg["alpha_c"] / (cfg["M"] * cfg["cp_w"]))


def build(cfg, device):
    """Model, the four constraints and the three validators of the reference example."""
    ppsci.utils.misc.set_random_seed(cfg["seed"])
    model = ppsci.arch.HEDeepONets(**cfg["MODEL"]).to(device)
    nqm, n_grid = cfg["NQM"], cfg["NPOINT"] * cfg["NTIME"]
    visu = grid(cfg)
    data_h = (np.random.rand(nqm).reshape([-1, 1]) * 2).astype("float32")
    data_c = (np.random.rand(nqm).reshape([-1, 1]) * 2).astype("float32")
    test_h = np.random.rand(1).reshape([-1, 1]).astype("float32")
    test_c = np.random.rand(1).reshape([-1, 1]).astype("float32")
    points = dict(visu)  # heat_exchanger.py:54-62
    points["t"] = np.repeat(points["t"], nqm, axis=0)
    points["x"] = np.repeat(points["x"], nqm, axis=0)
    points["qm_h"] = np.tile(data_h, (n_grid, 1))
    points["t"] = np.repeat(points["t"], nqm, axis=0)
    points["x"] = np.repeat(points["x"], nqm, axis=0)
    points["qm_h"] = np.repeat(points["qm_h"], nqm, axis=0)
    points["qm_c"] = np.tile(data_c, (n_grid * nqm, 1))
    visu["qm_h"] = np.tile(test_h, (n_grid, 1))
    visu["qm_c"] = np.tile(test_c, (n_grid, 1))

    keys = ("x", "t", "qm_h", "qm_c")
    pick = lambda d, i: {k: d[k][i] for k in keys}  # noqa: E731
    left = pick(points, np.where(points["x"][:, 0] == 0)[0])
    right = pick(points, np.where(points["x"][:, 0] == cfg["DL"])[0])
    initial = pick(points, np.where(points["t"][:, 0] == points["t"][0, 0])[0])
    initial["t"] = initial["t"] * 0
    interior = {k: points[k] for k in keys}
    eqs = _equation(cfg).equations
    T_hin, T_cin, T_win = cfg["T_hin"], cfg["T_cin"], cfg["T_win"]
    zeros = lambda d: np.zeros([d["x"].shape[0], 1], dtype="float32")  # noqa: E731

    def constraint(name, inputs, exprs):
        w = cfg["weight"][name]
        return ppsci.constraint.SupervisedConstraint(
            {"dataset": {"name": "NamedArrayDataset", "input": inputs, "label": {k: zeros(inputs) for k in exprs},
                         "weight": {k: np.full_like(inputs["x"], w[k]) for k in exprs}},
             "batch_size": cfg["batch_size"], "sampler": {"name": "BatchSampler", "drop_last": False, "shuffle": True}},
            ppsci.loss.MSELoss("mean"), output_expr=exprs, name=f"{name}_sup")

    csts = [constraint("left", left, {"T_h": lambda out: out["T_h"] - T_hin}),
            constraint("right", right, {"T_h": lambda out: out["T_c"] - T_cin}),
            constraint("interior", interior, eqs),
            constraint("initial", initial, {"T_h": lambda out: out["T_h"] - T_hin, "T_c": lambda out: out["T_c"] - T_cin,
                                            "T_w": lambda out: out["T_w"] - T_win})]

    def validator(name, inputs, exprs):
        return ppsci.validate.SupervisedValidator(
            {"dataset": {"name": "NamedArrayDataset", "input": inputs, "label": {k: zeros(inputs) for k in exprs}},
             "batch_size": cfg["NTIME"], "sampler": {"name": "BatchSampler", "drop_last": False, "shuffle": False}},
            ppsci.loss.MSELoss("mean"), output_expr=exprs, metric={"MSE": ppsci.metric.MSE()}, name=name)

    vals = [validator("left_mse", pick(visu, np.where(visu["x"][:, 0] == 0)[0]), {"T_h": lambda out: out["T_h"] - T_hin}),
            validator("right_mse", pick(visu, np.where(visu["x"][:, 0] == cfg["DL"])[0]),
                      {"T_h": lambda out: out["T_c"] - T_cin}),
            validator("interior_mse", {k: visu[k] for k in keys}, eqs)]
    return model, {c.name: c for c in csts}, {v.name: v for v in vals}


def full_batches(constraint, device):
    """(inputs, labels, weights) of every constraint: its whole point set as one batch, on the device."""
    to = lambda d: {k: torch.as_tensor(v).to(device) for k, v in d.items()}  # noqa: E731
    return [(to(c.data_loader.loader.ds.input), to(c.data_loader.loader.ds.label), to(c.data_loader.loader.ds.weight))
            for c in constraint.values()]


def reference_solution(cfg, qm_h, qm_c, nx=2001):
    """Upwind method of lines for the same three equations: T_h flows towards +x (inlet T_h(0, t) = T_hin), T_c towards
    -x (inlet T_c(DL, t) = T_cin); initial temperatures T_hin / T_cin / T_win.  Returns T_h, T_c, T_w on the
    NPOINT x NTIME grid (time-major, as ``grid``)."""
    from scipy.integrate import solve_ivp

    eq = dict(a_h=cfg["alpha_h"] / (cfg["L"] * cfg["cp_h"]), a_c=cfg["alpha_c"] / (cfg["L"] * cfg["cp_c"]),
              w_h=cfg["alpha_h"] / (cfg["M"] * cfg["cp_w"]), w_c=cfg["alpha_c"] / (cfg["M"] * cfg["cp_w"]))
    v_h, v_c = cfg["v_h"], cfg["v_c"]
    b_h, b_c = eq["a_h"] * v_h / qm_h, eq["a_c"] * v_c / qm_c
    xs = np.linspace(0.0, cfg["DL"], nx)
    dx = xs[1] - xs[0]

    def rhs(_, y):
        th, tc, tw = y[:nx].copy(), y[nx:2 * nx].copy(), y[2 * nx:]
        th[0], tc[-1] = cfg["T_hin"], cfg["T_cin"]
        dth = np.zeros(nx)
        dtc = np.zeros(nx)
        dth[1:] = -v_h * (th[1:] - th[:-1]) / dx + b_h * (tw[1:] - th[1:])  # T_h,t = -v_h T_h,x + beta_h (T_w - T_h)
        dtc[:-1] = v_c * (tc[1:] - tc[:-1]) / dx + b_c * (tw[:-1] - tc[:-1])  # T_c,t = v_c T_c,x + beta_c (T_w - T_c)
        dtw = eq["w_h"] * (th - tw) + eq["w_c"] * (tc - tw)
        return np.concatenate([dth, dtc, dtw])

    y0 = np.concatenate([np.full(nx, cfg["T_hin"]), np.full(nx, cfg["T_cin"]), np.full(nx, cfg["T_win"])])
    ts = np.linspace(0.0, 2, cfg["NTIME"] + 1)[1:]
    sol = solve_ivp(rhs, (0.0, ts[-1]), y0, t_eval=ts, method="RK45", rtol=1e-8, atol=1e-8)
    xg = np.linspace(0.0, cfg["DL"], cfg["NPOINT"])
    out = {}
    for i, k in enumerate(("T_h", "T_c", "T_w")):
        field = sol.y[i * nx:(i + 1) * nx]  # [nx, NTIME]
        out[k] = np.stack([np.interp(xg, xs, field[:, j]) for j in range(len(ts))]).reshape(-1, 1)
    return out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=CFG["iters"])
    ap.add_argument("--small", action="store_true")
    ap.add_argument("--device", default="cuda")
    ap.add_argument("--no-reference", action="store_true", help="skip the method-of-lines comparison")
    a = ap.parse_args(argv)
    cfg = {**CFG, **(SMALL if a.small else {})}
    model, constraint, validator = build(cfg, a.device)
    optimizer = ppsci.optimizer.Adam(learning_rate=cfg["lr"])(model)
    fh = ppsci.utils.ExpressionSolver()
    iters = [iter(c.data_loader) for c in constraint.values()]
    to = lambda d: {k: v.to(a.device, model.dtype) for k, v in d.items()}  # noqa: E731
    history = []
    t0 = time.perf_counter()
    for it in range(a.iters):  # Solver.train's step (solver/train.py) spelled out: one fused call per constraint
        batches = [next(b) for b in iters]
        losses, _ = fh.train_forward(tuple(c.output_expr for c in constraint.values()), [to(b[0]) for b in batches], model,
                                     constraint, [to(b[1]) for b in batches], [to(b[2]) for b in batches])
        optimizer.step()
        optimizer.clear_grad()
        if it % max(1, a.iters // 100) == 0 or it == a.iters - 1:
            history.append(float(sum(losses.values())))
    if a.device != "cpu":
        torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    out = {"iters": a.iters, "train_wall_s": wall, "loss": history}
    if not a.no_reference:
        vin = validator["interior_mse"].data_loader.loader.ds.input
        qm_h, qm_c = float(vin["qm_h"][0, 0]), float(vin["qm_c"][0, 0])
        ref = reference_solution(cfg, qm_h, qm_c)
        inputs = {k: torch.as_tensor(v).to(a.device, model.dtype) for k, v in vin.items()}
        pred = model.evaluate_expressions({k: (lambda out, k=k: out[k]) for k in ref}, inputs)
        out["qm_h"], out["qm_c"] = qm_h, qm_c
        for k, r in ref.items():
            p = pred[k].double().cpu().numpy()
            out[f"l2_rel_{k}"] = float(np.linalg.norm(p - r) / np.linalg.norm(r))
    return out


if __name__ == "__main__":
    res = main()
    print(json.dumps({k: (v[-1] if k == "loss" else v) for k, v in res.items()}))
