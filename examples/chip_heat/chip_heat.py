"""Chip heat operator learning with ChipDeepONets (the reference's examples/chip_heat/chip_heat.py and
conf/chip_heat.yaml), trained physics-informed without solution data.

Three branch nets read the heat source u on the 18 x 18 interior sensors, the boundary data on the 76 boundary
sensors and the boundary type bc (one column); the trunk net reads (x, y) on the unit square; the output is the
temperature T.  Five constraints, as in the reference: the steady heat equation T_xx + T_yy + 100 u = 0 inside, and on
each side a boundary condition selected by its type with nested ``torch.where``:

    bc = 0  Dirichlet    T - g                         bc = 1  Neumann     dT/dn - g
    bc = 2  convection   dT/dn + g (T - 1)             bc = 3  radiation   dT/dn + g (T^2 - 1)(T^2 + 1) 5.6 / 5e4

(n = x on the top and bottom sides, y on the left and right ones, as the reference writes them).  Every training sample
is one cell of the product point x source function x boundary type x boundary function (``ChipHeatDataset``); the
source and boundary functions are Gaussian random fields (the reference's GRF, numpy, seeded).

Besides training, ``main`` checks the trained operator against a solution the reference does not compute: the
Dirichlet case for the validation field ``test_u`` solved on the NL x NW grid with the 5-point finite-difference
Laplacian (-lap T = 100 u inside, T = u on the boundary), and prints the L2-relative error of T on the grid.

    python examples/chip_heat/chip_heat.py [--iters 20000] [--small] [--device cuda]
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
    "seed": 42, "DL": 1.0, "DW": 1.0, "NL": 20, "NW": 20, "NU": 500, "NBC": 500, "GRF_alpha": 4.0,
    "lr": 1e-3, "iters": 20000, "batch_size": 1000, "weight": 500.0,
    "MODEL": dict(branch_input_keys=("u",), BCtype_input_keys=("bc",), BC_input_keys=("bc_data",),
                  trunk_input_keys=("x", "y"), output_keys=("T",), num_loc=324, bctype_loc=1, BC_num_loc=76,
                  num_features=400, branch_num_layers=9, BC_num_layers=9, trunk_num_layers=6, branch_hidden_size=256,
                  BC_hidden_size=256, trunk_hidden_size=128, branch_activation="swish", BC_activation="swish",
                  trunk_activation="swish", use_bias=True),
}
SMALL = {"NL": 6, "NW": 6, "NU": 4, "NBC": 4, "batch_size": 64,
         "MODEL": {**CFG["MODEL"], "num_loc": 16, "BC_num_loc": 20, "num_features": 8, "branch_num_layers": 2,
                   "BC_num_layers": 2, "trunk_num_layers": 2, "branch_hidden_size": 16, "BC_hidden_size": 16,
                   "trunk_hidden_size": 16}}


def fftind(size):
    """Momentum indices of the 2-D FFT (chip_heat.py:fftind)."""
    k_ind = np.mgrid[:size, :size] - int((size + 1) / 2)
    return np.fft.fftshift(k_ind)  # every axis, as scipy.fftpack.fftshift


def GRF(alpha=3.0, size=128, flag_normalize=True):
    """Gaussian random field with a power-law spectrum 1 / |k|^(alpha / 2), as one row (chip_heat.py:GRF)."""
    k_idx = fftind(size)
    amplitude = np.power(k_idx[0] ** 2 + k_idx[1] ** 2 + 1e-10, -alpha / 4.0)
    amplitude[0, 0] = 0
    noise = np.random.normal(size=(size, size)) + 1j * np.random.normal(size=(size, size))
    gfield = np.fft.ifft2(noise * amplitude).real
    if flag_normalize:
        gfield = gfield - np.mean(gfield)
        gfield = gfield / np.std(gfield)
    return gfield.reshape([1, -1])


def boundary(d, jac, var):
    """The boundary residual of one side, selected by the boundary type (chip_heat.py, every *_sup constraint)."""
    return torch.where(
        d["bc"] == 1, jac(d["T"], d[var]) - d["u_one"],
        torch.where(d["bc"] == 0, d["T"] - d["u_one"],
                    torch.where(d["bc"] == 2, jac(d["T"], d[var]) + d["u_one"] * (d["T"] - 1),
                                jac(d["T"], d[var]) + d["u_one"] * (d["T"] ** 2 - 1) * (d["T"] ** 2 + 1) * 5.6 / 50000)))


def interior(d, jac):
    hess = lambda f, x: jac(jac(f, x), x)  # noqa: E731  (ppsci.autodiff.hessian)
    return hess(d["T"], d["x"]) + hess(d["T"], d["y"]) + 100 * d["u_one"]


def build(cfg, device):
    """Model, the five constraints and the validation inputs of the reference example."""
    np.random.seed(cfg["seed"])
    ppsci.utils.misc.set_random_seed(cfg["seed"])
    model = ppsci.arch.ChipDeepONets(**cfg["MODEL"]).to(device)
    NL, NW, DL, DW = cfg["NL"], cfg["NW"], cfg["DL"], cfg["DW"]
    pts = ppsci.geometry.Rectangle((0, 0), (DL, DW)).sample_interior(NL * NW, evenly=True)
    points = {"x": pts["x"], "y": pts["y"]}
    data_u = np.vstack([np.ones([1, (NL - 2) * (NW - 2)]), np.zeros([1, (NL - 2) * (NW - 2)])]
                       + [GRF(alpha=cfg["GRF_alpha"], size=NL - 2) for _ in range(cfg["NU"] - 2)]).astype("float32")
    data_BC = np.vstack([np.ones([1, NL * NW]), np.zeros([1, NL * NW])]
                        + [GRF(alpha=cfg["GRF_alpha"], size=NL) for _ in range(cfg["NBC"] - 2)]).astype("float32")
    test_u = GRF(alpha=4, size=NL).astype("float32")[0]
    x, y = points["x"][:, 0], points["y"][:, 0]
    bnd = np.where((x == 0) | (x == DW) | (y == 0) | (y == DL))[0]
    inner = np.where((x != 0) & (x != DW) & (y != 0) & (y != DL))[0]
    side = {"top": np.where(x == DW)[0], "down": np.where(x == 0)[0],
            "left": np.where((y == 0) & (x != 0) & (x != DW))[0], "right": np.where((y == DL) & (x != 0) & (x != DW))[0]}
    bc_types = np.array([[0], [1], [2], [3]], dtype="float32")

    def data(idx, u_one):
        return {"x": points["x"][idx], "y": points["y"][idx], "u": data_u, "u_one": u_one, "bc": bc_types,
                "bc_data": data_BC[:, bnd]}

    index = ("x", "u", "bc", "bc_data")
    label = {"chip": np.array([0], dtype="float32")}
    weight = {"chip": np.array([cfg["weight"]], dtype="float32")}

    def constraint(name, inputs, data_type, expr, w):
        return ppsci.constraint.SupervisedConstraint(
            {"dataset": {"name": "ChipHeatDataset", "input": inputs, "label": label, "index": index,
                         "data_type": data_type, **({"weight": weight} if w else {})},
             "batch_size": cfg["batch_size"], "sampler": {"name": "BatchSampler", "drop_last": False, "shuffle": True}},
            ppsci.loss.MSELoss("mean"), output_expr={"chip": expr}, name=f"{name}_sup")

    jac = ppsci.autodiff.jacobian
    csts = {}
    for name in ("down", "left", "right", "interior", "top"):  # the reference's constraint order
        if name == "interior":
            csts[name] = constraint(name, data(inner, data_u.T.reshape([-1, 1])), "u", lambda out: interior(out, jac), False)
        else:
            var = "x" if name in ("top", "down") else "y"
            csts[name] = constraint(name, data(side[name], data_BC[:, side[name]].T.reshape([-1, 1])), "bc_data",
                                    lambda out, var=var: boundary(out, jac, var), True)
    n = NL * NW
    valid = {"x": points["x"], "y": points["y"], "u": np.tile(test_u[inner], (n, 1)),
             "bc_data": np.tile(test_u[bnd], (n, 1)), "bc": np.zeros((n, 1), dtype="float32")}
    return model, {c.name: c for c in csts.values()}, valid, test_u


def dirichlet_solution(cfg, test_u):
    """-lap T = 100 u inside, T = u on the boundary: the 5-point Laplacian on the NL x NW grid of ``build`` (x-major
    point order, spacing DW / (NL - 1) in x and DL / (NW - 1) in y), one sparse solve.  Returns T at every point."""
    import scipy.sparse as sps
    from scipy.sparse.linalg import spsolve

    NL, NW = cfg["NL"], cfg["NW"]
    hx, hy = cfg["DW"] / (NL - 1), cfg["DL"] / (NW - 1)
    u = test_u.astype(np.float64).reshape(NL, NW)  # [i_x, i_y]
    inner = [(i, j) for i in range(1, NL - 1) for j in range(1, NW - 1)]
    num = {p: k for k, p in enumerate(inner)}
    rows, cols, vals = [], [], []
    rhs = np.array([100.0 * u[p] for p in inner])
    for k, (i, j) in enumerate(inner):
        rows.append(k), cols.append(k), vals.append(2 / hx ** 2 + 2 / hy ** 2)
        for (a, b), h in (((i - 1, j), hx), ((i + 1, j), hx), ((i, j - 1), hy), ((i, j + 1), hy)):
            if (a, b) in num:
                rows.append(k), cols.append(num[(a, b)]), vals.append(-1 / h ** 2)
            else:
                rhs[k] += u[a, b] / h ** 2
    A = sps.csr_matrix((vals, (rows, cols)), shape=(len(inner), len(inner)))
    T = u.copy()
    T[1:-1, 1:-1] = spsolve(A, rhs).reshape(NL - 2, NW - 2)
    return T.reshape(-1, 1)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=CFG["iters"])
    ap.add_argument("--small", action="store_true")
    ap.add_argument("--device", default="cuda")
    a = ap.parse_args(argv)
    cfg = {**CFG, **(SMALL if a.small else {})}
    model, constraint, valid, test_u = build(cfg, a.device)
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
            print(f"iter {it}: loss {history[-1]:.6g}", flush=True)
    if a.device != "cpu":
        torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ref = dirichlet_solution(cfg, test_u)
    inputs = {k: torch.as_tensor(v).to(a.device, model.dtype) for k, v in valid.items()}
    pred = model.evaluate_expressions({"T": lambda out: out["T"]}, inputs)["T"].double().cpu().numpy()
    return {"iters": a.iters, "train_wall_s": wall, "loss": history,
            "l2_rel": float(np.linalg.norm(pred - ref) / np.linalg.norm(ref))}


if __name__ == "__main__":
    res = main()
    print(json.dumps({k: (v[-1] if k == "loss" else v) for k, v in res.items()}))
