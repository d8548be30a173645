"""Allen-Cahn with PirateNet — the reference's SOTA example (examples/allen_cahn/allen_cahn_piratenet.py:63-193,
conf/allen_cahn_piratenet.yaml) on the H100-native engine: same script structure and the same ``ppsci`` calls
(PirateNet with fourier + random_weight + periods, CausalMSELoss on a freshly sampled PDE batch, supervised initial
condition, ExponentialDecay, mtl.GradNorm); the hydra / yaml layer is the plain dict below.

The reference reads the initial condition and the solution it validates against from ``allen_cahn.mat``, which is not
shipped (no network here).  The benchmark's initial condition is analytic — u(0, x) = x^2 cos(pi x) on [-1, 1], periodic —
so it is evaluated directly on the reference's 512-point grid; pass ``--data allen_cahn.mat`` (needs scipy) to add the
reference's L2Rel validator against ``usol``.

``--arch modifiedmlp`` runs the sibling example examples/allen_cahn/allen_cahn_sota.py (conf/allen_cahn_sota.yaml): the
same script with ``ppsci.arch.ModifiedMLP`` (4 x 256, the same fourier / random_weight / periods options).

    python examples/allen_cahn/allen_cahn_piratenet.py [--arch piratenet|modifiedmlp] [--epochs 300] [--small]
                                                       [--output_dir ./output_allen_cahn_piratenet]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import ppsci  # noqa: E402
from ppsci.loss import mtl  # noqa: E402

CFG = {
    "seed": 42,
    "MODEL": {"input_keys": ("t", "x"), "output_keys": ("u",), "num_blocks": 3, "hidden_size": 256, "activation": "tanh",
              "periods": {"x": (2.0, False)}, "fourier": {"dim": 256, "scale": 2.0},
              "random_weight": {"mean": 1.0, "std": 0.1}},
    "TRAIN": {"epochs": 300, "iters_per_epoch": 1000, "batch_size": 8192,
              "lr_scheduler": {"learning_rate": 1.0e-3, "gamma": 0.9, "decay_steps": 5000, "by_epoch": False},
              "causal": {"n_chunks": 32, "tol": 1.0}, "grad_norm": {"update_freq": 1000, "momentum": 0.9}},
    "GRID": {"nt": 201, "nx": 512, "t0": 0.0, "t1": 1.0, "x0": -1.0, "x1": 1.0},
}
MODEL_SOTA = {"input_keys": ("t", "x"), "output_keys": ("u",), "num_layers": 4, "hidden_size": 256, "activation": "tanh",
              "periods": {"x": (2.0, False)}, "fourier": {"dim": 256, "scale": 2.0},
              "random_weight": {"mean": 1.0, "std": 0.1}}  # conf/allen_cahn_sota.yaml:36-49
SMALL = {  # wiring / smoke configuration (tests/test_examples.py builds it on the CPU)
    "MODEL": {"num_blocks": 1, "hidden_size": 16, "fourier": {"dim": 16, "scale": 2.0}},
    "TRAIN": {"epochs": 1, "iters_per_epoch": 2, "batch_size": 32, "causal": {"n_chunks": 4, "tol": 1.0},
              "grad_norm": {"update_freq": 1, "momentum": 0.9}},
    "GRID": {"nt": 5, "nx": 16},
}


def merged(base, over):
    out = dict(base)
    for k, v in over.items():
        out[k] = merged(base[k], v) if isinstance(v, dict) and isinstance(base.get(k), dict) and k not in ("periods", "fourier") else v
    return out


def build(cfg, data_path=None, arch="piratenet"):
    """Model, equation, constraints, optimizer, validators and the Solver — everything up to ``solver.train()``."""
    ppsci.utils.misc.set_random_seed(cfg["seed"])
    dtype = "float32"
    if arch == "modifiedmlp":  # allen_cahn_sota.py:64
        mcfg = dict(MODEL_SOTA)
        if cfg["MODEL"]["hidden_size"] != CFG["MODEL"]["hidden_size"]:  # the small configuration
            mcfg.update(num_layers=2, hidden_size=cfg["MODEL"]["hidden_size"], fourier=cfg["MODEL"]["fourier"])
        model = ppsci.arch.ModifiedMLP(**mcfg)
    else:
        model = ppsci.arch.PirateNet(**cfg["MODEL"])
    equation = {"AllenCahn": ppsci.equation.AllenCahn(eps=0.01)}
    g = cfg["GRID"]
    x_star = np.linspace(g["x0"], g["x1"], g["nx"], endpoint=False).astype(dtype)  # the benchmark's periodic grid
    t_star = np.linspace(g["t0"], g["t1"], g["nt"]).astype(dtype)
    u_ref = None
    if data_path:
        import scipy.io as sio

        data = sio.loadmat(data_path)
        u_ref = data["usol"].astype(dtype)
        t_star, x_star = data["t"].flatten().astype(dtype), data["x"].flatten().astype(dtype)
    u0 = u_ref[0, :] if u_ref is not None else (x_star ** 2 * np.cos(np.pi * x_star)).astype(dtype)
    t0, t1, x0, x1 = float(t_star[0]), float(t_star[-1]), float(x_star[0]), float(x_star[-1])
    bs = cfg["TRAIN"]["batch_size"]

    def gen_input_batch():
        tx = np.random.uniform([t0, x0], [t1, x1], (bs, 2)).astype(dtype)
        return {"t": np.sort(tx[:, 0:1], axis=0), "x": tx[:, 1:2]}

    def gen_label_batch(input_batch):
        return {"allen_cahn": np.zeros([bs, 1], dtype)}

    pde_constraint = ppsci.constraint.SupervisedConstraint(
        {"dataset": {"name": "ContinuousNamedArrayDataset", "input": gen_input_batch, "label": gen_label_batch}},
        output_expr=equation["AllenCahn"].equations,
        loss=ppsci.loss.CausalMSELoss(cfg["TRAIN"]["causal"]["n_chunks"], "mean", tol=cfg["TRAIN"]["causal"]["tol"]),
        name="PDE")
    ic_input = {"t": np.full([len(x_star), 1], t0, dtype), "x": x_star.reshape([-1, 1])}
    ic_label = {"u": u0.reshape([-1, 1])}
    ic = ppsci.constraint.SupervisedConstraint(
        {"dataset": {"name": "IterableNamedArrayDataset", "input": ic_input, "label": ic_label}},
        output_expr={"u": lambda out: out["u"]}, loss=ppsci.loss.MSELoss("mean"), name="IC")
    constraint = {pde_constraint.name: pde_constraint, ic.name: ic}
    sched = cfg["TRAIN"]["lr_scheduler"]
    lr_scheduler = ppsci.optimizer.lr_scheduler.ExponentialDecay(
        epochs=cfg["TRAIN"]["epochs"], iters_per_epoch=cfg["TRAIN"]["iters_per_epoch"], **sched)()
    optimizer = ppsci.optimizer.Adam(lr_scheduler)(model)
    validator = None
    tx_star = ppsci.utils.misc.cartesian_product(t_star, x_star).astype(dtype)
    eval_data = {"t": tx_star[:, 0:1], "x": tx_star[:, 1:2]}
    if u_ref is not None:
        u_validator = ppsci.validate.SupervisedValidator(
            {"dataset": {"name": "NamedArrayDataset", "input": eval_data, "label": {"u": u_ref.reshape([-1, 1])}},
             "batch_size": 4096},
            ppsci.loss.MSELoss("mean"), {"u": lambda out: out["u"]}, metric={"L2Rel": ppsci.metric.L2Rel()}, name="u_validator")
        validator = {u_validator.name: u_validator}
    gn = cfg["TRAIN"]["grad_norm"]
    solver = ppsci.solver.Solver(
        model, constraint, None, optimizer, lr_scheduler, cfg["TRAIN"]["epochs"], cfg["TRAIN"]["iters_per_epoch"],
        equation=equation, validator=validator, eval_during_train=False,
        loss_aggregator=mtl.GradNorm(model, len(constraint), gn["update_freq"], gn["momentum"]))
    return solver, model, equation, constraint, eval_data


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=None)
    ap.add_argument("--arch", choices=("piratenet", "modifiedmlp"), default="piratenet")
    ap.add_argument("--small", action="store_true", help="tiny configuration (wiring check)")
    ap.add_argument("--data", default=None, help="allen_cahn.mat of the reference (optional: adds the L2Rel validator)")
    ap.add_argument("--output_dir", default="./output_allen_cahn_piratenet")
    args = ap.parse_args()
    cfg = merged(CFG, SMALL) if args.small else CFG
    if args.epochs is not None:
        cfg = merged(cfg, {"TRAIN": {"epochs": args.epochs}})
    solver, model, equation, constraint, eval_data = build(cfg, args.data, args.arch)
    tic = time.perf_counter()
    solver.train()
    train_s = time.perf_counter() - tic
    result = {"train_s": train_s, "epochs": cfg["TRAIN"]["epochs"], "iters_per_epoch": cfg["TRAIN"]["iters_per_epoch"]}
    if solver.validator:
        result["eval"] = solver.eval()
    # residual of the trained network on the evaluation grid (no reference data needed)
    res = ppsci.lambdify(equation["AllenCahn"].equations["allen_cahn"], model)
    import torch

    dev = model.flat.device
    r = res({k: torch.as_tensor(v, device=dev) for k, v in eval_data.items()})
    result["pde_residual_rms"] = float((r.double() ** 2).mean().sqrt())
    os.makedirs(args.output_dir, exist_ok=True)
    with open(os.path.join(args.output_dir, "result.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
