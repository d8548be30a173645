"""Step time of HEDeepONets at the heat-exchanger example's shapes (heat / cold branches 1 -> 256 x 9 -> 300, trunk
2 -> 128 x 6 -> 300, swish, fp32).

One run, three steps alternating: the example's step (its four constraints, 1,000 pairs each), the interior constraint
alone (the three HeatExchanger residuals) at ``--pairs`` pairs, and the same model trained supervised on the values of
T_h, T_c and T_w at ``--pairs`` pairs (the baseline: a values-only head, no trunk jets).  A step is
ExpressionSolver.train_forward + Adam + clear_grad, timed with a host clock around work that ends in a device
synchronise; medians over the timed rounds after the warm-up ones.  Prints the card's name and power limit with the
times.

    python tools/he_deeponet_timing.py [--pairs 65536] [--rounds 30] [--warmup 5] [--out result.json]
"""
import argparse
import json
import os
import statistics
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples", "heat_exchanger"))
import heat_exchanger as ex  # noqa: E402
import ppsci  # noqa: E402
from pi_deeponet_timing import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1 << 16)
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("he_deeponet_timing needs a CUDA (H100) device")
    dev = "cuda"
    cfg = dict(ex.CFG)
    model, constraint, _ = ex.build(cfg, dev)
    loaders = [iter(c.data_loader) for c in constraint.values()]
    to = lambda d: {k: v.to(dev, torch.float32) for k, v in d.items()}  # noqa: E731
    example_batches = [tuple(to(d) for d in next(b)) for b in loaders]  # one fixed batch of 1,000 pairs per constraint

    rng = np.random.RandomState(0)
    n = a.pairs
    t = lambda m: torch.as_tensor(m, dtype=torch.float32, device=dev)  # noqa: E731
    inputs = {"x": t(rng.rand(n, 1)), "t": t(2 * rng.rand(n, 1)), "qm_h": t(2 * rng.rand(n, 1)), "qm_c": t(2 * rng.rand(n, 1))}
    eqs = ex._equation(cfg).equations
    interior = types.SimpleNamespace(loss=ppsci.loss.MSELoss("mean"), output_expr=eqs)
    supervised = types.SimpleNamespace(loss=ppsci.loss.MSELoss("mean"), output_expr={})
    zeros = {k: t(np.zeros((n, 1))) for k in eqs}
    values = {k: t(rng.randn(n, 1)) for k in model.output_keys}
    opt = ppsci.optimizer.Adam(learning_rate=1e-4)(model)
    fh = ppsci.utils.ExpressionSolver()
    steps = {
        "example_4_constraints": lambda: fh.train_forward(
            tuple(c.output_expr for c in constraint.values()), [b[0] for b in example_batches], model, constraint,
            [b[1] for b in example_batches], [b[2] for b in example_batches]),
        "interior": lambda: fh.train_forward((eqs,), [inputs], model, {"interior": interior}, [zeros], [None]),
        "supervised_values": lambda: fh.train_forward(({},), [inputs], model, {"sup": supervised}, [values], [None]),
    }

    times = {k: [] for k in steps}
    for r in range(a.warmup + a.rounds):
        for k, fn in steps.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            opt.step()
            opt.clear_grad()
            torch.cuda.synchronize()
            if r >= a.warmup:
                times[k].append((time.perf_counter() - t0) * 1e3)
    name, q = card()
    res = {"card": name, "power_limit_and_max_sm_clock": q, "pairs": n, "example_batch": cfg["batch_size"],
           "rounds": a.rounds, **{f"{k}_ms_median": statistics.median(v) for k, v in times.items()},
           **{f"{k}_ms_min": min(v) for k, v in times.items()}}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
