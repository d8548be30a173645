"""Step time of ChipDeepONets at the chip-heat example's shapes (heat-source branch 324 -> 256 x 9 -> 400, boundary-data
and boundary-type branches 76 / 1 -> 256 x 9 -> 400, trunk 2 -> 128 x 6 -> 400, swish, fp32).

One run, two steps alternating: the example's step (its five constraints, 1,000 pairs each: four boundary constraints
whose residual is selected by boundary type, and the interior heat equation) and the interior constraint alone at
``--pairs`` pairs.  A step is ExpressionSolver.train_forward + Adam + clear_grad, timed with a host clock around work
that ends in a device synchronise; medians over the timed rounds after the warm-up ones.  Also reports which kernels
serve each sub-network (``uses_tcgen05``: the tensor-core kernels of sm_90a; otherwise the CUDA-core ones).  Prints the
card's name and power limit with the times.

    python tools/chip_deeponet_timing.py [--pairs 65536] [--rounds 30] [--warmup 5] [--out result.json]
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
sys.path.insert(0, os.path.join(ROOT, "examples", "chip_heat"))
import chip_heat as ex  # noqa: E402
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
        raise SystemExit("chip_deeponet_timing needs a CUDA (H100) device")
    dev = "cuda"
    cfg = dict(ex.CFG)
    model, constraint, _, _ = ex.build(cfg, dev)
    loaders = [iter(c.data_loader) for c in constraint.values()]
    to = lambda d: {k: v.to(dev, torch.float32) for k, v in d.items()}  # noqa: E731
    example_batches = [tuple(to(d) for d in next(b)) for b in loaders]  # one fixed batch of 1,000 pairs per constraint

    rng = np.random.RandomState(0)
    n = a.pairs
    m = cfg["MODEL"]
    t = lambda v: torch.as_tensor(v, dtype=torch.float32, device=dev)  # noqa: E731
    inputs = {"x": t(rng.rand(n, 1)), "y": t(rng.rand(n, 1)), "u": t(rng.randn(n, m["num_loc"])),
              "bc_data": t(rng.randn(n, m["BC_num_loc"])), "bc": t(rng.randint(0, 4, (n, 1))), "u_one": t(rng.randn(n, 1))}
    expr = {"chip": lambda out: ex.interior(out, ppsci.autodiff.jacobian)}
    interior = types.SimpleNamespace(loss=ppsci.loss.MSELoss("mean"), output_expr=expr)
    zeros = {"chip": t(np.zeros((n, 1)))}
    opt = ppsci.optimizer.Adam(learning_rate=1e-4)(model)
    fh = ppsci.utils.ExpressionSolver()
    steps = {
        "example_5_constraints": lambda: fh.train_forward(
            tuple(c.output_expr for c in constraint.values()), [b[0] for b in example_batches], model, constraint,
            [b[1] for b in example_batches], [b[2] for b in example_batches]),
        "interior": lambda: fh.train_forward((expr,), [inputs], model, {"interior": interior}, [zeros], [None]),
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
    plans = {name: p.uses_tcgen05 for name, p in zip(model._sub_names[:-1], model._get_plans()[:-1])}
    for head in model._jet_heads.values():
        plans[f"trunk_net (C={head.compiled.channels})"] = head.trunk_plan.uses_tcgen05
    name, q = card()
    res = {"card": name, "power_limit_and_max_sm_clock": q, "pairs": n, "example_batch": cfg["batch_size"],
           "rounds": a.rounds, **{f"{k}_ms_median": statistics.median(v) for k, v in times.items()},
           **{f"{k}_ms_min": min(v) for k, v in times.items()}, "uses_tcgen05": plans}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
