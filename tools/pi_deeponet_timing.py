"""Step time of physics-informed DeepONet against the supervised step, at the cfg5 shapes (branch 100 -> 128 x 3 -> 128,
trunk 1 -> 128 x 3 -> 128, fp32).

One run, the three steps alternating: the supervised step (loss on G, values only), the PI step at order 1 (dG/dy - u(y))
and the PI step at order 2 (G G_y + G_yy - f(y)).  A step is ExpressionSolver.train_forward + Adam + clear_grad, timed
with a host clock around work that ends in a device synchronise; medians over the timed rounds after the warm-up ones.
Prints the card's name and power limit with the times.

    python tools/pi_deeponet_timing.py [--pairs 65536] [--rounds 30] [--warmup 5] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ppsci  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1 << 16)
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pi_deeponet_timing needs a CUDA (H100) device")
    dev = "cuda"
    ppsci.utils.misc.set_random_seed(0)
    model = ppsci.arch.DeepONet("u", "y", "G", 100, 128, None, None, (128,) * 3, (128,) * 3).to(dev)
    rng = np.random.RandomState(0)
    n = a.pairs
    t = lambda m: torch.as_tensor(m, dtype=torch.float32, device=dev)  # noqa: E731
    inputs = {"u": t(rng.randn(n, 100)), "y": t(rng.rand(n, 1)), "u_y": t(rng.randn(n, 1)), "f": t(rng.randn(n, 1))}
    jac = ppsci.autodiff.jacobian
    steps = {
        "supervised": ({"G": lambda d: d["G"]}, {"G": t(rng.randn(n, 1))}),
        "pi_order1": ({"res": lambda d: jac(d["G"], d["y"]) - d["u_y"]}, {"res": t(np.zeros((n, 1)))}),
        "pi_order2": ({"res": lambda d: d["G"] * jac(d["G"], d["y"]) + jac(jac(d["G"], d["y"]), d["y"]) - d["f"]},
                      {"res": t(np.zeros((n, 1)))}),
    }
    opt = ppsci.optimizer.Adam(learning_rate=1e-4)(model)
    fh = ppsci.utils.ExpressionSolver()
    csts = {k: types.SimpleNamespace(loss=ppsci.loss.MSELoss("mean"), output_expr=e) for k, (e, _) in steps.items()}

    def step(k):
        fh.train_forward((csts[k].output_expr,), [inputs], model, {k: csts[k]}, [steps[k][1]], [None])
        opt.step()
        opt.clear_grad()

    times = {k: [] for k in steps}
    for r in range(a.warmup + a.rounds):
        for k in steps:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step(k)
            torch.cuda.synchronize()
            if r >= a.warmup:
                times[k].append((time.perf_counter() - t0) * 1e3)
    name, q = card()
    res = {"card": name, "power_limit_and_max_sm_clock": q, "pairs": n, "rounds": a.rounds,
           **{f"{k}_ms_median": statistics.median(v) for k, v in times.items()},
           **{f"{k}_ms_min": min(v) for k, v in times.items()}}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
