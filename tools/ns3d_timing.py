"""Step time of unsteady 3-D Navier-Stokes, fp32, on this build's native library and, alternating in the same run, on
a second build of the library (e.g. the previous commit's) given with --baseline-lib.

Three workloads, each a step = ExpressionSolver.train_forward (one fused call per plan) + Adam + clear_grad:
  (a) "beltrami": the Beltrami-flow example (examples/nsfnet/beltrami3d.py) at its configuration: 10 x 100 tanh MLP on
      (x, y, z, t), the three constraints in one batched call (70,000 + 59,400 + 29,791 points);
  (b) "wide_xyzt" / "wide_txyz": a 6 x 256 tanh MLP at 2^20 interior points on the four residuals of
      NavierStokes(0.01, 1, 3, True) alone, with the inputs in the order (x, y, z, t) and (t, x, y, z).
Each side has its own model, optimizer and plans, built while its library is the default, from the same seed.  The
sides alternate within each round; times are host clocks around work that ends in a device synchronise, medians over
the rounds after the warm-up ones.  The first step's losses of the two sides are printed beside each other.  Prints the
card's name and power limit with the times.

    python tools/ns3d_timing.py [--baseline-lib build/parent/libppsci_b200.so] [--rounds 20] [--warmup 5] [--out r.json]
"""
import argparse
import importlib.util
import json
import os
import statistics
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ppsci  # noqa: E402
from paddlescience_b200.engine import binding as B  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def _example():
    spec = importlib.util.spec_from_file_location("beltrami3d", os.path.join(ROOT, "examples", "nsfnet", "beltrami3d.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    return ex


def beltrami_side(dev):
    """The example's model, optimizer and three constraints; the (full) batches on the device."""
    ex = _example()
    solver, model, equation, geom, csts, test = ex.build(ex.CFG)
    model = model.to(dev)
    ins, labs, ws = [], [], []
    for c in csts.values():
        inp, lab, w = next(iter(c.data_loader.loader))
        ins.append({k: torch.as_tensor(v).to(dev) for k, v in inp.items()})
        labs.append({k: torch.as_tensor(v).to(dev) for k, v in lab.items()})
        ws.append({k: torch.as_tensor(v).to(dev) for k, v in w.items()} if w else None)
    opt = ppsci.optimizer.Adam(learning_rate=1e-3)(model)
    return model, opt, csts, (ins, labs, ws)


def wide_side(dev, n, keys):
    """6 x 256 tanh on ``keys``, the NS residuals at n seeded points in [0, 1]^4 (same points for both key orders)."""
    ppsci.utils.misc.set_random_seed(0)
    model = ppsci.arch.MLP(keys, ("u", "v", "w", "p"), 6, 256, "tanh").to(dev)
    eq = ppsci.equation.NavierStokes(0.01, 1.0, 3, True)
    rng = np.random.RandomState(0)
    inp = {k: torch.as_tensor(rng.rand(n, 1), dtype=torch.float32, device=dev) for k in ("x", "y", "z", "t")}
    lab = {k: torch.zeros(n, 1, device=dev) for k in eq.equations}
    csts = {"EQ": types.SimpleNamespace(loss=ppsci.loss.MSELoss("mean"), output_expr=dict(eq.equations))}
    opt = ppsci.optimizer.Adam(learning_rate=1e-4)(model)
    return model, opt, csts, ([inp], [lab], [None])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", default=None, help="second native library to alternate with (same C-ABI)")
    ap.add_argument("--points", type=int, default=1 << 20, help="interior points of the wide workloads")
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ns3d_timing needs a CUDA (H100) device")
    dev = "cuda"
    libs = {"this": B.Library()}
    if a.baseline_lib:
        libs["baseline"] = B.Library(os.path.abspath(a.baseline_lib))
    workloads = (("beltrami", lambda: beltrami_side(dev)),
                 ("wide_xyzt", lambda: wide_side(dev, a.points, ("x", "y", "z", "t"))),
                 ("wide_txyz", lambda: wide_side(dev, a.points, ("t", "x", "y", "z"))))
    sides = {}
    for wl, make in workloads:
        for lk, lib in libs.items():
            B._default = lib  # plans bind the default library at creation
            model, opt, csts, batch = make()
            sides[(wl, lk)] = dict(lib=lib, model=model, opt=opt, csts=csts, batch=batch, fh=ppsci.utils.ExpressionSolver())

    def step(s):
        B._default = s["lib"]  # Adam's kernel comes from the default library
        ins, labs, ws = s["batch"]
        la, lc = s["fh"].train_forward(tuple(c.output_expr for c in s["csts"].values()), ins, s["model"], s["csts"],
                                       labs, ws)
        s["opt"].step()
        s["opt"].clear_grad()
        return lc

    first = {}
    for key, s in sides.items():
        first[key] = {k: float(v) for k, v in step(s).items()}
    times = {key: [] for key in sides}
    for r in range(a.warmup + a.rounds):
        for key, s in sides.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step(s)
            torch.cuda.synchronize()
            if r >= a.warmup:
                times[key].append((time.perf_counter() - t0) * 1e3)
    name, q = card()
    res = {"card": name, "power_limit_and_max_sm_clock": q, "rounds": a.rounds, "wide_points": a.points,
           "libraries": {k: v.path for k, v in libs.items()},
           "ms_median": {f"{wl}/{lk}": statistics.median(v) for (wl, lk), v in times.items()},
           "ms_min_max": {f"{wl}/{lk}": [min(v), max(v)] for (wl, lk), v in times.items()},
           "first_step_losses": {f"{wl}/{lk}": v for (wl, lk), v in first.items()}}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
