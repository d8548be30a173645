"""Cost of learning a PeriodEmbedding frequency: an Allen-Cahn-sized fp32 MLP (u(t, x), 4 x 256 tanh, 2^18 collocation
points, residual u_t - 1e-4 u_xx + 5 u^3 - 5 u) with a FIXED versus a TRAINABLE x period.

The trainable plan folds dLoss/d omega into the thin first-layer weight-gradient kernel (thin::k_first_dw_v with its
OMEGA switch on) and adds one tiny launch that moves the fp64 sums into the gradient buffer.  Reported per training call
(one loss + weight gradient over all points): the device time of profile class 7 (thin first-layer dW, the kernel the
reduction is fused into), of class 4 (misc, which holds the extra launch) and of all classes, from the library's
per-launch CUDA-event profile; and the call time with profiling off (CUDA events around ``--steps`` calls).  The two
plans alternate for ``--rounds`` rounds so that drift on a shared machine hits both.  The GPU's name, power limit and
clocks are read in the same run and printed beside the numbers.

    python tools/omega_dw_timing.py [--points 262144] [--steps 20] [--rounds 3] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import sympy as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import ppsci  # noqa: E402
from paddlescience_b200.engine.compiler import compile_residuals  # noqa: E402
from paddlescience_b200.engine.plan import ResidualPlan  # noqa: E402


def _gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem,temperature.gpu"
    try:
        line = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              check=True).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in line.split(",")]))
    except (OSError, subprocess.CalledProcessError, IndexError):
        return {"name": torch.cuda.get_device_name(0)}


def _setup(trainable: bool, n: int):
    torch.manual_seed(0)
    m = ppsci.arch.MLP(("t", "x"), ("u",), 4, 256, "tanh", periods={"x": (2.0, trainable)}).to("cuda")
    t, x = sp.symbols("t x")
    u = sp.Function("u")(t, x)
    plan = ResidualPlan(compile_residuals(m.net_spec(), {"ac": u.diff(t) - 1e-4 * u.diff(x, 2) + 5 * u ** 3 - 5 * u},
                                          with_grad=True), torch.float32)
    g = torch.Generator(device="cuda").manual_seed(1)
    inp = {"t": torch.rand(n, 1, device="cuda", generator=g), "x": torch.rand(n, 1, device="cuda", generator=g) * 2 - 1}
    params = m.engine_params()
    grads = torch.zeros_like(params)
    return plan, inp, params, grads


def _call(s):
    plan, inp, params, grads = s
    plan.loss_fwd_bwd(inp, params, grads, label_consts={"ac": 0.0})


def _profiled(s, steps: int) -> dict:
    plan = s[0]
    plan.set_profile(True)
    acc = {}
    for _ in range(steps):
        _call(s)
        for k, v in plan.get_profile().items():
            acc[k] = acc.get(k, 0.0) + v["ms"]
    plan.set_profile(False)
    return {k: v / steps for k, v in acc.items()}


def _timed(s, steps: int) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        _call(s)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--points", type=int, default=1 << 18)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("omega_dw_timing needs an H100: the engine has no CPU fallback")
    plans = {"fixed": _setup(False, args.points), "trainable": _setup(True, args.points)}
    for s in plans.values():  # warm-up: module loads, workspaces
        for _ in range(3):
            _call(s)
    torch.cuda.synchronize()
    rows = {k: [] for k in plans}
    gpu_before = _gpu_info()
    for _ in range(args.rounds):
        for name, s in plans.items():
            prof = _profiled(s, args.steps)
            rows[name].append({"thin_dw_ms": prof["thin_dw"], "misc_ms": prof["misc"], "profiled_total_ms": sum(prof.values()),
                               "call_ms": _timed(s, args.steps)})
    out = {"gpu_before": gpu_before, "gpu_after": _gpu_info(), "points": args.points, "steps": args.steps, "rounds": rows}
    med = lambda xs: sorted(xs)[len(xs) // 2]  # noqa: E731
    summ = {}
    for name in plans:
        summ[name] = {k: med([r[k] for r in rows[name]]) for k in rows[name][0]}
    f, t = summ["fixed"], summ["trainable"]
    summ["thin_dw_extra_ms"] = t["thin_dw_ms"] - f["thin_dw_ms"]
    summ["thin_dw_extra_pct_of_thin_dw"] = 100.0 * summ["thin_dw_extra_ms"] / f["thin_dw_ms"]
    summ["extra_pct_of_call"] = 100.0 * (t["profiled_total_ms"] - f["profiled_total_ms"]) / f["profiled_total_ms"]
    out["median"] = summ
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
