"""Device time of the wgmma weight-gradient kernel (k_wg_dw) in one training call of the benchmark's plans, and its SM
cycles per chunk.

Builds the plan of ``bench.py --config 3`` (LDC Navier-Stokes, MLP 2 -> 256 x 6 -> 3, 5 jet channels, 2^20 points) and
of ``--config 2`` (Allen-Cahn, MLP 2 -> 128 x 4 -> 1, 4 jet channels, 2^18 points) and times one loss + weight-gradient
call of each with the library's per-launch CUDA-event profile on.  Reported per plan: the ``dw_gemm`` class (the
k_wg_dw launches) as the median over ``--rounds`` rounds of ``--steps`` calls, the launches per call, and SM cycles per
chunk = launch time x SM clock / chunks of the busiest CTA.  The chunk count follows the engine's launch geometry
(engine.cu, dW on the tensor cores): column blocks of at most dw_maxq(C) x 32 columns, fan-in blocks of 128 rows, and the
chunks of dw_pch(C) points split over the SMs the tiles leave.  The SM clock is sampled with nvidia-smi while the rounds
run; the GPU's name and power limit are read in the same run.

    python tools/wg_dw_timing.py [--configs 3,2] [--steps 10] [--rounds 5] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import ppsci  # noqa: E402

# the kernel's geometry (kernels_wgmma.cuh)
DW_TK = 128


def dw_pch(C: int) -> int:
    return 4 if C >= 8 else 8 if C >= 3 else 32 // C


def dw_maxq(C: int) -> int:
    return 4 if C <= 6 else 2 if C <= 8 else 1


def _gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"
    try:
        line = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              check=True).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in line.split(",")]))
    except (OSError, subprocess.CalledProcessError, IndexError):
        return {"name": torch.cuda.get_device_name(0)}


class _ClockSampler:
    """SM clock in MHz every 50 ms, from a child nvidia-smi that is stopped before the tool returns."""

    def __init__(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0",
                                          "-lms", "50"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except OSError:
            self.proc = None

    def stop(self):
        if self.proc is None:
            return []
        self.proc.terminate()
        out, _ = self.proc.communicate(timeout=10)
        return [int(float(v)) for v in out.split() if v.replace(".", "").isdigit()]


def _setup(cfg: int):
    """The plan bench.py builds for config ``cfg`` (same model, equation and point count; the constraint goes through
    ExpressionSolver as there), seeded inputs on the device and zero labels."""
    torch.manual_seed(0)
    g = torch.Generator(device="cuda").manual_seed(1)
    if cfg == 3:
        n = 1 << 20
        m = ppsci.arch.MLP(("x", "y"), ("u", "v", "p"), 6, 256, "tanh")
        equation = ppsci.equation.NavierStokes(0.01, 1.0, 2, False)
        inp = {"x": torch.rand(n, 1, device="cuda", generator=g), "y": torch.rand(n, 1, device="cuda", generator=g)}
    elif cfg == 2:
        n = 1 << 18
        m = ppsci.arch.MLP(("t", "x"), ("u",), 4, 128, "tanh", periods={"x": (2.0, False)})
        equation = ppsci.equation.AllenCahn(0.01)
        inp = {"t": torch.rand(n, 1, device="cuda", generator=g), "x": torch.rand(n, 1, device="cuda", generator=g) * 2 - 1}
    else:
        raise SystemExit(f"config {cfg}: only the MLP configs 2 and 3 are timed here")
    m = m.to("cuda")

    class _Cst:
        name = "EQ"
        loss = ppsci.loss.MSELoss("mean")
        output_expr = dict(equation.equations)
        output_keys = tuple(equation.equations.keys())

    plan = ppsci.utils.ExpressionSolver().compiled_for(m, _Cst(), None).plan(torch.float32)
    params = m.engine_params()
    grads = torch.zeros_like(params)
    return {"plan": plan, "inp": inp, "params": params, "grads": grads, "labels": {k: 0.0 for k in _Cst.output_keys},
            "n": n, "widths": list(m.net_spec().widths)}


def _call(s):
    s["plan"].loss_fwd_bwd(s["inp"], s["params"], s["grads"], label_consts=s["labels"])


def _chunks_per_cta(s) -> int:
    """Chunks of the busiest CTA summed over one call's k_wg_dw launches (hidden layers 256 -> 256 etc.; the thin first
    and last layers do not run on this kernel)."""
    plan, widths = s["plan"], s["widths"]
    C, sms, cp = plan.channels, torch.cuda.get_device_properties(0).multi_processor_count, plan.chunk_points
    total = 0
    for start in range(0, s["n"], cp):
        nc = min(cp, s["n"] - start)
        for l in range(2, len(widths)):
            K, N = widths[l - 1], widths[l]
            if K % 4 or N % 32 or not 32 <= N <= 256:
                continue
            nq = N // 32
            ncb = (nq + dw_maxq(C) - 1) // dw_maxq(C)
            tiles = (K + DW_TK - 1) // DW_TK * ncb
            chunks = (nc + dw_pch(C) - 1) // dw_pch(C)
            want = min(max(sms // tiles, 1), chunks)
            total += (chunks + want - 1) // want
    return total


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--configs", default="3,2")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wg_dw_timing needs an H100: the engine has no CPU fallback")
    out = {"gpu": _gpu_info(), "configs": {}}
    med = lambda xs: sorted(xs)[len(xs) // 2]  # noqa: E731
    for cfg in (int(c) for c in args.configs.split(",")):
        s = _setup(cfg)
        for _ in range(3):  # warm-up: module loads, workspaces
            _call(s)
        torch.cuda.synchronize()
        plan = s["plan"]
        plan.set_profile(True)
        sampler = _ClockSampler()
        rounds, launches = [], 0
        try:
            for _ in range(args.rounds):
                ms = 0.0
                for _ in range(args.steps):
                    _call(s)
                    p = plan.get_profile()["dw_gemm"]
                    ms += p["ms"]
                    launches = p["launches"]
                rounds.append(ms / args.steps)
        finally:
            clocks = sampler.stop()
            plan.set_profile(False)
        dw_ms = med(rounds)
        mhz = med(clocks) if clocks else None
        cpc = _chunks_per_cta(s)
        out["configs"][cfg] = {
            "dw_gemm_ms": round(dw_ms, 3), "dw_gemm_ms_rounds": [round(r, 3) for r in rounds], "launches": launches,
            "chunks_per_cta_per_call": cpc, "sm_mhz_median": mhz, "sm_mhz_min_max": [min(clocks), max(clocks)] if clocks else None,
            "sm_cycles_per_chunk": round(dw_ms * 1e-3 * mhz * 1e6 / cpc) if mhz and cpc else None,
        }
        del s
        torch.cuda.empty_cache()
    out["gpu_after"] = _gpu_info()
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
