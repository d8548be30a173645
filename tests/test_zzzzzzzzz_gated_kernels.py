"""GPU sweep of the gated networks' kernels (ModifiedMLP and PirateNet: k_gate_fwd / k_gate_bwd, k_mix_fwd / k_mix_bwd,
and the GEMM modes only gated plans use) one pass at a time, against the fp64 reference of tests/gated_ref.py on the
values each kernel read.

Each case runs ``gated_ref.run_case``: a call with PPSCI_B200_KEEP_ADJOINTS set checks every forward, adjoint and
gradient pass; a default call on a workspace of NaN bytes must give the same planes bitwise and a gradient within the
same bars; ``plan.forward`` the same Y; some cases also seed the gradient buffer or run over three workspace chunks.
The kernels each case launched are read from torch.profiler: the gates (and the mixes of an embedding layer or a
PirateNet) must have run in the case's dtype.  Run with -s for the per-pass error table."""
import re

import pytest
import torch

from tests.gated_ref import Case, run_case
from tests.layer_ref import all_layouts

pytestmark = pytest.mark.gpu

F32, F64 = torch.float32, torch.float64
U = {F32: 2.0 ** -24, F64: 2.0 ** -53}
# Bars per pass in units of the componentwise bound (forward, dW, db, d alpha, d omega) or of the plane's largest |ref|
# (dx, Zubar, Zvbar, Xres), about twice the largest error measured over this file's matrix on an H100 80GB HBM3 (700 W
# power limit):
#   fp32 (units of 2^-24): fwd 10.6, gate 5.7 (sigmoid 875: below), mix 4.6, dx 75.1 (after siren), Zubar 11.6,
#        Xres 8.9, dW 39.1 (70,001 points), db 23.9, d alpha 1.2, d omega 0.005;
#   fp64 (units of 2^-53): fwd 6.5, gate 7.0, mix 5.7, dx 6.6, Zubar 9.1, Xres 0 (the fp64 dx GEMM and the reference
#        sum in the same order; the emulation measured 3.1), dW 34.7 (seeded), db 24.6 (seeded), d alpha 1.6,
#        d omega 0.06.
# The fp32 sigmoid's closed-form Taylor coefficients are polynomials in sigma that cancel near z = 0; inside a GEMM the
# fan-in dilutes that rounding (tests/test_zzzzzz_layer_kernels.py), in a gate it stands alone, so sigmoid's fp32 gates
# have a bar of their own.  A dropped cross term, gate contribution or residual path is off by 2^20 units or more.
BAR = {F32: {"fwd": 22.0, "gate": 12.0, "gate:sigmoid": 1750.0, "mix": 10.0, "dx": 150.0, "zub": 24.0, "xres": 18.0,
             "dw": 80.0, "db": 48.0, "alpha": 2.5, "omega": 0.05},
       F64: {"fwd": 13.0, "gate": 14.0, "mix": 12.0, "dx": 14.0, "zub": 19.0, "xres": 4.0, "dw": 70.0, "db": 50.0,
             "alpha": 3.2, "omega": 0.12}}

ACTS = ["tanh", "sin", "cos", "sigmoid", "silu", "identity", "relu", "gelu", "elu", "selu", "leaky_relu", "siren"]
P_TRAIN = (("x", 2.0, True),)
P_FIX = (("x", 2.0, False),)


def _kind(k, H, E=None):
    """(gated, hidden, act_first): "M3" / "M5" ModifiedMLP with 3 / 5 linear layers, "ME" ModifiedMLP behind a sin
    embedding layer of width E, "P1" .. "P3" PirateNet with 1 .. 3 blocks."""
    if k == "M3":
        return 1, (H, H), None
    if k == "M5":
        return 1, (H,) * 4, None
    if k == "ME":
        return 1, (E or H + 2, H, H), "sin"
    return 2, (H,) * (1 + 3 * int(k[1])), "sin"


def _c(kind, layout, H=64, n=3013, dtype=F32, E=None, **kw):
    g, hidden, af = _kind(kind, H, E)
    return Case(layout, g, hidden, n, dtype, act_first=af, **kw)


def _cases():
    out = []
    kinds = ["M3", "ME", "P1", "M5", "P2", "P3"]
    for i, lay in enumerate(sorted(all_layouts())):  # every C: 1, 2, 3, 4, 5, 7, 8, 17, 29, 32 (KMAX 1 / 2 / 4, GATE_MAXC)
        out += [_c(kinds[i % 6], lay, dtype=F32), _c(kinds[(i + 3) % 6], lay, dtype=F64)]
    # every activation without a trainable parameter, through gates and mixes
    out += [_c(["M3", "P1", "ME"][i % 3], "Lay22", dtype=F32, act=a) for i, a in enumerate(ACTS)]
    out += [_c(k, "O3", dtype=F64, act=a) for k, a in (("P1", "sin"), ("M3", "sigmoid"), ("ME", "gelu"), ("P2", "siren"))]
    # widths: pitch != width, past one column tile (TN = 128 fp32 / 64 fp64), 256
    for H in (18, 50, 130, 256):
        out += [_c("M5", "Lay22", H=H, dtype=F32), _c("P1", "Lay12", H=H, dtype=F64), _c("ME", "Lay12", H=H, E=H + 6)]
    # alpha: 0 (the reference's start: Zbar of a block's third layer exactly 0), 1, negative, per block
    for dt in (F32, F64):
        out += [_c("P1", "Lay22", dtype=dt, alphas=(0.0,)), _c("P2", "Lay12", dtype=dt, alphas=(0.0, 0.0)),
                _c("P2", "Lay22", dtype=dt, alphas=(1.0, 1.0)), _c("P1", "O4", dtype=dt, alphas=(-0.7,)),
                _c("P3", "Lay22", dtype=dt, alphas=(0.3, -0.5, 1.2))]
    # periods: fixed and trainable; ModifiedMLP without an embedding reads the seeds in three GEMMs (three d omega consumers)
    for dt in (F32, F64):
        out += [_c("M3", "Lay12", dtype=dt, periods=P_TRAIN), _c("M5", "Lay22", dtype=dt, periods=P_FIX),
                _c("ME", "Lay12", dtype=dt, periods=P_TRAIN), _c("P2", "Lay12", dtype=dt, periods=P_TRAIN)]
    # point counts: 1, 127 / 128 / 129 around a 128-thread block, 70,001 (k_mix_bwd's grid-stride loop over a grid
    # capped at 8 CTAs per SM: n H > 135,168 on 132 SMs, so from 3,013 points at H = 64; many d alpha partials)
    for n in (1, 127, 128, 129):
        out += [_c("P2", "Lay22", n=n, dtype=F32), _c("M3", "O4", n=n, dtype=F64)]
    for dt in (F32, F64):
        out += [_c("P2", "Lay22", n=70001, dtype=dt, alphas=(0.4, -0.3)), _c("ME", "Lay12", n=70001, dtype=dt)]
    out += [_c("M3", "O4x7_3", H=32, n=70001, dtype=F32)]
    # three workspace chunks; the gradient buffer seeded
    for dt in (F32, F64):
        out += [_c("M3", "Lay22", dtype=dt, chunked=True, seeded=True, periods=P_TRAIN),
                _c("ME", "O3", dtype=dt, chunked=True, seeded=True),
                _c("P2", "Lay12", dtype=dt, chunked=True, seeded=True, periods=P_TRAIN, alphas=(0.4, -0.3)),
                _c("P3", "Lay4444", dtype=dt, chunked=True, seeded=True, alphas=(0.0, 0.5, -1.5))]
    seen = []
    for c in out:
        if c not in seen:
            seen.append(c)
    return seen


CASES = _cases()
SEEN = set()
_KERNEL = re.compile(r"k_(gate|mix)_(fwd|bwd)<(float|double), (\d)>")


def _launched(names):
    """{(kernel, dtype, KMAX)} of the gate / mix instances in the profiler's kernel names."""
    out = set()
    for nm in names:
        m = _KERNEL.search(nm)
        if m:
            out.add((f"k_{m[1]}_{m[2]}", "f32" if m[3] == "float" else "f64", int(m[4])))
    return out


def _bar(bars, key, act):
    kind = key.split("@")[0].split(":")[0]
    return bars.get(f"{kind}:{act}", bars.get(kind, 0.0))


def _check(name, e, dtype, act):
    e = {k: v / U[dtype] for k, v in e.items()}
    for k in sorted(e):
        print(f"[gated-kernels] {name} {k} {e[k]:.3f}", flush=True)
    bars = BAR[dtype]
    bad = {k: v for k, v in e.items() if not v <= _bar(bars, k, act)}
    assert not bad, f"{name}: {bad} (bars {bars})"


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_gated_kernels(case):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        e = run_case(case, device="cuda:0")
        torch.cuda.synchronize()
    ran = _launched({ev.key for ev in prof.key_averages()})
    dt = "f64" if case.dtype == F64 else "f32"
    want = {"k_gate_fwd", "k_gate_bwd"} | ({"k_mix_fwd", "k_mix_bwd"} if case.act_first or case.gated == 2 else set())
    got = {k for k, d, _ in ran if d == dt}
    assert want <= got, f"{case.name}: {sorted(want - got)} did not run; launched {sorted(ran)}"
    SEEN.update(ran)
    _check(case.name, e, case.dtype, case.act)


def test_every_kernel_ran():
    """Across the matrix above: k_gate_fwd / k_gate_bwd / k_mix_fwd / k_mix_bwd in f32 and f64 at KMAX 1, 2 and 4."""
    if not SEEN:
        pytest.skip("the sweep did not run in this session")
    want = {(f"k_{k}_{p}", d, m) for k in ("gate", "mix") for p in ("fwd", "bwd") for d in ("f32", "f64") for m in (1, 2, 4)}
    assert want <= SEEN, sorted(want - SEEN)
