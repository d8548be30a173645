"""The gated networks' kernels one pass at a time (ModifiedMLP and PirateNet: k_gate_fwd / k_gate_bwd, k_mix_fwd /
k_mix_bwd, and the GEMM modes only gated plans use), through the CPU emulation build of the kernel sources, against
the fp64 reference of tests/gated_ref.py on the exact values each kernel read.

Each case runs ``gated_ref.run_case``: a call with PPSCI_B200_KEEP_ADJOINTS set checks every forward, adjoint and
gradient pass; a default call on a workspace of NaN bytes must give the same planes bitwise and a gradient within the
same bars; ``plan.forward`` the same Y.  Some cases also seed the gradient buffer or run over three workspace chunks.
The emulation has 4 SMs, so k_mix_bwd's capped grid (8 CTAs per SM) loops once n H > 4,096.  The emulation runs every
CUDA thread as an OS thread, so the shapes stay small; tests/test_zzzzzzzzz_gated_kernels.py sweeps the wide ones on
the GPU."""
import pytest
import torch

from paddlescience_b200.engine import binding as B
from tests.emul.build_emul import build
from paddlescience_b200.engine.compiler import compile_residuals
from paddlescience_b200.engine.plan import ResidualPlan
from tests.cases import make_net
from tests.gated_ref import Case, run_case
from tests.layer_ref import all_layouts

F32, F64 = torch.float32, torch.float64
U = {F32: 2.0 ** -24, F64: 2.0 ** -53}
# Bars in units of the componentwise bound (forward, dW, db, d alpha, d omega) or of the plane's largest |ref| (dx,
# Zubar, Zvbar, Xres): about twice the largest error this file's matrix measured, in units of 2^-53 (fp64) and 2^-24
# (fp32): fp64 fwd 3.9, gate 3.8, mix 4.3, dx 12.3 (C = 17), Zubar 8.6, Xres 3.1, dW 15.8 (H = 130), db 4.3, d alpha
# 0.45, d omega 0.09; fp32 fwd 5.7, gate 2.9, mix 3.6, dx 10.6, Zubar 9.7, Xres 3.2, dW 8.7 (H = 256), db 3.2, d alpha
# 0.46, d omega 0.03.  A dropped cross term, gate contribution or residual path is off by 2^20 units or more in fp64.
BAR = {F64: {"fwd": 8.0, "gate": 8.0, "mix": 9.0, "dx": 25.0, "zub": 18.0, "xres": 7.0, "dw": 32.0, "db": 9.0,
             "alpha": 1.0, "omega": 0.2},
       F32: {"fwd": 12.0, "gate": 6.0, "mix": 8.0, "dx": 22.0, "zub": 20.0, "xres": 7.0, "dw": 18.0, "db": 7.0,
             "alpha": 1.0, "omega": 0.1}}

ACTS = ["tanh", "sin", "cos", "sigmoid", "silu", "identity", "relu", "gelu", "elu", "selu", "leaky_relu", "siren"]
P_TRAIN = (("x", 2.0, True),)
P_FIX = (("x", 2.0, False),)


def _kind(k, H, E=None):
    """(gated, hidden, act_first) of a kind: "M3" / "M5" ModifiedMLP with 3 / 5 linear layers, "ME" ModifiedMLP behind
    a sin embedding layer of width E, "P1" .. "P3" PirateNet with 1 .. 3 blocks."""
    if k == "M3":
        return 1, (H, H), None
    if k == "M5":
        return 1, (H,) * 4, None
    if k == "ME":
        return 1, (E or H + 2, H, H), "sin"
    return 2, (H,) * (1 + 3 * int(k[1])), "sin"


def _c(kind, layout, H=12, n=37, dtype=F64, E=None, **kw):
    g, hidden, af = _kind(kind, H, E)
    return Case(layout, g, hidden, n, dtype, act_first=af, **kw)


def _cases():
    out = []
    kinds = ["M3", "ME", "P1", "M5", "P2", "P3"]
    for i, lay in enumerate(sorted(all_layouts())):  # every layout: C = 1 .. 32, KMAX 1 / 2 / 4, GATE_MAXC
        n = 17 if all_layouts()[lay]["C"] > 8 else 29
        out.append(_c(kinds[i % 6], lay, n=n, dtype=(F64, F32)[i % 2]))
    for i, a in enumerate(ACTS):  # every activation without a trainable parameter, gates and mixes
        out.append(_c(["M3", "P1", "ME"][i % 3], "O2", n=17, dtype=(F32, F64)[i % 2], act=a))
    out += [
        # widths: pitch != width, past one column tile (TN = 64 / 128), 256; k_mix_bwd's grid-stride loop (n H > 4,096)
        _c("M3", "Lay22", H=18, n=23), _c("P1", "O3", H=50, n=17, dtype=F32), _c("ME", "O11", H=64, E=18, n=17),
        _c("P1", "Lay12", H=130, n=37, dtype=F32), _c("P1", "O2", H=130, n=37), _c("M5", "O1", H=256, n=17, dtype=F32),
        # alpha: 0 (the reference's start: Zbar of the block's third layer exactly 0), 1, negative, per block
        _c("P1", "Lay12", alphas=(0.0,)), _c("P2", "O3", dtype=F32, alphas=(0.0, 0.0)), _c("P2", "Lay22", alphas=(1.0, 1.0)),
        _c("P1", "O4", dtype=F32, alphas=(-0.7,)), _c("P3", "O2", n=17, alphas=(0.3, -0.5, 1.2)),
        # periods: fixed and trainable; ModifiedMLP without an embedding: three d omega consumers
        _c("M3", "Lay12", periods=P_TRAIN), _c("M5", "Lay12", dtype=F32, periods=P_TRAIN),
        _c("ME", "Lay12", periods=P_TRAIN), _c("P2", "Lay12", dtype=F32, periods=P_FIX),
        # point counts: one, and past one 128-thread block
        _c("M3", "O2", n=1), _c("P1", "O2", n=1, dtype=F32), _c("ME", "O2", n=129, dtype=F32),
        # three workspace chunks; the gradient buffer seeded
        _c("M3", "Lay22", chunked=True, seeded=True), _c("ME", "O3", dtype=F32, chunked=True, seeded=True),
        _c("P2", "Lay12", chunked=True, seeded=True, periods=P_TRAIN, alphas=(0.4, -0.3)),
        _c("P3", "O4x7", n=17, dtype=F32, chunked=True, seeded=True, alphas=(0.0, 0.5, -1.5)),
    ]
    seen = []
    for c in out:
        if c not in seen:
            seen.append(c)
    return seen


CASES = _cases()


@pytest.fixture(scope="module")
def emul_lib():
    return B.Library(build())


def _check(name, e, dtype):
    u = U[dtype]
    e = {k: v / u for k, v in e.items()}
    print(f"\n[gated-kernels emul] {name}: " + " ".join(f"{k}={v:.2f}" for k, v in sorted(e.items())))
    bars = BAR[dtype]
    bad = {k: v for k, v in e.items() if not v <= bars.get(k.split("@")[0].split(":")[0], 0.0)}
    assert not bad, f"{name}: {bad} (bars {bars})"


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_gated_kernels_emulated(emul_lib, case):
    e = run_case(case, library=emul_lib, device="cpu")
    L = len(case.hidden) + 1
    want = {f"fwd:Z{l}" for l in range(1, L)} | {f"dx:Zbar{l}" for l in range(1, L)} | {"fwd:Y", "zub:u", "zub:v"}
    want |= {f"dw:W{l}" for l in range(1, L + 1)} | {"dw:Wu", "dw:Wv", "db:bu", "db:bv"}
    if case.gated == 2:
        want |= {"xres"} | {f"alpha:{b}" for b in range((L - 2) // 3)}
    if case.periods and any(t for _, _, t in case.periods):
        want.add("omega")
    assert want <= set(e), sorted(want - set(e))
    _check(case.name, e, case.dtype)


@pytest.mark.parametrize("gated", [1, 2])
@pytest.mark.parametrize("act", ["stan", "swish_b"])
def test_gated_plans_refuse_trainable_activations(emul_lib, gated, act):
    spec = all_layouts()["O2"]
    net = make_net(spec["in_keys"], spec["out_keys"], (12,) * 4, act, gated=gated)
    net.act_first = "sin"
    cr = compile_residuals(net, spec["exprs"]())
    with pytest.raises(B.EngineError, match="trainable parameter"):
        ResidualPlan(cr, F64, backend=1, library=emul_lib)
