"""GPU sweep of the wgmma kernels one layer at a time: k_wg_layer (forward and dx) and k_wg_dw (weight and bias
gradient) against the fp64 reference of tests/layer_ref.py, evaluated on the fp32 values each kernel read from the
workspace after one fused call.  An error therefore belongs to one kernel of one layer, and is measured element by
element against the componentwise bound (units of 2^-24 |A| |W|), not diluted in a global rel-L2.

The layer under test is layer 2 of a two-hidden-layer fp32 plan (K = widths[1], N = widths[2]) on one equation per
compile-time jet layout (LayV C = 1, Lay12 C = 4, Lay22 C = 5, Lay222 C = 7, Lay4444 C = 17).  The matrix reaches every
forward / dx column count (NQ 1..8) and K-chunk count, every dW column-block width and block count, fan-ins that put
the dW alone on the tensor cores with a partial 8-row group, a 1024-long contraction, ragged point counts and every
activation without a trainable parameter.  Every case also runs with backend=1 (CUDA-core fp32 kernels) and prints
"case kernel e_tc e_cc" beside each other; run with -s to see the table."""
import pytest
import torch

from oracle import ppsci_oracle as O
from paddlescience_b200.engine.compiler import NetSpec, compile_residuals
from paddlescience_b200.engine.plan import ResidualPlan
from tests.layer_ref import U32, check_layer, layouts, param_blocks, run_fused, stash_views

pytestmark = pytest.mark.gpu

# Bars in units of 2^-24 of the componentwise bound (fwd, dW, db) or of the plane's largest |ref| (dx), about twice the
# largest error measured over this file's matrix with the 3xTF32 kernels on an H100 80GB HBM3 (700 W power limit):
# fwd 35.0 (Lay4444, K = 1024), dx 33.9 (Lay4444, sigmoid), dW 53.1 (Lay22, 70,001 points), db 10.3; accumulated onto
# a seeded gradient, dW 48.8 and db 6.2 in units of 2^-24 (|A| |Zbar| + |G0|).  The CUDA-core kernels measured up to
# 27.9, 35.1, 141.1 and 22.0 (19.5 and 14.1 accumulated) on the same cases.  The dropped A_lo B_lo term alone is worth
# up to ~4 units; a lost cross term shows at ~2^13.
BAR = {"fwd": 70.0, "dx": 70.0, "dw": 110.0, "db": 22.0}
BAR_ACC = {"acc_dw": 100.0, "acc_db": 12.0}

LAYOUT_C = {k: v["C"] for k, v in layouts().items()}
ACTS = ["tanh", "sin", "cos", "sigmoid", "silu", "identity", "relu", "gelu", "elu", "selu", "leaky_relu", "siren"]
SHAPES = [(32, 256), (64, 32), (96, 160), (128, 128), (160, 96), (192, 224), (224, 192), (256, 64)]
DW_ONLY = [(36, 64), (100, 224), (260, 96)]  # fan-ins that are not multiples of 32: only the dW is on wgmma


def dw_pch(C):  # points per k_wg_dw chunk (kernels_wgmma.cuh)
    return 4 if C >= 8 else 8 if C >= 3 else 32 // C


def point_counts(C):
    """1 and 3 points, one point into the second forward tile, a partial last dW chunk past the p+1..p+3 guards of the
    B loads, several persistent passes (3013) and many (70001)."""
    return sorted({1, 3, 64 // C + 1, 4 * dw_pch(C) + 3, 3013, 70001})


def _shape_ok(K, N):
    return K % 32 == 0 and 32 <= K <= 1024 and N % 32 == 0 and 32 <= N <= 256


def wg_kinds(widths, l, dense=False):
    """Passes of layer l that must run on the wgmma kernels of an fp32, ungated plan with a wgmma jet layout and an
    activation without a parameter (wg_fwd_ok / wg_dx_ok / wg_dw_ok of kernels_wgmma.cuh, restated)."""
    K, N = widths[l - 1], widths[l]
    out = set()
    if l >= 2 and _shape_ok(K, N) or l == 1 and dense and K % 4 == 0 and _shape_ok((K + 31) // 32 * 32, N):
        out.add("fwd")
    if l >= 2 and _shape_ok(N, K):
        out.add("dx")
    if (l >= 2 or dense) and K % 4 == 0 and N % 32 == 0 and 32 <= N <= 256:
        out.add("dw")
    return out


def _layer_case_ids():
    cases = []
    for lay in sorted(LAYOUT_C):
        for K, N in SHAPES + DW_ONLY:
            cases.append((lay, K, N, 3013, "tanh", None))
        for K, N in [(128, 128), (192, 224)]:
            cases += [(lay, K, N, n, "tanh", None) for n in point_counts(LAYOUT_C[lay])]
    cases += [(lay, 1024, 256, 3013, "tanh", None) for lay in ("Lay22", "Lay4444")]
    for act in ACTS:
        cases += [("Lay22", 128, 128, 3013, act, None), ("Lay4444", 64, 96, 3013, act, None)]
    cases.append(("Lay22", 64, 128, 3013, "tanh", "sin"))
    out = []
    for c in cases:  # first occurrence of each case
        if c not in out:
            out.append(c)
    return out


LAYER_CASES = _layer_case_ids()


def _cid(c):
    lay, K, N, n, act, first = c
    return f"{lay}-K{K}-N{N}-n{n}-{act}" + (f"-first_{first}" if first else "")


def _report(case, e_tc, e_cc):
    for k in sorted(e_tc):
        print(f"[tc-layers] {case} {k} e_tc={e_tc[k]:.3f} e_cc={e_cc.get(k, float('nan')):.3f}", flush=True)


def _errors(plan, params, grads, views, checks, seed=None, x_dense=None):
    e = {}
    for l, kinds in checks.items():
        for k, v in check_layer(plan, views, params, grads, l, kinds, seed=seed, x_dense=x_dense).items():
            e[f"{k}{l}"] = v / U32
    return e


def _assert_bars(case, e, bars):
    bad = {k: v for k, v in e.items() if not v <= bars[k.rstrip("0123456789")]}
    assert not bad, f"{case}: {bad} (bars {bars})"


@pytest.mark.parametrize("case", LAYER_CASES, ids=[_cid(c) for c in LAYER_CASES])
def test_wgmma_layer_kernels(case):
    lay, K, N, n, act, first = case
    name = _cid(case)
    runs = {}
    for backend in (2, 1):
        plan, params, grads, views = run_fused(lay, [K, N], n, act=act, act_first=first, backend=backend)
        widths = plan.compiled.net.widths
        L = len(widths) - 1
        # layer 2: every pass that must be on wgmma; the other wgmma layers: their forward
        checks = {l: (wg_kinds(widths, l) if l == 2 else wg_kinds(widths, l) & {"fwd"}) for l in range(2, L + 1)}
        checks = {l: ks for l, ks in checks.items() if ks}
        if backend == 2:
            assert plan.uses_tcgen05, "tensor-core backend was not selected"
            assert checks.get(2), f"{name}: no pass of layer 2 is eligible for the wgmma kernels"
        runs[backend] = _errors(plan, params, grads, views, checks)
        del plan, views
    _report(name, runs[2], runs[1])
    _assert_bars(name, runs[2], BAR)


def _dense_run(num_loc, n, backend, seed=0):
    """DeepONet's branch net as arch/deeponet.py builds it: the caller's [n, num_loc] matrix as a dense first-layer
    operand, widths [num_loc, 128, 128], values_fwd_bwd with seeded output adjoints."""
    torch.manual_seed(seed)
    widths = [num_loc, 128, 128]
    net = NetSpec(("u",), tuple(f"f{i}" for i in range(128)), [], [], [], widths, "tanh", dense_in=True)
    plan = ResidualPlan(compile_residuals(net, {}, with_grad=False), torch.float32, [], [], backend=backend)
    params = O.xavier_uniform_params(widths, 1, torch.float64)
    params = (params + 0.1 * torch.randn_like(params)).float().cuda()
    x = torch.rand(n, num_loc, dtype=torch.float64).float().cuda()
    ybar = (torch.randn(n, 128, dtype=torch.float64) / n).float().cuda()
    grads = torch.zeros_like(params)
    plan.values_fwd_bwd({"u": x}, params, grads, ybar)
    return plan, params, grads, x, stash_views(plan, n)


@pytest.mark.parametrize("num_loc", [4, 100, 1000])
def test_wgmma_dense_first_layer_and_wide_output(num_loc):
    """L = 2 and every pass on wgmma: the dense layer-1 forward (contraction padded to a multiple of 32 with zero
    columns), the 128-wide output forward (Y), dW_2 from the seeded output adjoints, the dx into Zbar_1 (buffer 0)
    and the dense dW_1."""
    n = 3013
    name = f"dense-nloc{num_loc}-n{n}"
    runs = {}
    for backend in (2, 1):
        plan, params, grads, x, views = _dense_run(num_loc, n, backend)
        widths = plan.compiled.net.widths
        checks = {1: wg_kinds(widths, 1, dense=True), 2: wg_kinds(widths, 2)}
        if backend == 2:
            assert plan.uses_tcgen05
            assert checks == {1: {"fwd", "dw"}, 2: {"fwd", "dx", "dw"}}, checks
            # the seeded adjoints are what the dW_2 reads
            assert float(views["Ybar"].abs().max()) > 0
        runs[backend] = _errors(plan, params, grads, views, checks, x_dense=x)
        del plan, views
    _report(name, runs[2], runs[1])
    _assert_bars(name, runs[2], BAR)


@pytest.mark.parametrize("layout", sorted(LAYOUT_C))
def test_wgmma_dw_accumulates(layout):
    """The C-ABI accumulates into grads (k_wg_dw adds its split point ranges with atomics): seeded with G0, the call
    must leave G0 + dW.  Checked for the wgmma blocks against the reference, the others against a zero-seeded run."""
    K, N, n = 192, 224, 3013
    name = f"acc-{layout}-K{K}-N{N}-n{n}"
    runs = {}
    for backend in (2, 1):
        plan0, _, g1, _ = run_fused(layout, [K, N], n, backend=backend)
        del plan0
        gen = torch.Generator().manual_seed(7)
        g0 = (torch.randn(g1.numel(), generator=gen, dtype=torch.float64) * float(g1.double().std())).float().cuda()
        plan, params, grads, views = run_fused(layout, [K, N], n, backend=backend, grads0=g0)
        if backend == 2:
            assert plan.uses_tcgen05
        e = _errors(plan, params, grads, views, {2: {"dw"}}, seed=g0)
        runs[backend] = {"acc_" + k: v for k, v in e.items()}
        # every other block (CUDA-core kernels): G0 plus what a zero-seeded call computes; an overwritten block is off
        # by |G0|
        for l, (w_sl, b_sl, _) in enumerate(param_blocks(plan.compiled.net.widths), start=1):
            for sl in ((w_sl, b_sl) if l != 2 else ()):
                d = (grads[sl].double() - g0[sl].double() - g1[sl].double()).norm()
                assert float(d) <= 1e-5 * float(g0[sl].double().norm() + g1[sl].double().norm()), (name, l)
        del plan, views
    _report(name, runs[2], runs[1])
    _assert_bars(name, runs[2], BAR_ACC)

