"""GPU checks of unsteady 2-D Navier-Stokes on (t, x, y): the jet layout (t: 1, x: 2, y: 2), C = 6, that
NavierStokes(nu, rho, 2, time=True) compiles to (Lay122 of csrc/jet_layout.cuh).

* Layer by layer against the fp64 reference of tests/layer_ref.py on the values each kernel read after one fused call:
  the vectorised thin first and last layers (k_first_fwd_v / k_first_dw_v / k_last_fwd_v / k_last_bwd_v, backend=1),
  and k_wg_layer (forward, dx) and k_wg_dw on layer 2 at widths 32..256, at point counts up to 70,001 including a call
  of several workspace chunks.  The kernels each call launched are read from torch.profiler.  Bars are those of
  tests/test_zzzzzz_layer_kernels.py (thin) and tests/test_gpu_tc_layers.py (wgmma).
* The whole call against the fp64 oracle: the 6 x 256 plan on the tensor cores and the unsteady cavity example's 9 x 50
  plan in fp32 and fp64, at the bars of the named shapes.

The layout's equation is added to layer_ref's table and thin-layout set for the duration of each test only."""
import pytest
import torch

from oracle import ppsci_oracle as O
from tests import layer_ref
from tests.cases import run_case
from tests.layer_ref import U32, all_errors, check_layer, run_fused, thin_kernels

pytestmark = pytest.mark.gpu

THIN_BAR = {"fwd": 28.0, "dx": 92.0, "dw": 88.0, "db": 80.0}  # tests/test_zzzzzz_layer_kernels.py, fp32
WG_BAR = {"fwd": 70.0, "dx": 70.0, "dw": 110.0, "db": 22.0}  # tests/test_gpu_tc_layers.py


def _ns2t():
    return O.navier_stokes_expr(0.01, 1.0, 2, True)


LAY122 = dict(in_keys=("t", "x", "y"), out_keys=("u", "v", "p"), exprs=_ns2t, C=6)


@pytest.fixture
def lay122(monkeypatch):
    table = {**layer_ref.all_layouts(), "Lay122": LAY122}
    monkeypatch.setattr(layer_ref, "all_layouts", lambda: table)
    monkeypatch.setattr(layer_ref, "THIN_LAYS", layer_ref.THIN_LAYS | {(1, 2, 2)})
    return "Lay122"


def _profiled(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, {e.key for e in prof.key_averages()}


def _launched(names, kernel, lay="SLay<1, 2, 2, 0>"):
    return [nm for nm in names if f"::{kernel}<" in nm and lay in nm]


def _check(name, e, bars, u=U32):
    e = {k: v / u for k, v in e.items()}
    for k in sorted(e):
        print(f"[time-dependent] {name} {k} {e[k]:.3f}", flush=True)
    bad = {k: v for k, v in e.items() if not v <= bars[k.rstrip("0123456789")]}
    assert not bad, f"{name}: {bad} (bars {bars})"


def test_compiled_layout_is_lay122():
    from paddlescience_b200.engine.compiler import compile_residuals
    from tests.cases import make_net

    cr = compile_residuals(make_net(("t", "x", "y"), ("u", "v", "p"), [50] * 9, "tanh"), _ns2t())
    assert [d.order for d in cr.dirs] == [1, 2, 2] and cr.channels == 6


@pytest.mark.parametrize("n", [1, 11, 3013, 70001])
@pytest.mark.parametrize("hidden", [(64, 96), (48, 52)])
def test_thin_layers_vectorised(lay122, hidden, n):
    """Layers 1 and 3 on the vectorised thin kernels of Lay122 (layer 2 on the CUDA-core tiles), one chunk."""
    name = f"thin-h{hidden[0]}-{hidden[1]}-n{n}"
    (plan, params, grads, views), names = _profiled(
        lambda: run_fused(lay122, list(hidden), n, backend=1, chunk_points=n))
    want = thin_kernels(plan)
    assert want["first_fwd"] == "k_first_fwd_v" and want["first_dw"] == "k_first_dw_v"
    assert want["last_fwd"] == "k_last_fwd_v" and want["last_bwd"] == "k_last_bwd_v"
    for k in ("k_first_fwd_v", "k_first_dw_v", "k_last_fwd_v", "k_last_bwd_v"):
        assert _launched(names, k), f"{name}: {k} of Lay122 did not run; launched {sorted(names)}"
    _check(name, all_errors(plan, params, grads, views), THIN_BAR)


WG_WIDTHS = [32, 64, 96, 128, 224, 256]


@pytest.mark.parametrize("n", [3013])
@pytest.mark.parametrize("N", WG_WIDTHS)
def test_wgmma_layer2(lay122, N, n):
    """Layer 2 (K = 128 -> N, and N -> N for the dx of layer 3's fan-in) on k_wg_layer forward / dx and k_wg_dw."""
    _wg_case(lay122, [128, N], n)


@pytest.mark.parametrize("K,N", [(256, 256), (224, 32), (32, 224)])
def test_wgmma_layer2_shapes(lay122, K, N):
    _wg_case(lay122, [K, N], 3013)


@pytest.mark.parametrize("n", [1, 4, 11, 70001])
def test_wgmma_point_counts(lay122, n):
    """1 point, a partial tile (TP = 10), a partial dW chunk, and 70,001 points (several dW splits)."""
    _wg_case(lay122, [128, 128], n)


def test_wgmma_several_chunks(lay122):
    """70,001 points through workspace chunks of 20,000: forward and dx of the last chunk (layer_ref.all_errors)."""
    _wg_case(lay122, [256, 256], 70001, chunk_points=20000)


def _wg_case(lay, hidden, n, chunk_points=0):
    K, N = hidden
    name = f"wg-K{K}-N{N}-n{n}" + (f"-chunk{chunk_points}" if chunk_points else "")
    (plan, params, grads, views), names = _profiled(
        lambda: run_fused(lay, list(hidden), n, backend=2, chunk_points=chunk_points))
    assert plan.uses_tcgen05
    chunked = getattr(plan, "views_last_chunk", False)
    kinds = {"fwd"} | ({"dx"} if K % 32 == 0 else set()) | (set() if chunked else {"dw"})
    assert _launched(names, "k_wg_layer"), f"{name}: k_wg_layer of Lay122 did not run; launched {sorted(names)}"
    if not chunked:
        assert _launched(names, "k_wg_dw"), f"{name}: k_wg_dw of Lay122 did not run"
    e = {f"{k}2": v for k, v in check_layer(plan, views, params, grads, 2, kinds).items()}
    _check(name, e, WG_BAR)


def _case(hidden, dtype):
    return dict(in_keys=("t", "x", "y"), out_keys=("u", "v", "p"), hidden=list(hidden), act="tanh", exprs=_ns2t,
                dtype=dtype)


def test_whole_call_6x256_tensor_cores():
    r = run_case(_case([256] * 6, torch.float32), 4096, device="cuda:0", backend=0)
    print(f"[time-dependent] 6x256 f32 {r}")
    assert r["tc"] and r["res"] <= 1e-5 and r["loss"] <= 1e-5 and r["grad"] <= 5e-5, r


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_whole_call_example_plan(dtype):
    """The unsteady cavity's 9 x 50 tanh MLP: hidden layers on the CUDA-core tiles, first and last layer on the generic
    thin kernels (the vectorised ones take widths that are multiples of 4)."""
    r = run_case(_case([50] * 9, dtype), 4096, device="cuda:0", backend=0)
    print(f"[time-dependent] 9x50 {dtype} {r}")
    if dtype == torch.float32:
        assert r["res"] <= 1e-5 and r["loss"] <= 1e-5 and r["grad"] <= 5e-5, r
    else:
        assert r["res"] <= 1e-11 and r["loss"] <= 1e-12 and r["grad"] <= 1e-11, r
