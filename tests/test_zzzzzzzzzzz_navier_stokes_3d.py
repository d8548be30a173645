"""GPU checks of unsteady 3-D Navier-Stokes: the jet layouts (x: 2, y: 2, z: 2, t: 1) and (t: 1, x: 2, y: 2, z: 2),
C = 8, that NavierStokes(nu, rho, 3, time=True) compiles to on (x, y, z, t) and (t, x, y, z) (Lay2221 and Lay1222 of
csrc/jet_layout.cuh).

* Layer by layer against the fp64 reference of tests/layer_ref.py on the values each kernel read after one fused call:
  the vectorised thin first and last layers of Lay2221 (k_first_fwd_v / k_first_dw_v, with and without trainable
  periods, and k_last_fwd_v / k_last_bwd_v for 1 to 4 outputs, backend=1), and, for both layouts, k_wg_layer (forward,
  dx) and k_wg_dw on layer 2 at widths 32..256, at point counts up to 70,001 including a call of several workspace
  chunks.  Lay1222 is in WgLays only: its plans keep the generic thin first and last layer kernels.  The kernels each call
  launched are read from torch.profiler.  Bars are those of tests/test_zzzzzz_layer_kernels.py (thin) and
  tests/test_gpu_tc_layers.py (wgmma).
* The whole call against the fp64 oracle: a 6 x 256 plan on the tensor cores, and the Beltrami example's 10 x 100 plan
  (CUDA-core hidden layers) in fp32 and fp64, with the kernels that served it.

The layouts' equations are added to layer_ref's table, and Lay2221 to its ThinLays, for the duration of each test only:
NS on both key orders (4 outputs) and a heat equation on (x, y, z, t) (1 output, more by ``out_keys``)."""
import pytest
import sympy as sp
import torch

from oracle import ppsci_oracle as O
from tests import layer_ref
from tests.cases import run_case
from tests.layer_ref import U32, all_errors, check_layer, run_fused, thin_kernels

pytestmark = pytest.mark.gpu

THIN_BAR = {"fwd": 28.0, "dx": 92.0, "dw": 88.0, "db": 80.0, "omega": 0.15}  # tests/test_zzzzzz_layer_kernels.py, fp32
WG_BAR = {"fwd": 70.0, "dx": 70.0, "dw": 110.0, "db": 22.0}  # tests/test_gpu_tc_layers.py

XYZT, TXYZ = ("x", "y", "z", "t"), ("t", "x", "y", "z")
SLAY = {"Lay2221": "SLay<2, 2, 2, 1>", "Lay1222": "SLay<1, 2, 2, 2>"}
RANGES = {"x": (-1, 1), "y": (-1, 1), "z": (-1, 1), "t": (0, 1)}


def _ns3t():
    return O.navier_stokes_expr(1.0, 1.0, 3, True)


def _heat_xyzt():
    x, y, z, t = sp.symbols("x y z t")
    u = sp.Function("u")(x, y, z, t)
    return {"heat": u.diff(t) - 0.1 * (u.diff(x, 2) + u.diff(y, 2) + u.diff(z, 2)) + u ** 2}


NS = {"Lay2221": dict(in_keys=XYZT, out_keys=("u", "v", "w", "p"), exprs=_ns3t, C=8, ranges=RANGES),
      "Lay1222": dict(in_keys=TXYZ, out_keys=("u", "v", "w", "p"), exprs=_ns3t, C=8, ranges=RANGES)}


@pytest.fixture
def ns3d(monkeypatch):
    table = {**layer_ref.all_layouts(), **NS,
             "Heat2221": dict(in_keys=XYZT, out_keys=("u",), exprs=_heat_xyzt, C=8)}
    monkeypatch.setattr(layer_ref, "all_layouts", lambda: table)
    monkeypatch.setattr(layer_ref, "THIN_LAYS", layer_ref.THIN_LAYS | {(2, 2, 2, 1)})


def _profiled(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, {e.key for e in prof.key_averages()}


def _launched(names, kernel, lay):
    return [nm for nm in names if f"::{kernel}<" in nm and SLAY[lay] in nm]


def _check(name, e, bars, u=U32):
    e = {k: v / u for k, v in e.items()}
    for k in sorted(e):
        print(f"[ns3d] {name} {k} {e[k]:.3f}", flush=True)
    bad = {k: v for k, v in e.items() if not v <= bars[k.rstrip("0123456789")]}
    assert not bad, f"{name}: {bad} (bars {bars})"


@pytest.mark.parametrize("keys,lay", [(XYZT, "Lay2221"), (TXYZ, "Lay1222")])
def test_compiled_layout(keys, lay):
    from paddlescience_b200.engine.compiler import compile_residuals
    from tests.cases import make_net

    cr = compile_residuals(make_net(keys, ("u", "v", "w", "p"), [100] * 10, "tanh"), _ns3t())
    want = [2, 2, 2, 1] if lay == "Lay2221" else [1, 2, 2, 2]
    assert [d.order for d in cr.dirs] == want and cr.channels == 8


def _thin_case(lay, hidden, n, m=4, periods=None):
    """Layers 1 and 3 on the vectorised thin kernels of the layout (layer 2 on the CUDA-core tiles), one chunk; m
    outputs (NS for 4, the heat equation plus value residuals below)."""
    name = f"{lay}-thin-h{hidden[0]}-{hidden[1]}-m{m}-n{n}" + (f"-{sorted(periods)}" if periods else "")
    spec = lay if m == 4 else "Heat2221"
    out_keys = None if m == 4 else ("u", "a", "b")[:m]
    (plan, params, grads, views), names = _profiled(
        lambda: run_fused(spec, list(hidden), n, backend=1, chunk_points=n, out_keys=out_keys, periods=periods))
    want = thin_kernels(plan)
    assert want["first_fwd"] == "k_first_fwd_v" and want["first_dw"] == "k_first_dw_v"
    assert want["last_fwd"] == "k_last_fwd_v" and want["last_bwd"] == "k_last_bwd_v"
    for k in ("k_first_fwd_v", "k_first_dw_v", "k_last_fwd_v", "k_last_bwd_v"):
        assert _launched(names, k, lay), f"{name}: {k} of {lay} did not run; launched {sorted(names)}"
    for k in ("k_first_fwd", "k_first_dw", "k_last_fwd", "k_last_bwd"):
        assert not _launched(names, k, lay) and not any(f"::{k}<" in nm for nm in names), f"{name}: {k} ran"
    assert any(f"{SLAY[lay]}, {m}>" in nm for nm in _launched(names, "k_last_fwd_v", lay)), f"{name}: M = {m} did not run"
    if periods and any(t for _, t in periods.values()):
        omega = [nm for nm in _launched(names, "k_first_dw_v", lay) if "true" in nm.split("(")[0]]
        assert omega, f"{name}: the OMEGA instance of k_first_dw_v did not run"
        assert plan.compiled.net.n_omega == 1
    _check(name, all_errors(plan, params, grads, views), THIN_BAR)


@pytest.mark.parametrize("m", [1, 2, 3, 4])
def test_thin_layers_outputs(ns3d, m):
    _thin_case("Lay2221", (64, 96), 3013, m)


@pytest.mark.parametrize("n", [1, 11, 70001])
def test_thin_layers_point_counts(ns3d, n):
    _thin_case("Lay2221", (48, 52), n)


def test_thin_first_layer_trainable_period(ns3d):
    """Periodic t (cos / sin features, 5 in all) with a trainable frequency: k_first_dw_v's OMEGA instance."""
    _thin_case("Lay2221", (64, 96), 3013, 4, periods={"t": (1.5, True)})


def test_thin_first_layer_fixed_period(ns3d):
    _thin_case("Lay2221", (64, 96), 3013, 4, periods={"x": (2.0, False)})


WG_WIDTHS = [32, 64, 96, 128, 160, 192, 224, 256]


@pytest.mark.parametrize("lay", ["Lay2221", "Lay1222"])
@pytest.mark.parametrize("N", WG_WIDTHS)
def test_wgmma_layer2(ns3d, lay, N):
    """Layer 2 (K = 128 -> N, and N -> N for the dx of layer 3's fan-in) on k_wg_layer forward / dx and k_wg_dw."""
    _wg_case(lay, [128, N], 3013)


@pytest.mark.parametrize("lay", ["Lay2221", "Lay1222"])
@pytest.mark.parametrize("K,N", [(256, 256), (224, 32), (32, 224)])
def test_wgmma_layer2_shapes(ns3d, lay, K, N):
    _wg_case(lay, [K, N], 3013)


@pytest.mark.parametrize("lay", ["Lay2221", "Lay1222"])
@pytest.mark.parametrize("n", [1, 5, 11, 70001])
def test_wgmma_point_counts(ns3d, lay, n):
    """1 point, a partial tile (TP = 8), a partial dW chunk, and 70,001 points (several dW splits)."""
    _wg_case(lay, [128, 128], n)


@pytest.mark.parametrize("lay", ["Lay2221", "Lay1222"])
def test_wgmma_several_chunks(ns3d, lay):
    """70,001 points through workspace chunks of 20,000: forward and dx of the last chunk (layer_ref.all_errors)."""
    _wg_case(lay, [256, 256], 70001, chunk_points=20000)


def _wg_case(lay, hidden, n, chunk_points=0):
    K, N = hidden
    name = f"{lay}-wg-K{K}-N{N}-n{n}" + (f"-chunk{chunk_points}" if chunk_points else "")
    (plan, params, grads, views), names = _profiled(
        lambda: run_fused(lay, list(hidden), n, backend=2, chunk_points=chunk_points))
    assert plan.uses_tcgen05
    chunked = getattr(plan, "views_last_chunk", False)
    kinds = {"fwd"} | ({"dx"} if K % 32 == 0 else set()) | (set() if chunked else {"dw"})
    assert _launched(names, "k_wg_layer", lay), f"{name}: k_wg_layer of {lay} did not run; launched {sorted(names)}"
    if not chunked:
        assert _launched(names, "k_wg_dw", lay), f"{name}: k_wg_dw of {lay} did not run"
    e = {f"{k}2": v for k, v in check_layer(plan, views, params, grads, 2, kinds).items()}
    _check(name, e, WG_BAR)


def _assert_thin(names, lay):
    """fp32 first and last layers: the vectorised thin kernels of Lay2221, the generic ones for Lay1222."""
    for k in ("k_first_fwd", "k_first_dw", "k_last_fwd", "k_last_bwd"):
        vec = _launched(names, k + "_v", lay)
        generic = any(f"::{k}<" in nm for nm in names)
        assert (vec and not generic) if lay == "Lay2221" else (generic and not vec), (lay, k, sorted(names))


def _case(keys, hidden, dtype):
    return dict(in_keys=keys, out_keys=("u", "v", "w", "p"), hidden=list(hidden), act="tanh", exprs=_ns3t, dtype=dtype,
                ranges=RANGES)


@pytest.mark.parametrize("keys,lay", [(XYZT, "Lay2221"), (TXYZ, "Lay1222")])
def test_whole_call_6x256_tensor_cores(keys, lay):
    r, names = _profiled(lambda: run_case(_case(keys, [256] * 6, torch.float32), 4096, device="cuda:0", backend=0))
    print(f"[ns3d] 6x256 {lay} f32 {r}")
    assert r["tc"] and _launched(names, "k_wg_layer", lay) and _launched(names, "k_wg_dw", lay)
    _assert_thin(names, lay)
    assert r["res"] <= 1e-5 and r["loss"] <= 1e-5 and r["grad"] <= 5e-5, r


@pytest.mark.parametrize("keys,lay", [(XYZT, "Lay2221"), (TXYZ, "Lay1222")])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_whole_call_beltrami_plan(keys, lay, dtype):
    """The Beltrami example's 10 x 100 tanh MLP: hidden layers on the CUDA-core tiles (100 is not a multiple of 32); in
    fp32 the first and last layers of Lay2221 on the vectorised thin kernels (100 is a multiple of 4, M = 4)."""
    r, names = _profiled(lambda: run_case(_case(keys, [100] * 10, dtype), 4096, device="cuda:0", backend=0))
    print(f"[ns3d] 10x100 {lay} {dtype} {r}")
    assert not r["tc"] and not any("k_wg_" in nm for nm in names)
    assert any("::k_gemm_fwd<" in nm for nm in names) and any("::k_gemm_dw<" in nm for nm in names)
    if dtype == torch.float32:
        _assert_thin(names, lay)
        assert r["res"] <= 5e-6 and r["loss"] <= 2e-6 and r["grad"] <= 1e-5, r
    else:
        assert r["res"] <= 1e-11 and r["loss"] <= 1e-12 and r["grad"] <= 1e-11, r
