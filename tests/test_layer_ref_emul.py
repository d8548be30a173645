"""CPU self-test of the per-layer fp64 reference (tests/layer_ref.py) through the emulation build of the engine: the
workspace offsets of the stash accessor, the Zbar ping-pong rule and the reference's activation jets, adjoint and
weight gradient are checked against the emulated CUDA-core kernels for every jet layout the tensor-core kernels take.
In fp64 they must agree to ~1e-12; in fp32 the errors in units of 2^-24 are printed (the CUDA-core side of the bars
of tests/test_gpu_tc_layers.py)."""
import pytest
import torch

from paddlescience_b200.engine import binding as B
from tests.emul.build_emul import build
from tests.layer_ref import U32, check_layer, layouts, run_fused


@pytest.fixture(scope="module")
def emul_lib():
    return B.Library(build())


def _errors(plan, params, grads, views):
    L = len(plan.compiled.net.widths) - 1
    e = {f"{k}2": v for k, v in check_layer(plan, views, params, grads, 2, {"fwd", "dx", "dw"}).items()}
    e["fwdY"] = check_layer(plan, views, params, grads, L, {"fwd"})["fwd"]
    return e


@pytest.mark.parametrize("hidden", [[16, 24], [12, 16, 8]], ids=["h16-24", "h12-16-8"])
@pytest.mark.parametrize("layout", sorted(layouts()))
def test_reference_matches_emulated_kernels_f64(emul_lib, layout, hidden):
    # L = 3 and L = 4: Zbar_1 and Zbar_2 sit in buffers (1, 0) and (0, 1); a wrong rule reads another layer's adjoint
    n = 37
    plan, params, grads, views = run_fused(layout, hidden, n, dtype=torch.float64, backend=1, library=emul_lib,
                                           device="cpu", seed=3)
    e = _errors(plan, params, grads, views)
    assert set(e) == {"fwd2", "dx2", "dw2", "db2", "fwdY"}
    assert max(e.values()) <= 1e-12, e
    # the stash is not all zeros (a wrong offset into zeroed memory would pass the comparisons above)
    assert float(views["Zbar1"].abs().max()) > 0 and float(views["Z1"].abs().max()) > 0


@pytest.mark.parametrize("layout", sorted(layouts()))
def test_reference_on_emulated_kernels_f32(emul_lib, layout):
    n = 29
    plan, params, grads, views = run_fused(layout, [16, 24], n, dtype=torch.float32, backend=1, library=emul_lib,
                                           device="cpu", seed=4)
    e = {k: v / U32 for k, v in _errors(plan, params, grads, views).items()}
    print(f"\n[layer_ref emul f32] {layout}: " + " ".join(f"{k}={v:.2f}" for k, v in sorted(e.items())))
    # the CUDA-core kernels accumulate in fp32: a few units of the componentwise bound, far below a wrong term
    assert max(e.values()) <= 64, e
