"""GPU tests of the tensor-core path: parity against the oracle through the C-ABI with backend=2 (forward, dx and dW
of the eligible layers on the wgmma kernels, required), tolerance of the 3xTF32 scheme stated here."""
import pytest
import torch

from tests.cases import TC_CASES, run_case

pytestmark = pytest.mark.gpu

# hi/lo operand splits + fp32 tensor-core accumulation: residual rel-L2 <= 1e-5 is the north-star bar and the loss
# (a mean of squares) is held to the same; the weight gradient to 5e-5.
TOL_TC = dict(loss=1e-5, res=1e-5, grad=5e-5)


# PPSCI_B200_TC_MASK selects the passes on the tensor cores: bit 0 forward, bit 1 dx, bit 2 dW; the others run on the
# CUDA cores, so 3, 1, 2 and 4 check each wgmma pass against CUDA-core neighbours.  Its higher bits chose kernel variants
# of the Blackwell build that Hopper does not have: 255, 63 and 7 all put every pass on wgmma.
@pytest.mark.parametrize("mask", [255, 63, 7, 3, 1, 2, 4])
@pytest.mark.parametrize("name", sorted(TC_CASES))
def test_tc_case_matches_oracle(name, mask, monkeypatch):
    assert torch.cuda.is_available()
    monkeypatch.setenv("PPSCI_B200_TC_MASK", str(mask))
    r = run_case(name, 3000, device="cuda:0", backend=2)
    assert r["tc"], "tensor-core backend was not selected"
    assert r["loss"] <= TOL_TC["loss"], r
    assert r["res"] <= TOL_TC["res"], r
    assert r["grad"] <= TOL_TC["grad"], r


@pytest.mark.parametrize("n", [13, 3013, 70001])
def test_tc_ragged_point_counts(n):
    """A partial last tile, fewer tiles than CTAs, and more than one pass of the persistent loop."""
    r = run_case("ns_f32_tc_256", n, device="cuda:0", backend=2)
    assert r["tc"]
    assert r["loss"] <= TOL_TC["loss"], r
    assert r["res"] <= TOL_TC["res"], r
    assert r["grad"] <= TOL_TC["grad"], r
