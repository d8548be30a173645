"""GPU test of the wgmma weight gradient at widths whose fan-in and column blocks are not multiples of 128: layer 192 ->
224 splits its columns into two 128-wide blocks, the second one reaching past the last column, and layer 224 -> 256
has a second fan-in block of 96 rows.  Checked with every pass on wgmma and with the dW pass alone on it."""
import pytest
import torch

from tests.cases import TC_CASES, run_case
from tests.test_gpu_tc import assert_tc

pytestmark = pytest.mark.gpu

CASE = dict(TC_CASES["ns_f32_tc_256"], hidden=[192, 224, 256])


@pytest.mark.parametrize("mask", [7, 4])
def test_tc_dw_uneven_blocks(mask, monkeypatch):
    assert torch.cuda.is_available()
    monkeypatch.setenv("PPSCI_B200_TC_MASK", str(mask))
    r = run_case(CASE, 3000, device="cuda:0", backend=2)
    print(f"[tc] dw_uneven mask={mask} {r}")
    assert_tc(r)
