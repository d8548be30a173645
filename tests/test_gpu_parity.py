"""GPU parity: the CUDA library (through the C-ABI) versus the torch oracle on the same inputs."""
import pytest
import torch

from tests.cases import CASES, TOL, run_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(CASES))
def test_case_matches_oracle_gpu(name):
    assert torch.cuda.is_available(), "GPU tests need an H100"
    n = 3000 if CASES[name]["hidden"][0] > 64 else 5000
    r = run_case(name, n, device="cuda:0", backend=1)
    tl, tr, tg = TOL[CASES[name]["dtype"]]
    assert r["loss"] <= tl, r
    assert r["res"] <= tr, r
    assert r["grad"] <= tg, r
    assert r["fwd_vs_fused"] == 0.0, r
