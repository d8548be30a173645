"""CPU tests of the SIMT kernel SOURCES through the emulation build (tests/emul/cuda_emul.h):
every CUDA thread is an OS thread, blocks run one at a time.  Same C-ABI, same host code."""
import pytest
import torch

from paddlescience_b200.engine import binding as B
from tests.cases import CASES, LATE_CASES, TOL, run_case
from tests.emul.build_emul import build


@pytest.fixture(scope="module")
def emul_lib():
    return B.Library(build())


@pytest.mark.parametrize("name", sorted(CASES) + sorted(LATE_CASES))
def test_case_matches_oracle(emul_lib, name):
    c = CASES.get(name) or LATE_CASES[name]
    n = 45 if c["hidden"][0] > 64 else 70
    r = run_case(name, n, library=emul_lib, device="cpu")
    tl, tr, tg = TOL[c["dtype"]]
    assert r["loss"] <= tl, r
    assert r["res"] <= tr, r
    assert r["grad"] <= tg, r
    assert r["fwd_vs_fused"] == 0.0, r


@pytest.mark.parametrize("name", ["ns_f32", "allen_cahn_period_f64", "biharmonic_f64"])
def test_tile_gemm_path_for_thin_layers(emul_lib, name, monkeypatch):
    """The dedicated first/last-layer kernels can be switched off: the generic tile GEMMs must agree."""
    monkeypatch.setenv("PPSCI_B200_NO_THIN", "1")
    r = run_case(name, 60, library=emul_lib, device="cpu")
    tl, tr, tg = TOL[CASES[name]["dtype"]]
    assert r["loss"] <= tl and r["res"] <= tr and r["grad"] <= tg, r

