"""GPU sweep of the residual-program head (k_head) against the fp64 reference of tests/head_ref.py on the output jets
the head read: the directed cases (every opcode, exact ties of Max / Min / where, selects with a NaN or Inf in the
untaken branch, a program of at least 248 registers on the C = 29 layout with 8 outputs, 16 slots mixing every loss
option, 32 learnable-parameter gradient terms, point counts 1, 127, 128, 129, 3,013 and 70,001) and seeded random
programs, in fp32 and fp64.

Each case runs twice: on a plan whose output jets come from the CUDA-core tile GEMM (backend=1 with
PPSCI_B200_NO_THIN=1) and on a default plan (the thin last-layer kernels).  Every run also checks a call on a workspace
of NaN bytes (bitwise equal), ``plan.forward`` (bitwise equal), the seeded parameter-gradient buffer over two calls and,
for the chunked cases, a call over three workspace chunks (``head_ref.run_case``).  Run with -s for the error table."""
import pytest
import torch

from tests import head_ref as H

pytestmark = pytest.mark.gpu

# Bars in units of the rounding u of the dtype (residuals: of the running-error bound M; Ybar: of its plane's largest
# |ref|; dLoss/dparameter: of sum_p |term|; losses: relative), about twice the largest error measured over this file's
# matrix on an H100 80GB HBM3 (700 W power limit):
#   fp32 (units of 2^-24): residual 1.0, loss 6.5 (one point), Ybar 52.5 (random program), dLoss/dparameter 1.6, the
#        seeded parameter-gradient buffer 0.0 (its fp64 sums);
#   fp64 (units of 2^-53): residual 1.3, loss 12.3 (70,001 points: 547 head blocks' atomic partial sums), Ybar 10.5
#        (chunked random program), dLoss/dparameter 2.3, the seeded parameter-gradient buffer 2.5.
# A dropped or wrong partial is off by O(1) relative: 2^53 units in fp64, 2^24 in fp32.
BAR = {torch.float32: {"res": 2.0, "loss": 13.0, "ybar": 105.0, "pgrad": 3.2, "pgrad_acc": 2.0},
       torch.float64: {"res": 2.6, "loss": 25.0, "ybar": 21.0, "pgrad": 4.6, "pgrad_acc": 5.0}}

CASES = H.matrix(torch.float32, gpu=True) + H.matrix(torch.float64, gpu=True)
PLANS = {"gemm": (1, {"PPSCI_B200_NO_THIN": "1"}), "default": (0, {})}


@pytest.mark.parametrize("plan", list(PLANS))
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_head_program_gpu(monkeypatch, case, plan):
    backend, env = PLANS[plan]
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, v)
        e = H.run_case(case, device="cuda:0", backend=backend)
    print(f"\n[head gpu] {case.name} [{plan}]: " + " ".join(f"{k}={v:.2f}" for k, v in sorted(e.items())))
    bar = BAR[case.dtype]
    bad = {k: v for k, v in e.items() if not v <= bar[k.replace("_chunked", "")]}
    assert not bad, f"{case.name} [{plan}]: {bad} (bars {bar})"
