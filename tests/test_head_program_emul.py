"""The residual-program head (k_head) through the CPU emulation build of the kernel sources, opcode by opcode and on
seeded random programs, against the fp64 reference of tests/head_ref.py on the output jets the head read.

Each case runs the checks of ``head_ref.run_case``: residual_out, the losses, the output-jet adjoints Ybar and
dLoss/d(learnable parameter) against the reference; the same call on a workspace of NaN bytes (bitwise equal);
``plan.forward`` (residuals bitwise equal); the parameter-gradient buffer seeded over two calls; and for the chunked
cases a call over three workspace chunks.  The emulation runs every CUDA thread as an OS thread, so the point counts stay
small; tests/test_zzzzzzzz_head_program.py runs the same matrix on the GPU at its full sizes."""
import pytest
import sympy as sp
import torch

from oracle import ppsci_oracle as O
from paddlescience_b200.engine import binding as B
from tests import head_ref as H
from tests.emul.build_emul import build

# Bars in units of the rounding u of the dtype: residuals of the running-error bound M, Ybar of its plane's largest
# |ref|, dLoss/dparameter of sum_p |term|, losses relative.  A dropped or wrong partial is off by O(1) relative (about
# 2^53 units in fp64, 2^24 in fp32).
BAR = {torch.float64: {"res": 8.0, "loss": 16.0, "ybar": 64.0, "pgrad": 64.0, "pgrad_acc": 16.0},
       torch.float32: {"res": 8.0, "loss": 16.0, "ybar": 64.0, "pgrad": 64.0, "pgrad_acc": 16.0}}

CASES = H.matrix(torch.float64, gpu=False) + H.matrix(torch.float32, gpu=False)


@pytest.fixture(scope="module")
def emul_lib():
    return B.Library(build())


def check(case, e):
    print(f"\n[head emul] {case.name}: " + " ".join(f"{k}={v:.2f}" for k, v in sorted(e.items())))
    bar = BAR[case.dtype]
    bad = {k: v for k, v in e.items() if not v <= bar[k.replace("_chunked", "")]}
    assert not bad, f"{case.name}: {bad} (bars {bar})"


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_head_program_emulated(emul_lib, case):
    check(case, H.run_case(case, library=emul_lib, device="cpu", backend=1))


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
def test_directed_cases_emit_every_opcode(dtype):
    """The directed programs of one dtype together run all 25 opcodes."""
    seen = set()
    for case in H.matrix(dtype, gpu=False):
        if case.name.startswith(("opcodes", "ties", "selects", "slots16", "params", "reglimit")):
            net = H.make_net(H.all_layouts()[case.layout]["in_keys"], case.out_keys or
                             H.all_layouts()[case.layout]["out_keys"], [8], "tanh")
            seen |= H.ops_of(H.compile_residuals(net, case.exprs(), param_keys=list(case.learn or {})))
    assert seen == set(B.OPS), sorted(set(B.OPS) - seen)


def test_sign_and_heaviside_gradient_matches_oracle(emul_lib):
    """sign(u) v + Heaviside(u - 0.3) u compiles (the partials' DiracDelta terms are zero), and the engine's Ybar is
    the oracle's gradient through torch.sign / torch.heaviside (zero almost everywhere) on the same output jets."""
    x, y = sp.symbols("x y")
    u, v = sp.Function("u")(x, y), sp.Function("v")(x, y)
    exprs = {"r": sp.sign(u) * v + sp.Heaviside(u - 0.3) * u, "r2": sp.Heaviside(v - u) * u * v}
    run = H.setup("LayV", exprs, 29, dtype=torch.float64, library=emul_lib, device="cpu", backend=1,
                  slots=[H.Slot(out=True)] * 2)
    assert H.ops_of(run.cr) >= {"sign", "heaviside"}
    run.plan._workspace(run.n, run.params.device).zero_()
    _, outs, _ = H.call(run)
    V = H.views(run)
    Y = V["Y"].double().detach().requires_grad_(True)
    data = {"u": Y[0, :, 0], "v": Y[0, :, 1], "x": run.inputs["x"].view(-1).double(),
            "y": run.inputs["y"].view(-1).double()}
    loss = 0.0
    for k, ex in exprs.items():
        r = O.eval_expr(ex, data)
        assert torch.allclose(outs[k].view(-1), r.detach(), rtol=1e-14, atol=1e-14), k
        loss = loss + (r * r).sum() / run.n
    (g,) = torch.autograd.grad(loss, Y)
    assert torch.allclose(V["Ybar"], g, rtol=1e-13, atol=1e-15)
    assert float(V["Ybar"][0, :, 0].abs().max()) > 0 and float(V["Ybar"][0, :, 1].abs().max()) > 0
