"""GPU parity at the five BASELINE.json configurations' NAMED shapes (SURVEY.md section 8(d)): the CUDA library through
the C-ABI against the fp64 oracle on the same seeded inputs, default backend selection (what a user gets).

Tolerances (relative; the oracle runs in fp64 and is treated as ground truth — "parity unpinned" against Paddle's
absolute outputs, DESIGN.md section 6):
  fp32 on the tensor cores: residual rel-L2 <= 1e-5 (the north-star bar), loss <= 1e-5, weight gradient <= 5e-5
  fp32 on the CUDA cores:   residual <= 5e-6, loss <= 2e-6, gradient <= 1e-5
  fp64:                     residual <= 1e-11, loss <= 1e-12, gradient <= 1e-11"""
import numpy as np
import pytest
import torch

from tests.cases import NAMED_CASES, TOL, run_case

pytestmark = pytest.mark.gpu

TOL_TC = dict(loss=1e-5, res=1e-5, grad=5e-5)


def _check(name, r):
    dtype = NAMED_CASES[name.split("@")[0]]["dtype"]
    if r["tc"]:
        tl, tr, tg = TOL_TC["loss"], TOL_TC["res"], TOL_TC["grad"]
    else:
        tl, tr, tg = TOL[dtype]
    assert r["loss"] <= tl, (name, r)
    assert r["res"] <= tr, (name, r)
    if not np.isnan(r["grad"]):
        assert r["grad"] <= tg, (name, r)


@pytest.mark.parametrize("name", sorted(NAMED_CASES))
def test_named_shape_matches_oracle(name):
    assert torch.cuda.is_available()
    c = NAMED_CASES[name]
    r = run_case(name, c["n"], device="cuda:0", backend=0)
    if name.startswith(("cfg2", "cfg3")):
        assert r["tc"], "the 128 / 256-wide fp32 tanh configurations must run on the tensor-core kernels"
    _check(name, r)


def test_cfg3_full_batch_subsampled_residual_check():
    """cfg3 exactly as benchmarked: one call over 2^20 points; the oracle evaluates 4,096 evenly strided points of the
    same batch, the loss is checked against the fp64 reduction of the engine's own residuals."""
    r = run_case("cfg3_ldc_6x256", 1 << 20, device="cuda:0", backend=0, oracle_subset=4096)
    assert r["tc"]
    _check("cfg3_ldc_6x256@2^20", r)


def test_cfg4_weight_norm_biharmonic_through_the_public_api():
    """cfg4 as the example configures it (examples/biharmonic2d/conf/biharmonic2d.yaml:45, weight_norm: true):
    MLP(5 x 128, weight_norm=True) in fp64 through ExpressionSolver.train_forward, oracle with the
    reparametrisation W = g V / ||V|| under autograd."""
    import sympy as sp

    import ppsci
    from oracle import ppsci_oracle as O
    from tests.test_weight_norm import _eff_from_raw

    n = 4096
    ppsci.utils.misc.set_random_seed(5)
    m = ppsci.arch.MLP(("x", "y"), ("u",), 5, 128, "tanh", weight_norm=True, dtype=torch.float64)
    with torch.no_grad():
        m.flat.data += 0.05 * torch.randn_like(m.flat.data)
    m = m.to("cuda")
    xs, ys = sp.symbols("x y")
    q = 2.0 * sp.sin(sp.pi * xs / 2) * sp.sin(sp.pi * ys / 3)
    eq = ppsci.equation.Biharmonic(2, q, 1.5)
    rect = ppsci.geometry.Rectangle((0, 0), (2, 3))
    cst = ppsci.constraint.InteriorConstraint(eq.equations, {"biharmonic": 0}, rect,
                                              {"dataset": "IterableNamedArrayDataset", "iters_per_epoch": 1, "batch_size": n},
                                              ppsci.loss.MSELoss("mean"), name="EQ")
    ds = cst.data_loader.loader
    inp = {k: v.to("cuda", torch.float64) for k, v in ds.input.items()}
    lab = {k: v.to("cuda", torch.float64) for k, v in ds.label.items()}
    fh = ppsci.utils.ExpressionSolver()
    losses_all, _ = fh.train_forward((cst.output_expr,), [inp], m, {"EQ": cst}, [lab], [None])
    got_loss = float(losses_all["biharmonic"])
    got_grad = m.flat.grad.detach().cpu().double()
    raw = m.flat.data.detach().cpu().double().requires_grad_(True)
    om = O.OracleMLP(("x", "y"), ("u",), [128] * 5, "tanh")
    x = {k: inp[k].detach().cpu().double().requires_grad_(True) for k in ("x", "y")}
    out = om(_eff_from_raw(m, raw), x)
    data = dict(x)
    data.update(out)
    loss = (O.eval_expr(O.biharmonic_expr(2, q, 1.5)["biharmonic"], data) ** 2).mean()
    loss.backward()
    lerr = abs(got_loss - float(loss.detach())) / abs(float(loss.detach()))
    gerr = float((got_grad - raw.grad).norm() / raw.grad.norm())
    assert lerr <= 1e-11, lerr
    assert gerr <= 1e-10, gerr


def test_cfg5_deeponet_at_2_16_pairs():
    from tests.test_zz_deeponet import _oracle, _setup, _train_forward

    hidden = [128, 128, 128]
    model, cst, data = _setup(torch.float32, "cuda", 1 << 16, 100, 128, hidden)
    g = model({"u": torch.as_tensor(data["u"], dtype=torch.float32, device="cuda"),
               "y": torch.as_tensor(data["y"], dtype=torch.float32, device="cuda")})["G"]
    losses_all, _ = _train_forward(model, cst, "cuda", torch.float32)
    g_ref, loss, grad = _oracle(model, cst, hidden)
    gv = float((g.cpu().double() - g_ref).norm() / g_ref.norm())
    lerr = abs(float(losses_all["G"]) - loss) / abs(loss)
    gerr = float((model.flat.grad.detach().cpu().double() - grad).norm() / grad.norm())
    assert gv <= 1e-5 and lerr <= 1e-5 and gerr <= 5e-5, (gv, lerr, gerr)


# ---- detach (reference: test/equation/test_detach.py:12-175 — the reference's only weight-gradient pin) ----------
_DETACH_ITEMS = ["u", "u__x", "u__y", "u__x__x", "v", "v__x", "v__y", "v__x__x", "p", "p__x", "p__y"]


@pytest.mark.parametrize("state", [0, 5, 85, 341, 682, 1365, 2047])
def test_detach_subsets_match_oracle(state):
    """Several ``detach_keys`` subsets of the N-S equations (the reference sweeps range(0, 2^11, 5)): the loss must not
    depend on the subset, the weight gradient must match the oracle's (<= 1e-5, the reference's tolerance)."""
    import ppsci
    from oracle import ppsci_oracle as O

    keys = tuple(k for i, k in enumerate(_DETACH_ITEMS) if (1 << i) & state)
    nu, rho = 1.314, 0.156  # the reference test's constants
    eqs = ppsci.equation.NavierStokes(nu, rho, 2, False, detach_keys=keys).equations
    case = dict(in_keys=("x", "y"), out_keys=("u", "v", "p"), hidden=[16, 16, 16], act="tanh",
                exprs=lambda: dict(eqs), dtype=torch.float32, reduction="sum")
    r = run_case(case, 4096, device="cuda:0", backend=0)
    assert r["loss"] <= 2e-6 and r["res"] <= 5e-6 and r["grad"] <= 1e-5, (keys, r)
    # the same subset on the tensor-core path (3 x 128 hidden)
    case_tc = dict(case, hidden=[128, 128, 128])
    r = run_case(case_tc, 4096, device="cuda:0", backend=0)
    assert r["tc"]
    assert r["loss"] <= TOL_TC["loss"] and r["res"] <= TOL_TC["res"] and r["grad"] <= TOL_TC["grad"], (keys, r)
