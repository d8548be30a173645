"""ChipDeepONets: three branch nets (heat source, boundary data, boundary type) and an (x, y) trunk trained through the
operator jet head with a third branch factor, on residuals that select their form by boundary type
(``torch.where(bc == k, ...)``, lowered to the residual program's EQ + SELECT).  Also ChipHeatDataset and plain-MLP
``where`` residuals.

Oracle: ``O.train_forward_backward`` over ``OracleChipDeepONets`` (tests/chip_deeponet_ref.py); autograd supplies the x
and y derivatives and torch.where the selection.  CPU: the emulation build of the same kernel sources, fp64.  GPU: the
example's shapes in fp32, small shapes in fp64, and Solver steps on the example's small configuration."""
import ctypes as C
import os
import sys
import types

import numpy as np
import pytest
import sympy as sp
import torch

import ppsci
from oracle import ppsci_oracle as O
from paddlescience_b200.engine import binding as B
from tests.chip_deeponet_ref import OracleChipDeepONets, eval_piecewise
from tests.test_zzzz_pi_deeponet import _check, _effective, _emul

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = (("u",), ("bc",), ("bc_data",), ("x", "y"), ("T",))
INPUTS = ("x", "y", "u", "bc_data", "bc", "u_one")


def _model(dtype, feats, hb, hbc, ht, num_loc=6, bc_loc=5, act="tanh", bc_act="sin", seed=5, **options):
    ppsci.utils.misc.set_random_seed(seed)
    model = ppsci.arch.ChipDeepONets(*KEYS, num_loc, 1, bc_loc, feats, None, None, None, tuple(hb), tuple(hbc), tuple(ht),
                                     branch_activation=act, BC_activation=bc_act, trunk_activation=act, dtype=dtype,
                                     **options)
    with torch.no_grad():
        model.flat.data += 0.05 * torch.randn_like(model.flat.data)
    return model


def _oracle(model, hb, hbc, ht):
    m = model
    act, bc_act = m.trunk_activation, m._nets[1].act  # branch and trunk share ``act`` in these tests
    return OracleChipDeepONets(*KEYS, m._branch_locs[0], 1, m._branch_locs[2], m.num_features, hb, hbc, ht, act, bc_act, act,
                               effective=lambda flat, j, p: _effective(m, flat, m._subnets[j]))


def _data(n, seed=11, num_loc=6, bc_loc=5, bc_values=(0, 1, 2, 3)):
    rng = np.random.RandomState(seed)
    return {"x": rng.rand(n, 1), "y": rng.rand(n, 1), "u": rng.randn(n, num_loc), "bc_data": rng.randn(n, bc_loc),
            "bc": rng.choice(np.array(bc_values, dtype=np.float64), size=(n, 1)), "u_one": rng.randn(n, 1),
            "w": rng.rand(n, 1) + 0.5}


def _boundary(d, jac, where, var):
    """The example's boundary residual as it writes it (chip_heat.py: top / down with x, left / right with y)."""
    return where(d["bc"] == 1, jac(d["T"], d[var]) - d["u_one"],
                 where(d["bc"] == 0, d["T"] - d["u_one"],
                       where(d["bc"] == 2, jac(d["T"], d[var]) + d["u_one"] * (d["T"] - 1),
                             jac(d["T"], d[var]) + d["u_one"] * (d["T"] ** 2 - 1) * (d["T"] ** 2 + 1) * 5.6 / 50000)))


def _interior(d, jac, where):
    hess = lambda f, x: jac(jac(f, x), x)  # noqa: E731
    return hess(d["T"], d["x"]) + hess(d["T"], d["y"]) + 100 * d["u_one"]


EXAMPLE = {"top": lambda d, j, w: _boundary(d, j, w, "x"), "down": lambda d, j, w: _boundary(d, j, w, "x"),
           "left": lambda d, j, w: _boundary(d, j, w, "y"), "right": lambda d, j, w: _boundary(d, j, w, "y"),
           "interior": _interior}


def _both(fn):
    """(traced by the model, run by the oracle) versions of a residual written once over (jacobian, where)."""
    return (lambda d: fn(d, ppsci.autodiff.jacobian, torch.where)), (lambda d: fn(d, O.jacobian, torch.where))


def _run(model, hb, hbc, ht, exprs, oracle_exprs, data, device, dtype, labels, weights=None, calls=1):
    t = lambda a: torch.as_tensor(a, dtype=dtype, device=device)  # noqa: E731
    n = len(data["x"])
    inputs = {k: t(data[k]) for k in INPUTS}
    lab = {k: t(np.full((n, 1), v)) for k, v in labels.items()}
    wts = {k: t(data[v]) for k, v in (weights or {}).items()}
    cst = types.SimpleNamespace(loss=ppsci.loss.MSELoss("mean"), output_expr=exprs)
    fh = ppsci.utils.ExpressionSolver()
    for _ in range(calls):
        losses_all, losses_cst = fh.train_forward((exprs,), [inputs], model, {"c": cst}, [lab], [wts or None])
    cpu = {k: v.detach().cpu().double() for k, v in inputs.items()}
    o_losses, o_res, o_grad = O.train_forward_backward(
        _oracle(model, hb, hbc, ht), model.flat.detach().cpu().double(), oracle_exprs, cpu,
        {k: v.cpu().double() for k, v in lab.items()}, {k: v.cpu().double() for k, v in wts.items()} or None)
    return losses_all, losses_cst, o_losses, o_res, o_grad


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", list(EXAMPLE))
def test_example_constraints_through_emulated_kernels_match_oracle(monkeypatch, which):
    """The five constraint expressions exactly as the example writes them; the batch holds all four boundary types."""
    _emul(monkeypatch)
    hb, hbc, ht = [8, 8], [7, 7], [9, 9]
    model = _model(torch.float64, 6, hb, hbc, ht)
    ours, theirs = _both(EXAMPLE[which])
    data = _data(53)
    assert set(np.unique(data["bc"])) == {0.0, 1.0, 2.0, 3.0}
    losses_all, _, o_losses, _, o_grad = _run(model, hb, hbc, ht, {"chip": ours}, {"chip": theirs}, data, "cpu",
                                              torch.float64, {"chip": 0.0}, weights={"chip": "w"})
    _check(model, losses_all, o_losses, o_grad)


def test_weight_norm_skip_multi_chunk_and_accumulation_through_emulated_kernels(monkeypatch):
    """A weight-norm branch net, skip-connection BC nets, 2,300 pairs over 1,024-point chunks, two calls."""
    _emul(monkeypatch)
    monkeypatch.setenv("PPSCI_B200_CHUNK_POINTS", "1024")
    hb, hbc, ht = [8, 8, 8], [6, 6, 6], [8, 8]
    model = _model(torch.float64, 4, hb, hbc, ht, branch_weight_norm=True, BC_skip_connection=True)
    ours, theirs = _both(EXAMPLE["left"])
    losses_all, _, o_losses, _, o_grad = _run(model, hb, hbc, ht, {"chip": ours}, {"chip": theirs}, _data(2300), "cpu",
                                              torch.float64, {"chip": 0.0}, calls=2)
    assert model._get_plans()[0].chunk_points == 1024
    _check(model, losses_all, o_losses, o_grad, calls=2, rtol=1e-8)


def test_state_dict_round_trip_with_reference_keys():
    hb, hbc, ht = [6, 6], [5], [4]
    model = _model(torch.float64, 3, hb, hbc, ht, BC_weight_norm=True)
    sd = model.state_dict()
    expect = {f"branch_net.linears.{i}.{p}" for i in range(2) for p in ("weight", "bias")}
    for net in ("BCtype_net", "BC_net"):
        expect |= {f"{net}.linears.0.weight_v", f"{net}.linears.0.weight_g", f"{net}.linears.0.bias"}
    for net in ("branch_net", "BCtype_net", "BC_net", "trunk_net"):
        expect |= {f"{net}.last_fc.weight", f"{net}.last_fc.bias"}
    expect |= {"trunk_net.linears.0.weight", "trunk_net.linears.0.bias", "b"}
    assert set(sd) == expect
    assert tuple(sd["b"].shape) == (1,)
    assert tuple(sd["branch_net.linears.0.weight"].shape) == (6, 6) and tuple(sd["BCtype_net.linears.0.weight_v"].shape) == (1, 5)
    assert tuple(sd["BC_net.linears.0.weight_v"].shape) == (5, 5) and tuple(sd["trunk_net.last_fc.weight"].shape) == (4, 3)
    other = _model(torch.float64, 3, hb, hbc, ht, seed=9, BC_weight_norm=True)
    assert not torch.equal(other.state_dict()["branch_net.last_fc.weight"], sd["branch_net.last_fc.weight"])
    other.load_state_dict(sd)
    back = other.state_dict()
    assert all(torch.equal(back[k], v) for k, v in sd.items())


def test_sub_network_settings_follow_the_reference():
    model = ppsci.arch.ChipDeepONets(*KEYS, 6, 1, 5, 4, 2, 3, 1, 8, 7, 9, branch_activation="relu", BC_activation="sin",
                                     trunk_activation="tanh", dtype=torch.float64)
    assert model.input_keys == ("x", "y", "u", "bc_data", "bc")
    assert [n.widths for n in model._nets] == [[6, 8, 8, 4], [1, 7, 7, 7, 4], [5, 7, 7, 7, 4], [2, 9, 4]]
    assert [n.act for n in model._nets] == ["relu", "sin", "sin", "tanh"]


def test_refusals(monkeypatch):
    _emul(monkeypatch)
    model = _model(torch.float64, 3, [6], [6], [6])
    data = _data(9)
    fh = ppsci.utils.ExpressionSolver()
    inputs = {k: torch.as_tensor(data[k]) for k in INPUTS}

    def call(expr):
        cst = types.SimpleNamespace(loss=ppsci.loss.MSELoss(), output_expr={"res": expr})
        return fh.train_forward((cst.output_expr,), [inputs], model, {"c": cst},
                                [{"res": torch.zeros(9, 1, dtype=torch.float64)}], [None])

    for cond in (lambda d: d["bc"] > 1, lambda d: d["bc"] != 1, lambda d: d["bc"] <= 2):
        with pytest.raises(NotImplementedError, match=r"must be equalities, as in torch.where\(x == c, a, b\)"):
            call(lambda d: torch.where(cond(d), d["T"], d["T"] - d["u_one"]))
    with pytest.raises(NotImplementedError, match="branch input 'u'"):
        call(lambda d: d["T"] * d["u"])


def test_third_branch_factor_needs_the_second_at_the_c_abi(monkeypatch):
    """deeponet_jet_head_run: b3 without b2, b3bar without b3 and a short ldb3 are refused before any launch."""
    _emul(monkeypatch)
    model = _model(torch.float64, 3, [6], [6], [6])
    d = _data(4)
    head = model._jet_head({"chip": lambda o: o["T"] - o["u_one"]}, ("u_one",))
    lib = head.lib
    buf = torch.zeros(64, dtype=torch.float64)
    col = torch.as_tensor(d["x"]).reshape(-1).contiguous()

    def args(**kw):
        a = B.DeepONetJetArgs()
        a.b, a.ldb, a.t, a.ldt, a.tplane, a.n, a.n_features = buf.data_ptr(), 3, buf.data_ptr(), 3, 12, 4, 3
        for j in range(2):
            a.x_cols[j] = col.data_ptr()
        a.aux_cols[0] = col.data_ptr()
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    def run(a):
        return lib.lib.ppsci_b200_deeponet_jet_head_run(head.handle, C.byref(a), None)

    assert run(args(b2=buf.data_ptr(), ldb2=3, b3=buf.data_ptr(), ldb3=3)) == 0
    assert run(args(b3=buf.data_ptr(), ldb3=3)) != 0
    assert "needs the second one, b2" in lib.last_error()
    assert run(args(b2=buf.data_ptr(), ldb2=3, b3=buf.data_ptr(), ldb3=2)) != 0
    assert "row pitch" in lib.last_error()
    full = dict(b2=buf.data_ptr(), ldb2=3, bbar=buf.data_ptr(), tbar=buf.data_ptr(), b2bar=buf.data_ptr())
    assert run(args(**full, b3=buf.data_ptr(), ldb3=3)) != 0
    assert "b3bar" in lib.last_error()
    assert run(args(**full, b3bar=buf.data_ptr())) != 0
    assert "b3bar" in lib.last_error()


# ---------------------------------------------------------------------------------------------------------------------
def _reference_getitem(ds_input, label, weight, index, data_type, idx):
    """chip_heat's ChipHeatDataset.__getitem__ restated literally (array_dataset.py:282-305)."""
    quotient = idx
    index_ir = dict()
    for i in index:
        index_ir[i] = 0
    for i in index_ir:
        num = len(ds_input[i])
        index_ir[i] = quotient % num
        quotient = quotient // num
    input_item = {}
    for key in ds_input:
        if key == "y":
            input_item[key] = ds_input[key][index_ir["x"]]
        elif key == "u_one":
            input_item[key] = ds_input[key][len(ds_input[data_type]) * index_ir["x"] + index_ir[data_type]]
        else:
            input_item[key] = ds_input[key][index_ir[key]]
    return input_item, dict(label), dict(weight)


def _chip_input(rng, data_type):
    n_x, n_u, n_bcd = 5, 3, 4
    return {"x": rng.rand(n_x, 1), "y": rng.rand(n_x, 1), "u": rng.randn(n_u, 6), "u_one": rng.randn(n_x * (n_u if data_type == "u" else n_bcd), 1),
            "bc": np.array([[0], [1], [2], [3]], dtype=np.float64), "bc_data": rng.randn(n_bcd, 5)}


@pytest.mark.parametrize("data_type", ["u", "bc_data"])
def test_chip_heat_dataset_matches_the_reference_loop(data_type):
    rng = np.random.RandomState(0)
    inp = _chip_input(rng, data_type)
    label, weight = {"chip": np.array([0.0])}, {"chip": np.array([500.0])}
    index = ("x", "u", "bc", "bc_data")
    ds = ppsci.data.dataset.build_dataset({"name": "ChipHeatDataset", "input": inp, "label": label, "index": index,
                                           "data_type": data_type, "weight": weight})
    assert len(ds) == 5 * 3 * 4 * 4
    for i in range(len(ds)):
        got, ref = ds[i], _reference_getitem(inp, label, weight, index, data_type, i)
        for a, b in zip(got, ref):
            assert list(a) == list(b)
            assert all(np.array_equal(a[k], b[k]) for k in a)
    idx = rng.permutation(len(ds))[:37]
    inp_b, lab_b, wt_b = ds[idx]
    for k in inp:
        assert np.array_equal(inp_b[k], np.stack([ds[int(i)][0][k] for i in idx])), k
    assert lab_b["chip"].shape == (37, 1) and np.all(lab_b["chip"] == 0.0)
    assert wt_b["chip"].shape == (37, 1) and np.all(wt_b["chip"] == 500.0)


def test_chip_heat_dataset_through_a_shuffled_constraint_loader():
    rng = np.random.RandomState(1)
    inp = _chip_input(rng, "u")
    cst = ppsci.constraint.SupervisedConstraint(
        {"dataset": {"name": "ChipHeatDataset", "input": inp, "label": {"chip": np.array([0.0])},
                     "index": ("x", "u", "bc", "bc_data"), "data_type": "u", "weight": {"chip": np.array([500.0])}},
         "batch_size": 50, "sampler": {"name": "BatchSampler", "drop_last": False, "shuffle": True}},
        ppsci.loss.MSELoss("mean"), output_expr={"chip": lambda out: out["T"]}, name="c")
    cat = lambda d: np.concatenate([np.asarray(d[k]).reshape(len(d["x"]), -1) for k in ("x", "y", "u", "bc", "bc_data", "u_one")], 1)  # noqa: E731
    it = iter(cst.data_loader)
    rows = np.concatenate([cat(next(it)[0]) for _ in range(5)])  # 240 samples in batches of 50: one epoch
    every = cat(ppsci.data.dataset.ChipHeatDataset(inp, {"chip": np.array([0.0])}, ("x", "u", "bc", "bc_data"), "u")[np.arange(240)][0])
    key = lambda a: np.lexsort(a.T[::-1])  # noqa: E731
    assert rows.shape == every.shape and np.array_equal(rows[key(rows)], every[key(every)])
    lab_b, wt_b = next(it)[1:]
    assert lab_b["chip"].shape == wt_b["chip"].shape == (50, 1) and float(wt_b["chip"][0]) == 500.0


# ---------------------------------------------------------------------------------------------------------------------
def _mlp_case(dtype, device, n=64):
    ppsci.utils.misc.set_random_seed(7)
    model = ppsci.arch.MLP(("x", "y"), ("T",), 2, 12, "tanh", dtype=dtype).to(device)
    with torch.no_grad():
        model.flat.data += 0.1 * torch.randn_like(model.flat.data)
    rng = np.random.RandomState(3)
    data = {"x": rng.rand(n, 1), "y": rng.rand(n, 1), "bc": rng.choice([0.0, 1.0, 2.0, 3.0], size=(n, 1)),
            "g": rng.randn(n, 1)}
    return model, {k: torch.as_tensor(v, dtype=dtype, device=device) for k, v in data.items()}


def _mlp_where(d, jac, safe):
    """The example's boundary selection with branches that are non-finite where they are not taken: T / (bc - 1) at
    bc = 1, T^2 / (bc - 2) at bc = 2 and log(bc - 2.5) for bc < 3.  ``safe`` guards them for the oracle, whose autograd
    through torch.where would otherwise multiply the untaken branch's infinite partials by zero."""
    bc = d["bc"]
    d1 = torch.where(bc == 1, bc + 1, bc - 1) if safe else bc - 1
    d2 = torch.where(bc == 2, bc + 1, bc - 2) if safe else bc - 2
    arg = torch.where(bc == 3, bc - 2.5, bc * 0 + 1) if safe else bc - 2.5
    return torch.where(bc == 1, jac(d["T"], d["x"]) - d["g"],
                       torch.where(bc == 0, d["T"] / d1 - d["g"],
                                   torch.where(bc == 2, jac(d["T"], d["y"]) + d["g"] * (d["T"] - 1),
                                               d["T"] * torch.log(arg) + d["T"] ** 2 / d2)))


def _mlp_oracle(model, inputs, fn, label):
    raw = model.flat.data.detach().cpu().double().clone().requires_grad_(True)
    om = O.OracleMLP(("x", "y"), ("T",), [12, 12], "tanh")
    x = {k: v.detach().cpu().double().clone().requires_grad_(k in ("x", "y")) for k, v in inputs.items()}
    data = dict(x)
    data.update(om(raw, {k: x[k] for k in ("x", "y")}))
    res = fn(data)
    loss = ((res - label) ** 2).mean()
    loss.backward()
    return float(loss.detach()), raw.grad, res.detach()


def _mlp_train(model, inputs, fn, label):
    cst = types.SimpleNamespace(name="c", loss=ppsci.loss.MSELoss("mean"), output_expr={"res": fn}, output_keys=("res",))
    fh = ppsci.utils.ExpressionSolver()
    lab = {"res": torch.full_like(inputs["x"], label)}
    losses_all, _ = fh.train_forward((cst.output_expr,), [inputs], model, {"c": cst}, [lab], [None])
    return float(losses_all["res"]), model.flat.grad.detach().cpu().double()


def test_mlp_where_residual_with_non_finite_untaken_branches_through_emulated_kernels(monkeypatch):
    _emul(monkeypatch)
    model, inputs = _mlp_case(torch.float64, "cpu")
    loss, grad = _mlp_train(model, inputs, lambda d: _mlp_where(d, ppsci.autodiff.jacobian, False), 0.25)
    o_loss, o_grad, _ = _mlp_oracle(model, inputs, lambda d: _mlp_where(d, O.jacobian, True), 0.25)
    assert np.isfinite(loss) and torch.isfinite(grad).all()
    assert abs(loss - o_loss) <= 1e-11 * abs(o_loss)
    np.testing.assert_allclose(grad.numpy(), o_grad.numpy(), rtol=1e-8, atol=1e-12 * float(o_grad.abs().max()))


def test_piecewise_sympy_residual_matches_the_oracle_evaluator(monkeypatch):
    """A residual given as a sympy Piecewise (as torch.where traces it) through the emulated kernels, against the
    oracle's eval_expr extended to Piecewise / Eq."""
    _emul(monkeypatch)
    model, inputs = _mlp_case(torch.float64, "cpu", n=40)
    x, y, bc, g = sp.symbols("x y bc g")
    T = sp.Function("T")(x, y)
    expr = sp.Piecewise((T.diff(x) - g, sp.Eq(bc, 1)), (T - g, sp.Eq(bc, 0)), (T.diff(y, 2) * T + g, True))
    loss, grad = _mlp_train(model, inputs, expr, 0.0)
    o_loss, o_grad, _ = _mlp_oracle(model, inputs, lambda d: eval_piecewise(expr, d), 0.0)
    assert abs(loss - o_loss) <= 1e-11 * abs(o_loss)
    np.testing.assert_allclose(grad.numpy(), o_grad.numpy(), rtol=1e-8, atol=1e-12 * float(o_grad.abs().max()))


def test_compiler_lowers_where_to_eq_and_select():
    from paddlescience_b200.engine.compiler import compile_residuals
    from tests.cases import make_net

    net = make_net(("x",), ("T",), [4], "tanh")
    x, bc = sp.symbols("x bc")
    T = sp.Function("T")(x)
    cr = compile_residuals(net, {"r": sp.Piecewise((T.diff(x), sp.Eq(bc, 1)), (sp.log(bc) * T, True))})
    ops = [op for op, *_ in cr.prog]
    assert B.OPS["eq"] in ops and B.OPS["select"] in ops
    # the untaken log(bc) is only ever an operand of a select: no op reads the register it lands in except a select
    with pytest.raises(NotImplementedError, match="final default branch"):
        compile_residuals(net, {"r": sp.Piecewise((T, sp.Eq(bc, 1)))})


# ---------------------------------------------------------------------------------------------------------------------
def _example():
    sys.path.insert(0, os.path.join(ROOT, "examples", "chip_heat"))
    try:
        import chip_heat as ex
    finally:
        sys.path.pop(0)
    return ex


def test_example_small_trains_two_iterations(monkeypatch):
    _emul(monkeypatch)
    from paddlescience_b200.optimizer.optimizer import FlatAdam

    def sgd_step(self):  # FlatAdam.step runs its fused kernel on the device only: a plain step stands in on the CPU
        with torch.no_grad():
            self.model.flat.data -= 1e-3 * self.model.flat.grad

    monkeypatch.setattr(FlatAdam, "step", sgd_step)
    res = _example().main(["--small", "--iters", "2", "--device", "cpu"])
    assert len(res["loss"]) == 2 and all(np.isfinite(res["loss"])) and np.isfinite(res["l2_rel"])


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("which", ["left", "interior"])
def test_example_shapes_fp32_on_gpu_match_oracle(which):
    """The example's sub-networks (9 x 256 swish branches on 324 / 76 / 1 sensors, a 6 x 128 swish trunk, F = 400),
    4,096 pairs with all four boundary types: a boundary constraint (C = 2) and the interior one (C = 5)."""
    hb, hbc, ht = [256] * 9, [256] * 9, [128] * 6
    model = _model(torch.float32, 400, hb, hbc, ht, num_loc=324, bc_loc=76, act="swish", bc_act="swish").to("cuda")
    ours, theirs = _both(EXAMPLE[which])
    data = _data(4096, num_loc=324, bc_loc=76)
    losses_all, _, o_losses, o_res, o_grad = _run(model, hb, hbc, ht, {"chip": ours}, {"chip": theirs}, data, "cuda",
                                                  torch.float32, {"chip": 0.0}, weights={"chip": "w"})
    inputs = {k: torch.as_tensor(data[k], dtype=torch.float32, device="cuda") for k in INPUTS}
    res = model.evaluate_expressions({"chip": ours}, inputs, ("u_one",))["chip"].cpu().double()
    assert float((res - o_res["chip"]).norm() / o_res["chip"].norm()) <= 1e-5
    assert abs(float(losses_all["chip"]) - float(o_losses["chip"])) <= 2e-5 * abs(float(o_losses["chip"]))
    got = model.flat.grad.detach().cpu().double()
    assert float((got - o_grad).norm() / o_grad.norm()) <= 5e-5


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["top", "right", "interior"])
def test_small_shapes_fp64_on_gpu_match_oracle(which):
    hb, hbc, ht = [16, 16], [12, 12], [12, 12]
    model = _model(torch.float64, 8, hb, hbc, ht, branch_weight_norm=True).to("cuda")
    ours, theirs = _both(EXAMPLE[which])
    data = _data(777)
    _, _, o_losses, o_res, o_grad = _run(model, hb, hbc, ht, {"chip": ours}, {"chip": theirs}, data, "cuda", torch.float64,
                                         {"chip": 0.0}, weights={"chip": "w"})
    inputs = {k: torch.as_tensor(data[k], device="cuda") for k in INPUTS}
    res = model.evaluate_expressions({"chip": ours}, inputs, ("u_one",))["chip"].cpu()
    assert float((res - o_res["chip"]).norm() / o_res["chip"].norm()) <= 1e-11
    got = model.flat.grad.detach().cpu()
    assert float((got - o_grad).norm() / o_grad.norm()) <= 1e-11


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-10), (torch.float32, 1e-4)])
def test_mlp_where_residual_on_gpu(dtype, tol):
    model, inputs = _mlp_case(dtype, "cuda", n=5000)
    loss, grad = _mlp_train(model, inputs, lambda d: _mlp_where(d, ppsci.autodiff.jacobian, False), 0.25)
    o_loss, o_grad, _ = _mlp_oracle(model, inputs, lambda d: _mlp_where(d, O.jacobian, True), 0.25)
    assert np.isfinite(loss) and torch.isfinite(grad).all()
    assert abs(loss - o_loss) <= tol * abs(o_loss)
    assert float((grad - o_grad).norm() / o_grad.norm()) <= tol


@pytest.mark.gpu
def test_example_solver_steps_on_gpu(tmp_path):
    """20 Adam steps of ppsci.solver.Solver on the example's small configuration: the loss on fixed batches goes down."""
    ex = _example()
    cfg = {**ex.CFG, **ex.SMALL}
    model, constraint, _, _ = ex.build(cfg, "cuda")
    fh = ppsci.utils.ExpressionSolver()
    to = lambda d: {k: v.to("cuda", model.dtype) for k, v in d.items()}  # noqa: E731
    fixed = []
    for c in constraint.values():  # every sample of the small product, one batch per constraint
        ds = c.data_loader.loader.ds
        fixed.append(tuple(to({k: torch.as_tensor(v) for k, v in d.items()}) for d in ds[np.arange(len(ds))]))

    def loss():
        losses, _ = fh.train_forward(tuple(c.output_expr for c in constraint.values()), [d[0] for d in fixed], model,
                                     constraint, [d[1] for d in fixed], [d[2] for d in fixed])
        model.flat.grad.zero_()
        return float(sum(losses.values()))

    before = loss()
    solver = ppsci.solver.Solver(model, constraint, str(tmp_path), ppsci.optimizer.Adam(cfg["lr"])(model), epochs=20,
                                 iters_per_epoch=1, log_freq=5)
    solver.train()
    after = loss()
    assert np.isfinite(before) and np.isfinite(after) and after < before, (before, after)
