"""``DeepONet`` (reference: ppsci/arch/deeponet.py:28-154; BASELINE cfg5): branch / trunk MLPs in the native kernels,
product + loss in torch, weight gradients through ``ppsci_b200_values_fwd_bwd``.

CPU: the full fused training call runs through the emulation build of the same kernel sources and is compared with the
oracle under autograd (fp64).  GPU: the cfg5 shapes (100 -> 128x3 -> 128, 1 -> 128x3 -> 128) in fp32."""
import numpy as np
import pytest
import torch

import ppsci
from oracle import ppsci_oracle as O
from paddlescience_b200.engine import binding as B


def _setup(dtype, device, n, num_loc, feats, hidden, seed=5, weights=True, **options):
    ppsci.utils.misc.set_random_seed(seed)
    model = ppsci.arch.DeepONet("u", "y", "G", num_loc, feats, None, None, tuple(hidden), tuple(hidden), dtype=dtype, **options)
    with torch.no_grad():
        model.flat.data += 0.05 * torch.randn_like(model.flat.data)
    model.to(device)
    rng = np.random.RandomState(seed)
    data = {"u": rng.randn(n, num_loc), "y": rng.rand(n, 1), "G": rng.randn(n, 1), "w": rng.rand(n, 1) + 0.5}
    np_dtype = np.float64 if dtype == torch.float64 else np.float32
    cst = ppsci.constraint.SupervisedConstraint(
        {"dataset": {"name": "IterableNamedArrayDataset", "input": {k: data[k].astype(np_dtype) for k in ("u", "y")},
                     "label": {"G": data["G"].astype(np_dtype)},
                     "weight": {"G": data["w"].astype(np_dtype)} if weights else None},
         "batch_size": n}, ppsci.loss.MSELoss("mean"), name="Sup")
    return model, cst, data


def _effective(model, raw, r):
    """Independent restatement of the sub-network reparametrisation: W = g V / ||V||_col on weight-normalised hidden
    layers (mlp.py:31-53), doubled pre-activation at even hidden layers >= 2 under skip_connection (mlp.py:281-296)."""
    sub = raw[r.lo: r.lo + r.n]
    parts = []
    for i, (a, b) in enumerate(r.shapes):
        w = sub[r.w_off[i]: r.w_off[i] + a * b].view(a, b)
        bias = sub[r.b_off[i]: r.b_off[i] + b]
        if r.weight_norm and i < len(r.shapes) - 1:
            g = raw[r.g_off[i]: r.g_off[i] + b]
            w = g * w / torch.sqrt((w * w).sum(dim=0, keepdim=True))
        if i in r.skip_layers:
            w, bias = 2 * w, 2 * bias
        parts += [w.reshape(-1), bias]
    return torch.cat(parts)


def _oracle(model, cst, hidden, weights=True):
    ds = cst.data_loader.loader  # the tensors the constraint actually delivers (weights are stored in the default dtype)
    data = {"u": ds.input["u"].cpu(), "y": ds.input["y"].cpu(), "G": ds.label["G"].cpu(),
            "w": ds.weight["G"].cpu() if weights else None}
    od = O.OracleDeepONet(model.num_loc, model.num_features, hidden, hidden)
    raw = model.flat.detach().cpu().double().clone().requires_grad_(True)
    pb = _effective(model, raw, model._rb)
    pt = _effective(model, raw, model._rt)
    b = raw[model._bias_off: model._bias_off + 1]
    g = od(pb, pt, b, torch.as_tensor(data["u"]).double(), torch.as_tensor(data["y"]).double())
    sq = (g - torch.as_tensor(data["G"]).double()) ** 2
    if weights:
        sq = sq * torch.as_tensor(data["w"]).double()
    loss = sq.mean()
    loss.backward()
    return g.detach(), float(loss.detach()), raw.grad


def _train_forward(model, cst, device, dtype):
    ds = cst.data_loader.loader
    to = lambda d: None if d is None else {k: v.to(device, dtype) for k, v in d.items()}  # noqa: E731
    fh = ppsci.utils.ExpressionSolver()
    losses_all, losses_cst = fh.train_forward((cst.output_expr,), [to(ds.input)], model, {"Sup": cst}, [to(ds.label)],
                                              [to(ds.weight)])
    return losses_all, losses_cst


def test_constructor_layout_and_unsupported_flags():
    m = ppsci.arch.DeepONet("u", "y", "G", 100, 40, 1, 1, 40, 40, branch_activation="relu", trunk_activation="relu")
    assert m.input_keys == ("u", "y") and m.output_keys == ("G",)
    assert m.num_params == (100 * 40 + 40) + (40 * 40 + 40) + (1 * 40 + 40) + (40 * 40 + 40) + 1
    sd = m.state_dict()
    assert sd["branch_net.linears.0.weight"].shape == (100, 40) and sd["trunk_net.last_fc.weight"].shape == (40, 40)
    assert float(sd["b"]) == 0.0 and float(sd["branch_net.linears.0.bias"].abs().max()) == 0.0
    m2 = ppsci.arch.DeepONet("u", "y", "G", 100, 40, 1, 1, 40, 40, branch_activation="relu", trunk_activation="relu")
    m2.load_state_dict(sd)
    np.testing.assert_array_equal(m2.flat.data.numpy(), m.flat.data.numpy())
    with pytest.raises(NotImplementedError):
        ppsci.arch.DeepONet("u", "y", "G", 10, 8, 1, 1, 8, 8, branch_weight_norm=True, branch_skip_connection=True)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m({"u": torch.zeros(3, 100), "y": torch.zeros(3, 1)})


@pytest.mark.parametrize("weights", [True, False])
def test_fused_training_call_through_emulated_kernels_matches_oracle(monkeypatch, weights):
    from tests.emul.build_emul import build

    monkeypatch.setattr(B, "_default", B.Library(build()))  # test infrastructure: same kernel sources, compiled for the CPU
    hidden = [16, 16]
    model, cst, data = _setup(torch.float64, "cpu", 53, 10, 12, hidden, weights=weights)
    losses_all, losses_cst = _train_forward(model, cst, "cpu", torch.float64)
    _, loss, grad = _oracle(model, cst, hidden, weights=weights)
    assert abs(float(losses_all["G"]) - loss) <= 1e-12 * abs(loss)
    assert abs(float(losses_cst["Sup"]) - loss) <= 1e-12 * abs(loss)
    np.testing.assert_allclose(model.flat.grad.numpy(), grad.numpy(), rtol=1e-9, atol=1e-13 * float(grad.abs().max()))
    # a second call accumulates (update_freq > 1)
    _train_forward(model, cst, "cpu", torch.float64)
    np.testing.assert_allclose(model.flat.grad.numpy(), 2 * grad.numpy(), rtol=1e-9, atol=1e-13 * float(grad.abs().max()))


@pytest.mark.parametrize("options", [dict(branch_weight_norm=True, trunk_weight_norm=True),
                                     dict(branch_skip_connection=True, trunk_skip_connection=True),
                                     dict(branch_weight_norm=True, trunk_skip_connection=True)])
def test_subnet_weight_norm_and_skip_connection_through_emulated_kernels(monkeypatch, options):
    """``*_weight_norm`` / ``*_skip_connection`` (deeponet.py:96-119 hands them to the two MLPs): host-side
    reparametrisation around the unchanged native calls, checked against the oracle with the reparametrisation under
    autograd; reference-style checkpoint keys."""
    from tests.emul.build_emul import build

    monkeypatch.setattr(B, "_default", B.Library(build()))
    hidden = [12, 12, 12]
    model, cst, data = _setup(torch.float64, "cpu", 41, 7, 9, hidden, **options)
    with torch.no_grad():
        model.flat.data += 0.05 * torch.randn_like(model.flat.data)  # gains off 1
    losses_all, _ = _train_forward(model, cst, "cpu", torch.float64)
    _, loss, grad = _oracle(model, cst, hidden)
    assert abs(float(losses_all["G"]) - loss) <= 1e-12 * abs(loss)
    np.testing.assert_allclose(model.flat.grad.numpy(), grad.numpy(), rtol=1e-8, atol=1e-12 * float(grad.abs().max()))
    sd = model.state_dict()
    if options.get("branch_weight_norm"):
        assert "branch_net.linears.0.weight_v" in sd and "branch_net.linears.0.weight_g" in sd and "branch_net.last_fc.weight" in sd
    m2 = ppsci.arch.DeepONet("u", "y", "G", 7, 9, None, None, tuple(hidden), tuple(hidden), dtype=torch.float64, **options)
    m2.load_state_dict(sd)
    sd2 = m2.state_dict()  # (the flat buffer has alignment gaps between the sub-networks that no key covers)
    assert list(sd2) == list(sd) and all(torch.equal(sd2[k], sd[k]) for k in sd)


@pytest.mark.gpu
@pytest.mark.parametrize("options", [{}, dict(branch_weight_norm=True, trunk_skip_connection=True)])
def test_cfg5_shapes_on_gpu_match_oracle(options):
    hidden = [128, 128, 128]
    model, cst, data = _setup(torch.float32, "cuda", 4096, 100, 128, hidden, **options)
    g = model({"u": torch.as_tensor(data["u"], dtype=torch.float32, device="cuda"),
               "y": torch.as_tensor(data["y"], dtype=torch.float32, device="cuda")})["G"]
    losses_all, _ = _train_forward(model, cst, "cuda", torch.float32)
    g_ref, loss, grad = _oracle(model, cst, hidden)
    assert float((g.cpu().double() - g_ref).norm() / g_ref.norm()) <= 1e-5
    assert abs(float(losses_all["G"]) - loss) <= 2e-5 * abs(loss)
    got = model.flat.grad.detach().cpu().double()
    assert float((got - grad).norm() / grad.norm()) <= 5e-5
