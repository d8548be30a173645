"""CUDA-core tile GEMMs (k_gemm_fwd / dx / dw) and the thin first / last layer kernels (k_first_fwd / dw, k_last_fwd /
bwd, their vectorised twins in kernels_thin.cuh, k_omega_grad) one layer at a time, through the CPU emulation build of
the kernel sources, against the fp64 reference of tests/layer_ref.py on the exact values each kernel read.

Every case is an MLP with three linear layers (the last layer's dx lands in Zbar_2 beside Zbar_1), so one call checks
layer 1 from the input seeds (forward, dW, db, dLoss/d omega), layer 2 on the tile GEMMs (forward, dx, dW, db,
dLoss/d beta of layer 1's activation) and layer 3 (forward, dx, dW, db, dLoss/d beta of layer 2's).  Each case with a
thin first or last layer runs three times with the same inputs: by default, with PPSCI_B200_NO_THINV=1 (the generic
thin kernels) and with PPSCI_B200_NO_THIN=1 (the tile GEMMs).  The emulation runs every CUDA thread as an OS thread,
so the shapes stay small; tests/test_zzzzzz_layer_kernels.py sweeps the wide ones on the GPU."""
import pytest
import torch

from paddlescience_b200.engine import binding as B
from tests.emul.build_emul import build
from tests.layer_ref import THIN_MODES, U32, all_errors, all_layouts, last_chunk, run_fused, thin_kernels

U64 = 2.0 ** -53

# Bars in units of the componentwise bound (fwd, dW, db, d omega, d beta) or of the plane's largest |ref| (dx): about
# twice the largest error this file's matrix measured, fp64 16.0 units of 2^-53 (dw2, C = 17) and fp32 32.8 units of
# 2^-24 (fwd2 after a sigmoid: the fp32 closed-form activation coefficients, not the GEMM; the GEMM-only passes stay
# under 5).  A dropped K chunk, channel or point, or a wrong seed coefficient, is off by 2^20 units or more in fp64.
BAR = {torch.float64: 32.0, torch.float32: 66.0}

P_FIX = {"x": (2.0, False)}
P_TRAIN = {"x": (2.0, True)}
P_MANY = {"x": (2.0, True), "y": (1.5, False), "z": (3.0, True), "s": (2.5, True)}  # 9 features: A_SEED tile GEMM
P_ALL4 = {"t": (1.5, True), "x": (2.0, False), "y": (1.25, True), "z": (3.0, True)}  # 8 features = THIN_MAXF
P_T = {"t": (1.5, True)}  # 5 features


def _case(lay, hidden, n=37, dtype=torch.float64, **kw):
    return (lay, tuple(hidden), n, dtype, kw)


def _cases():
    out = []
    for lay in sorted(all_layouts()):  # every layout; C = 3, 4, 5, 7, 8, 17, 29 and 32
        n = 17 if all_layouts()[lay]["C"] > 17 else 37
        for dtype in (torch.float64, torch.float32):
            out.append(_case(lay, [12, 20], n, dtype))
    out += [
        # tile GEMM edges: fan-in not a multiple of KC = 16, fan-out past one column tile (TN = 64 / 128), pitch != width
        _case("O3", [20, 65]), _case("O3", [20, 70]), _case("O11", [36, 18]),
        _case("O3", [20, 130], dtype=torch.float32), _case("Lay12", [50, 70], dtype=torch.float32),
        # dW with two row blocks (K > TM = 128)
        _case("O2", [150, 20], n=9),
        # point counts: one, TP - 1 and TP + 1 (C = 5: TP = 25), a ragged last dW chunk (PT = 6)
        _case("O4", [12, 20], n=1), _case("O4", [12, 20], n=24), _case("O4", [12, 20], n=26, dtype=torch.float32),
        _case("Lay22", [12, 20], n=31, dtype=torch.float32),
        # thin first layer: nf = 1, 2, 5, 8, 9; N = 4, 18, 20; around PB = 32; fixed and trainable periods
        _case("O2", [4, 20]), _case("O11", [18, 12], dtype=torch.float32),
        _case("O1222", [20, 12], periods=P_T), _case("O1222", [20, 12], dtype=torch.float32, periods=P_ALL4),
        _case("O211", [20, 12], periods=P_MANY), _case("O211", [20, 12], dtype=torch.float32, periods=P_MANY),
        _case("Lay12", [20, 12], n=33, dtype=torch.float32, periods=P_FIX),
        _case("Lay12", [20, 12], n=64, dtype=torch.float32, periods=P_TRAIN),
        _case("Lay12", [18, 12], n=31, periods=P_TRAIN), _case("Lay4444", [12, 16], n=33, dtype=torch.float32, periods=P_TRAIN),
        # thin last layer: m = 1, 3, 4, 5, 8; C m = 64 (C = 8, m = 8) and 51 (C = 17, m = 3); K % 4 != 0
        _case("LayV", [12, 20], dtype=torch.float32, out_keys=("u", "v", "a")),
        _case("LayV", [12, 20], dtype=torch.float32, out_keys=("u", "v", "a", "b")),
        _case("LayV", [12, 18], dtype=torch.float32, out_keys=("u", "v", "a", "b", "c")),
        _case("O1222", [12, 20], n=17, dtype=torch.float32, out_keys=tuple("uabcdefg")),
        _case("Lay4444", [12, 20], n=17, out_keys=("u", "a", "b")),
        _case("Lay12", [12, 18], dtype=torch.float32),
        # every activation path with a parameter, and act_first != act
        _case("Lay22", [12, 20], act="stan"), _case("Lay22", [12, 20], dtype=torch.float32, act="stan"),
        _case("O3", [12, 20], act="swish_b"), _case("O3", [12, 20], dtype=torch.float32, act="swish_b", act_first="sin"),
        _case("Lay12", [12, 20], dtype=torch.float32, act="sin", act_first="tanh"),
        _case("O11", [12, 20], act="gelu"), _case("O2", [12, 20], dtype=torch.float32, act="sigmoid"),
    ]
    seen = []
    for c in out:
        if c not in seen:
            seen.append(c)
    return seen


CASES = _cases()


def _cid(c):
    lay, hidden, n, dtype, kw = c
    s = f"{lay}-h{'-'.join(map(str, hidden))}-n{n}-{'f64' if dtype == torch.float64 else 'f32'}"
    for k, v in sorted(kw.items()):
        s += f"-{k}_" + ("".join(v) if k == "out_keys" else
                         "".join(f"{p}{'T' if t else 'F'}" for p, (_, t) in v.items()) if k == "periods" else str(v))
    return s


@pytest.fixture(scope="module")
def emul_lib():
    return B.Library(build())


def _modes(plan):
    """The implementations to run: all three when the default plan has a thin first or last layer."""
    k = thin_kernels(plan)
    thin = k["first_fwd"] != "k_gemm_fwd" or k["last_fwd"] != "k_gemm_fwd"
    return list(THIN_MODES) if thin else ["default"]


def _run(lib, c, monkeypatch, mode, grads0=None, chunk_points=0):
    lay, hidden, n, dtype, kw = c
    with monkeypatch.context() as m:
        for k, v in THIN_MODES[mode].items():
            m.setenv(k, v)
        return run_fused(lay, list(hidden), n, dtype=dtype, backend=1, library=lib, device="cpu", seed=3,
                         grads0=grads0, chunk_points=chunk_points, **kw)


def _check(case, e, dtype):
    u = U64 if dtype == torch.float64 else U32
    e = {k: v / u for k, v in e.items()}
    print(f"\n[layer-kernels emul] {case}: " + " ".join(f"{k}={v:.2f}" for k, v in sorted(e.items())))
    bad = {k: v for k, v in e.items() if not v <= BAR[dtype]}
    assert not bad, f"{case}: {bad} (bar {BAR[dtype]})"
    return e


@pytest.mark.parametrize("case", CASES, ids=[_cid(c) for c in CASES])
def test_layer_kernels_emulated(emul_lib, monkeypatch, case):
    name = _cid(case)
    plan, params, grads, views = _run(emul_lib, case, monkeypatch, "default")
    modes = _modes(plan)
    del plan
    for mode in modes:
        plan, params, grads, views = _run(emul_lib, case, monkeypatch, mode)
        ks = thin_kernels(plan, THIN_MODES[mode])
        if mode == "no_thin":
            assert ks["first_fwd"] == "k_gemm_fwd" and ks["last_fwd"] == "k_gemm_fwd", ks
        e = all_errors(plan, params, grads, views)
        assert {"fwd1", "dw1", "db1", "fwd2", "dx2", "dw2", "fwd3", "dx3", "dw3", "db3"} <= set(e), e
        if plan.compiled.net.n_omega:
            assert "omega" in e
        # the stash is not all zeros (a wrong offset into zeroed memory would pass the comparisons)
        assert float(views["Zbar1"].abs().max()) > 0 and float(views["Ybar"].abs().max()) > 0
        _check(f"{name} [{mode}: {ks['first_fwd']} / {ks['last_fwd']}]", e, case[3])
        del plan, views


ACC_CASES = [_case("Lay12", [20, 12], dtype=torch.float32, periods=P_TRAIN),
             _case("O211", [20, 12], periods=P_MANY),
             _case("Lay22", [12, 20], act="stan"),
             _case("O3", [12, 20], dtype=torch.float32, act="swish_b")]


@pytest.mark.parametrize("case", ACC_CASES, ids=[_cid(c) for c in ACC_CASES])
def test_layer_kernels_accumulate_emulated(emul_lib, monkeypatch, case):
    """Seeded with G0, every block of the gradient (tile GEMM, thin first and last layer, d omega, d beta) must come
    out as G0 + its gradient: an overwritten block is off by |G0|."""
    name = "acc-" + _cid(case)
    _, _, g1, _ = _run(emul_lib, case, monkeypatch, "default")
    gen = torch.Generator().manual_seed(7)
    g0 = (torch.randn(g1.numel(), generator=gen, dtype=torch.float64) * float(g1.double().std())).to(case[3])
    plan, params, grads, views = _run(emul_lib, case, monkeypatch, "default", grads0=g0)
    for mode in _modes(plan):
        plan, params, grads, views = _run(emul_lib, case, monkeypatch, mode, grads0=g0)
        _check(f"{name} [{mode}]", all_errors(plan, params, grads, views, seed=g0), case[3])


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
def test_last_chunk_of_a_multi_chunk_call_emulated(emul_lib, monkeypatch, dtype):
    """A call over three workspace chunks: the seeds of the last chunk are read at x_off = 32, not 0."""
    n, ch = 37, 16
    case = _case("Lay12", [20, 12], n, dtype, periods=P_TRAIN)
    plan, params, grads, views = _run(emul_lib, case, monkeypatch, "default", chunk_points=ch)
    assert plan.chunk_points == ch and last_chunk(plan, n) == (32, 5)
    assert views["Z1"].shape[1] == 5
    e = all_errors(plan, params, grads, views, chunked=True)
    assert set(e) == {"fwd1", "fwd2", "dx2", "fwd3", "dx3"}, e
    _check(f"chunked-{_cid(case)}", e, dtype)
