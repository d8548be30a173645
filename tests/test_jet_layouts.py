"""CPU check of the compile-time jet layouts (SLay, csrc/jet_layout.cuh).

The vectorised fp32 kernels and the tensor-core kernels take the per-element jet step (jet_fwd / jet_adj) through SLay,
whose index math folds into constants; every other kernel takes it through DynLay, which reads the plan's JetLayout and
is pinned against the fp64 reference by tests/test_layer_ref_emul.py.  Here both run on the host, on the same seeded
random jets, and must give bitwise the same activation jets and adjoints: for every layout a kernel instantiates, every
activation without a trainable parameter, fp32 and fp64, and activation coefficients up to the order the step needs
(NS = KM, as the forward kernels compute them) or one further (NS = KM + 1, as the adjoint kernels do).  SLay<1, 2, 3, 4>,
which no kernel takes, gives every direction a different order and base."""
import ctypes

import numpy as np
import pytest

from tests.emul.build_emul import build_jet_layouts

MAXC = 32
N = 256
# harness layout id -> direction orders
LAYOUTS = {"Lay22": (0, (2, 2)), "Lay12": (1, (1, 2)), "Lay222": (2, (2, 2, 2)), "LayV": (3, ()),
           "Lay4444": (4, (4, 4, 4, 4)), "Lay1234": (5, (1, 2, 3, 4))}
ACTS = range(12)  # jet_math.h ActId 0..11: the activations without a trainable parameter


@pytest.fixture(scope="module")
def step():
    fn = ctypes.CDLL(build_jet_layouts()).jet_layout_step
    dp = ctypes.POINTER(ctypes.c_double)
    fn.argtypes = [ctypes.c_int] * 5 + [ctypes.c_longlong, dp, dp, dp, dp]
    fn.restype = ctypes.c_int

    def run(lay, dyn, dbl, ns_plus, act, z, yb):
        y = np.full((N, MAXC), np.nan)  # sentinel: channels the step must not write
        zb = np.full((N, MAXC), np.nan)
        ptr = lambda a: a.ctypes.data_as(dp)  # noqa: E731
        C = fn(lay, dyn, dbl, ns_plus, act, N, ptr(z), ptr(yb), ptr(y), ptr(zb))
        return C, y, zb

    return run


def _jets(orders, dtype, seed):
    rng = np.random.default_rng(seed)
    C = 1 + sum(orders)
    z = np.zeros((N, MAXC))
    yb = np.zeros((N, MAXC))
    z[:, 0] = rng.uniform(-2.5, 2.5, N)  # covers both branches of relu / elu / leaky_relu
    z[:, 1:C] = rng.normal(0.0, 0.7, (N, C - 1))
    yb[:, :C] = rng.normal(0.0, 1.0, (N, C))
    return z.astype(dtype).astype(np.float64), yb.astype(dtype).astype(np.float64), C


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", list(LAYOUTS))
def test_static_layout_matches_runtime_layout(step, name, dtype):
    lay, orders = LAYOUTS[name]
    dbl = int(dtype == np.float64)
    z, yb, C = _jets(orders, dtype, seed=lay)
    for act in ACTS:
        for ns_plus in (0, 1):
            Cs, ys, zbs = step(lay, 0, dbl, ns_plus, act, z, yb)
            Cd, yd, zbd = step(lay, 1, dbl, ns_plus, act, z, yb)
            assert Cs == Cd == C
            where = f"{name} act {act} NS = KM{' + 1' if ns_plus else ''}"
            # every channel of the layout is written, none past it
            assert not np.isnan(yd[:, :C]).any() and np.isnan(yd[:, C:]).all(), where
            assert not np.isnan(zbd[:, :C]).any() and np.isnan(zbd[:, C:]).all(), where
            assert np.array_equal(ys.view(np.uint64), yd.view(np.uint64)), f"activation jets differ: {where}"
            assert np.array_equal(zbs.view(np.uint64), zbd.view(np.uint64)), f"adjoints differ: {where}"
