"""CPU check of the compile-time jet layouts (SLay, csrc/jet_layout.cuh) and of the picker that matches a plan's layout
to one of them.

The vectorised fp32 kernels and the tensor-core kernels take the per-element jet step (jet_fwd / jet_adj) through SLay,
whose index math folds into constants; every other kernel takes it through DynLay, which reads the plan's JetLayout and
is pinned against the fp64 reference by tests/test_layer_ref_emul.py.  Here both run on the host, on the same seeded
random jets, and must give bitwise the same activation jets and adjoints: for every layout a kernel family instantiates
(ThinLays, WgLays), every activation without a trainable parameter, fp32 and fp64, and activation coefficients up to the
order the step needs (NS = KM, as the forward kernels compute them) or one further (NS = KM + 1, as the adjoint kernels
do).  SLay<1, 2, 3, 4>, which no kernel takes, gives every direction a different order and base.

with_lay picks the kernel instance for a plan: it must pick a layout of the family exactly when that layout has the
plan's directions, orders and channel bases."""
import ctypes
import functools
import itertools

import numpy as np
import pytest

from tests.emul.build_emul import build_jet_layouts

MAXC = 32
N = 256
ACTS = range(12)  # jet_math.h ActId 0..11: the activations without a trainable parameter
FAMILIES = {"ThinLays": 0, "WgLays": 1}
STEP_FAMILY = 2  # the layouts of every family, then SLay<1, 2, 3, 4>
IntArr = ctypes.c_int * 8


@functools.lru_cache(maxsize=None)
def _lib():
    lib = ctypes.CDLL(build_jet_layouts())
    dp = ctypes.POINTER(ctypes.c_double)
    ip = ctypes.POINTER(ctypes.c_int)
    lib.jet_layout_info.argtypes = [ctypes.c_int, ctypes.c_int, ip, ip]
    lib.jet_layout_step.argtypes = [ctypes.c_int] * 5 + [ctypes.c_longlong, dp, dp, dp, dp]
    lib.jet_layout_pick.argtypes = [ctypes.c_int, ctypes.c_int, ip, ip, ip]
    return lib


def _family(family):
    """[(index, orders, bases)] of the layouts of a family, as SLay reports them."""
    out = []
    for i in itertools.count():
        orders, bases = IntArr(), IntArr()
        nd = _lib().jet_layout_info(family, i, orders, bases)
        if nd < 0:
            return out
        out.append((i, tuple(orders[:nd]), tuple(bases[:nd])))


def _step_layouts():
    """name -> (harness index, direction orders), each layout once: Lay22, ..., LayV (no directions)"""
    out = {}
    for i, orders, _ in _family(STEP_FAMILY):
        out.setdefault("Lay" + ("".join(map(str, orders)) or "V"), (i, orders))
    return out


LAYOUTS = _step_layouts()  # builds the harness at collection: the layout lists of csrc/jet_layout.cuh name the tests


def _step(lay, dyn, dbl, ns_plus, act, z, yb):
    dp = ctypes.POINTER(ctypes.c_double)
    y = np.full((N, MAXC), np.nan)  # sentinel: channels the step must not write
    zb = np.full((N, MAXC), np.nan)
    ptr = lambda a: a.ctypes.data_as(dp)  # noqa: E731
    C = _lib().jet_layout_step(lay, dyn, dbl, ns_plus, act, N, ptr(z), ptr(yb), ptr(y), ptr(zb))
    return C, y, zb


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
def test_static_layout_matches_runtime_layout(name, dtype):
    lay, orders = LAYOUTS[name]
    dbl = int(dtype == np.float64)
    z, yb, C = _jets(orders, dtype, seed=list(LAYOUTS).index(name))
    for act in ACTS:
        for ns_plus in (0, 1):
            Cs, ys, zbs = _step(lay, 0, dbl, ns_plus, act, z, yb)
            Cd, yd, zbd = _step(lay, 1, dbl, ns_plus, act, z, yb)
            assert Cs == Cd == C
            where = f"{name} act {act} NS = KM{' + 1' if ns_plus else ''}"
            # every channel of the layout is written, none past it
            assert not np.isnan(yd[:, :C]).any() and np.isnan(yd[:, C:]).all(), where
            assert not np.isnan(zbd[:, :C]).any() and np.isnan(zbd[:, C:]).all(), where
            assert np.array_equal(ys.view(np.uint64), yd.view(np.uint64)), f"activation jets differ: {where}"
            assert np.array_equal(zbs.view(np.uint64), zbd.view(np.uint64)), f"adjoints differ: {where}"


def _pick(family, orders):
    """(direction count, orders, bases) of the layout with_lay picks for the plan layout of these direction orders"""
    o, bases = IntArr(), IntArr()
    nd = _lib().jet_layout_pick(family, len(orders), IntArr(*orders), o, bases)
    return None if nd < 0 else (nd, tuple(o[:nd]), tuple(bases[:nd]))


@pytest.mark.parametrize("family", list(FAMILIES))
def test_layout_picker(family):
    fam = FAMILIES[family]
    members = [(len(orders), orders, bases) for _, orders, bases in _family(fam)]
    # every layout of up to 4 directions of orders 1..4 (341), and a few of 5..8 directions, some of which begin with the
    # directions of a family member
    plans = [o for nd in range(5) for o in itertools.product(range(1, 5), repeat=nd)]
    plans += [(2, 2, 2, 2, 2), (4, 4, 4, 4, 4), (2, 2, 1, 1, 1, 1), (1, 2, 1, 2, 1, 2, 1), (1,) * 8]
    bad = []
    for orders in plans:
        bases = tuple(1 + sum(orders[:d]) for d in range(len(orders)))
        want = (len(orders), orders, bases)
        got = _pick(fam, orders)
        if got != (want if want in members else None):
            bad.append((orders, got))
    assert not bad, f"{len(bad)} of {len(plans)} plan layouts picked wrongly (orders, picked): {bad[:8]}"
    # the orders of Lay12 in the other order, and four directions with one of order 3, are no layout of a family
    assert _pick(fam, (2, 1)) is None
    assert _pick(fam, (4, 4, 3, 4)) is None and _pick(fam, (4, 4, 4, 3)) is None
