// Host harness of tests/test_jet_layouts.py: the per-element jet step (jet_fwd, jet_adj) of jet_layout.cuh through a
// compile-time layout (SLay) or through the runtime layout (DynLay) of the same channel structure, and the layout
// picker with_lay over the kernel families' layout lists.
#include "jet_layout.cuh"

using namespace ppsci;

namespace {

constexpr int MAXC = 32;

// family 0: ThinLays, 1: WgLays, 2: the layouts of the jet-step test, i.e. those of every family, plus SLay<1, 2, 3, 4>
// (every direction of a different order, which no kernel takes)
template <class... A, class... B, class... C>
LayList<A..., B..., C...> cat(LayList<A...>, LayList<B...>, LayList<C...>);
using StepLays = decltype(cat(WgLays{}, ThinLays{}, LayList<SLay<1, 2, 3, 4>>{}));

// f(L{}) for the i-th layout L of the list; false past its end
template <class... Ls, class F>
bool with_nth(LayList<Ls...>, int i, F&& f) {
  int k = 0;
  return ((k++ == i ? (f(Ls{}), true) : false) || ...);
}
template <class F>
bool with_family(int family, int i, F&& f) {
  return family == 0 ? with_nth(ThinLays{}, i, f) : family == 1 ? with_nth(WgLays{}, i, f) : with_nth(StepLays{}, i, f);
}

// direction count of layout L; its orders and channel bases -> orders[d], bases[d]
template <class L>
int describe(int* orders, int* bases) {
  const JetLayout J{};
  for (int d = 0; d < L::n_dir(J); ++d) {
    orders[d] = L::order(J, d);
    bases[d] = L::cbase(J, d);
  }
  return L::n_dir(J);
}

// The JetLayout of n_dir directions of the given orders, built as the engine builds it, independently of SLay's index math.
JetLayout make_layout(int n_dir, const int* orders) {
  JetLayout J{};
  J.C = 1;
  J.n_dir = n_dir;
  for (int d = 0; d < PPSCI_MAX_DIR; ++d) {
    J.dir_order[d] = d < n_dir ? orders[d] : 0;
    J.dir_base[d] = J.C;
    if (d < n_dir) J.C += orders[d];
  }
  return J;
}

// One element per row of z / yb ([n][MAXC], channels past the layout's C ignored).  Outputs y = act(z) jets and zb,
// the adjoint of z, are [n][MAXC] too; channels the step does not write keep the sentinel the caller filled in.
template <class Lay, typename T, int NS>
void run(const JetLayout& J, int act, long long n, const double* z, const double* yb, double* y, double* zb) {
  for (long long i = 0; i < n; ++i) {
    T zi[MAXC], ybi[MAXC], yo[MAXC], zbo[MAXC];
    for (int c = 0; c < MAXC; ++c) {
      zi[c] = c < J.C ? T(z[i * MAXC + c]) : T(0);
      ybi[c] = c < J.C ? T(yb[i * MAXC + c]) : T(0);
      yo[c] = T(y[i * MAXC + c]);
      zbo[c] = T(zb[i * MAXC + c]);
    }
    T s[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
    act_coef<T, NS>(act, zi[0], yo[0], s);
    auto ldz = [&](int c) { return zi[c]; };
    jet_fwd<T, Lay>(J, s, ldz, [&](int c, T v) { yo[c] = v; });
    zbo[0] = jet_adj<T, Lay>(J, s, ldz, [&](int c) { return ybi[c]; }, [&](int c, T v) { zbo[c] = v; });
    for (int c = 0; c < MAXC; ++c) {
      y[i * MAXC + c] = double(yo[c]);
      zb[i * MAXC + c] = double(zbo[c]);
    }
  }
}

template <class L>
int step(int dyn, int dbl, int ns_plus, int act, long long n, const double* z, const double* yb, double* y, double* zb) {
  int orders[4], bases[4];
  const JetLayout J = make_layout(describe<L>(orders, bases), orders);
  using D = DynLay<L::KM>;
  constexpr int NS = L::KM;
  if (dbl) {
    if (dyn) ns_plus ? run<D, double, NS + 1>(J, act, n, z, yb, y, zb) : run<D, double, NS>(J, act, n, z, yb, y, zb);
    else ns_plus ? run<L, double, NS + 1>(J, act, n, z, yb, y, zb) : run<L, double, NS>(J, act, n, z, yb, y, zb);
  } else {
    if (dyn) ns_plus ? run<D, float, NS + 1>(J, act, n, z, yb, y, zb) : run<D, float, NS>(J, act, n, z, yb, y, zb);
    else ns_plus ? run<L, float, NS + 1>(J, act, n, z, yb, y, zb) : run<L, float, NS>(J, act, n, z, yb, y, zb);
  }
  return J.C;
}

}  // namespace

// Layout i of family (see above): returns its direction count and writes its orders and channel bases, -1 past the end.
extern "C" int jet_layout_info(int family, int i, int* orders, int* bases) {
  int nd = -1;
  with_family(family, i, [&](auto lay) { nd = describe<decltype(lay)>(orders, bases); });
  return nd;
}

// The jet step through layout i of family 2.  dyn: DynLay instead of SLay.  ns_plus: act_coef with NS = KM + 1 instead
// of KM.  Returns C, -1 past the end of the list.
extern "C" int jet_layout_step(int i, int dyn, int dbl, int ns_plus, int act, long long n, const double* z,
                               const double* yb, double* y, double* zb) {
  int C = -1;
  with_family(2, i, [&](auto lay) { C = step<decltype(lay)>(dyn, dbl, ns_plus, act, n, z, yb, y, zb); });
  return C;
}

// with_lay over family 0 or 1 for the JetLayout of n_dir directions of the given orders: the direction count, orders and
// channel bases of the layout it picks, -1 if it picks none.
extern "C" int jet_layout_pick(int family, int n_dir, const int* orders, int* orders_out, int* bases_out) {
  const JetLayout J = make_layout(n_dir, orders);
  int nd = -1;
  auto f = [&](auto lay) { nd = describe<decltype(lay)>(orders_out, bases_out); };
  if (family == 0) with_lay(ThinLays{}, J, f);
  if (family == 1) with_lay(WgLays{}, J, f);
  return nd;
}
