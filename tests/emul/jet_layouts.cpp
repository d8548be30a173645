// Host harness of tests/test_jet_layouts.py: the per-element jet step (jet_fwd, jet_adj) of jet_layout.cuh through a
// compile-time layout (SLay) or through the runtime layout (DynLay) of the same channel structure.
#include "jet_layout.cuh"

using namespace ppsci;

namespace {

constexpr int MAXC = 32;

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

// The JetLayout is built from the direction orders as the engine builds it, independently of SLay's index math.
template <int O0, int O1, int O2, int O3>
int dispatch(int dyn, int dbl, int ns_plus, int act, long long n, const double* z, const double* yb, double* y,
             double* zb) {
  using L = SLay<O0, O1, O2, O3>;
  const int orders[4] = {O0, O1, O2, O3};
  JetLayout J{};
  J.C = 1;
  for (int d = 0; d < 4 && orders[d] > 0; ++d) {
    J.dir_order[d] = orders[d];
    J.dir_base[d] = J.C;
    J.C += orders[d];
    J.n_dir = d + 1;
  }
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

// lay: 0 Lay22, 1 Lay12, 2 Lay222, 3 LayV, 4 Lay4444 (the kernels' layouts), 5 SLay<1, 2, 3, 4> (every direction of a
// different order).  dyn: DynLay instead of SLay.  ns_plus: act_coef with NS = KM + 1 instead of KM.  Returns C.
extern "C" int jet_layout_step(int lay, int dyn, int dbl, int ns_plus, int act, long long n, const double* z,
                               const double* yb, double* y, double* zb) {
  switch (lay) {
    case 0: return dispatch<2, 2, 0, 0>(dyn, dbl, ns_plus, act, n, z, yb, y, zb);
    case 1: return dispatch<1, 2, 0, 0>(dyn, dbl, ns_plus, act, n, z, yb, y, zb);
    case 2: return dispatch<2, 2, 2, 0>(dyn, dbl, ns_plus, act, n, z, yb, y, zb);
    case 3: return dispatch<0, 0, 0, 0>(dyn, dbl, ns_plus, act, n, z, yb, y, zb);
    case 4: return dispatch<4, 4, 4, 4>(dyn, dbl, ns_plus, act, n, z, yb, y, zb);
    case 5: return dispatch<1, 2, 3, 4>(dyn, dbl, ns_plus, act, n, z, yb, y, zb);
    default: return -1;
  }
}
