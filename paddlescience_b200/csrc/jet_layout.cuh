// jet_layout.cuh — jet channel layouts and the per-element jet step of every kernel: the activation jets of one
// (point, unit) element from its pre-activation jets (jet_fwd), and their adjoint (jet_adj).
//
// A layout policy names the channels of each Taylor direction d: order(J, d) coefficients of orders 1..order, at
// channels cbase(J, d) .. cbase(J, d) + order - 1; channel 0 is the value.  DynLay reads them from the plan's JetLayout
// at run time (any layout up to KMAX).  SLay fixes them at compile time: the vectorised fp32 kernels are
// instruction-bound, so for the common PDE layouts all index math folds into constants.  Host + device, so the same
// code is checked on the CPU (tests/test_jet_layouts.py).
#pragma once

#include <type_traits>
#include <utility>

#include "jet_math.h"
#include "ppsci_b200.h"

namespace ppsci {

struct JetLayout {
  int C;
  int n_dir;
  int dir_order[PPSCI_MAX_DIR];
  int dir_base[PPSCI_MAX_DIR];  // channel index of order-1 coefficient of direction d
};

template <int KMAX>
struct DynLay {
  static constexpr int KM = KMAX;
  PPSCI_HD static int n_dir(const JetLayout& J) { return J.n_dir; }
  PPSCI_HD static int order(const JetLayout& J, int d) { return J.dir_order[d]; }
  PPSCI_HD static int cbase(const JetLayout& J, int d) { return J.dir_base[d]; }
};

template <int O0, int O1, int O2, int O3>
struct SLay {
  static constexpr int ND = (O0 > 0) + (O1 > 0) + (O2 > 0) + (O3 > 0);
  static constexpr int CS = 1 + O0 + O1 + O2 + O3;  // compile-time channel count
  static constexpr int KMAX = (O0 > O1 ? O0 : O1) > (O2 > O3 ? O2 : O3) ? (O0 > O1 ? O0 : O1) : (O2 > O3 ? O2 : O3);
  static constexpr int KM = KMAX < 1 ? 1 : KMAX;
  PPSCI_HD static int n_dir(const JetLayout&) { return ND; }
  PPSCI_HD static int order(const JetLayout&, int d) { return d == 0 ? O0 : d == 1 ? O1 : d == 2 ? O2 : O3; }
  PPSCI_HD static int cbase(const JetLayout&, int d) { return 1 + (d > 0 ? O0 : 0) + (d > 1 ? O1 : 0) + (d > 2 ? O2 : 0); }
  // J has this layout's directions (its channel bases follow from the orders)
  PPSCI_HD static bool matches(const JetLayout& J) {
    bool ok = J.n_dir == ND;
    for (int d = 0; d < ND; ++d) ok = ok && J.dir_order[d] == order(J, d);
    return ok;
  }
};

// The compile-time layouts of the kernels: Navier-Stokes / Poisson in 2-D (Lay22) and 3-D (Lay222), a first-order time
// and a second-order space direction (Lay12), values only (LayV), and the polarised biharmonic operator (Lay4444).
using Lay22 = SLay<2, 2, 0, 0>;
using Lay12 = SLay<1, 2, 0, 0>;
using Lay222 = SLay<2, 2, 2, 0>;
using LayV = SLay<0, 0, 0, 0>;
using Lay4444 = SLay<4, 4, 4, 4>;

// The layouts each kernel family is instantiated for; with_lay picks among them.
template <class... Ls>
struct LayList {};
using ThinLays = LayList<Lay22, Lay12, Lay222, LayV>;           // kernels_thin.cuh
using WgLays = LayList<Lay22, Lay12, Lay222, LayV, Lay4444>;    // kernels_wgmma.cuh

// f(L{}) for the layout L of the list that J matches; false if none does
template <class... Ls, class F>
bool with_lay(LayList<Ls...>, const JetLayout& J, F&& f) {
  return ((Ls::matches(J) ? (f(Ls{}), true) : false) || ...);
}

// f(std::integral_constant<int, V>{}) for V = v in 1..MAX; false if v is outside
template <class F, int... I>
bool with_int_(int v, F& f, std::integer_sequence<int, I...>) {
  return ((v == I + 1 ? (f(std::integral_constant<int, I + 1>{}), true) : false) || ...);
}
template <int MAX, class F>
bool with_int(int v, F&& f) {
  return with_int_(v, f, std::make_integer_sequence<int, MAX>{});
}

// Channels 1..C-1 of y = act(z) for one element: channel c of z comes from ld(c), channel c of y goes to st(c, y_c).
// s[1..Lay::KM] from act_coef / act_coef_p at z0; the caller handles channel 0 (y0).
template <typename T, class Lay, typename Ld, typename St>
PPSCI_HD void jet_fwd(const JetLayout& J, const T (&s)[6], Ld ld, St st) {
#pragma unroll
  for (int d = 0; d < Lay::n_dir(J); ++d) {
    const int K = Lay::order(J, d), cb = Lay::cbase(J, d);
    T zz[4], yy[4];
#pragma unroll
    for (int o = 0; o < 4; ++o) zz[o] = (o < Lay::KM && o < K) ? ld(cb + o) : T(0);
    jet_fwd_dir<T, Lay::KM>(s, zz, yy);
#pragma unroll
    for (int o = 0; o < Lay::KM; ++o)
      if (o < K) st(cb + o, yy[o]);
  }
}

// Adjoint of y = act(z) for one element: channel c of z from ldz(c), of the adjoint of y from ldyb(c); the adjoint of z
// goes to st(c, zb_c) for c >= 1 and channel 0's is returned.  s[1..Lay::KM + 1] at z0.
template <typename T, class Lay, typename Ldz, typename Ldyb, typename St>
PPSCI_HD T jet_adj(const JetLayout& J, const T (&s)[6], Ldz ldz, Ldyb ldyb, St st) {
  T sb[5] = {T(0), T(0), T(0), T(0), T(0)};
#pragma unroll
  for (int d = 0; d < Lay::n_dir(J); ++d) {
    const int K = Lay::order(J, d), cb = Lay::cbase(J, d);
    T zz[4], yb[4], zb[4];
#pragma unroll
    for (int o = 0; o < 4; ++o) {
      const bool on = o < Lay::KM && o < K;
      zz[o] = on ? ldz(cb + o) : T(0);
      yb[o] = on ? ldyb(cb + o) : T(0);
      zb[o] = T(0);
    }
    jet_adj_dir<T, Lay::KM>(s, zz, yb, zb, sb);
#pragma unroll
    for (int o = 0; o < Lay::KM; ++o)
      if (o < K) st(cb + o, zb[o]);
  }
  return jet_adj_z0<T, Lay::KM>(s, ldyb(0), sb);
}

}  // namespace ppsci
