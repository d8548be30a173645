// jet_layout.cuh — compile-time jet channel layouts for the vectorised fp32 kernels (kernels_thin.cuh).
//
// The vectorised kernels are instruction-bound, so the channel structure of the common PDE layouts is a template
// parameter (all index math folds into constants); plans with any other layout take the runtime-layout kernels.
#pragma once

#include "kernels_simt.cuh"

namespace ppsci {

template <int O0, int O1, int O2, int O3>
struct SLay {
  static constexpr int ND = (O0 > 0) + (O1 > 0) + (O2 > 0) + (O3 > 0);
  static constexpr int CS = 1 + O0 + O1 + O2 + O3;  // compile-time channel count
  static constexpr int KMAX = (O0 > O1 ? O0 : O1) > (O2 > O3 ? O2 : O3) ? (O0 > O1 ? O0 : O1) : (O2 > O3 ? O2 : O3);
  static constexpr int KM = KMAX < 1 ? 1 : KMAX;
  __device__ static __forceinline__ int order(const JetLayout&, int d) { return d == 0 ? O0 : d == 1 ? O1 : d == 2 ? O2 : O3; }
  __device__ static __forceinline__ int cbase(const JetLayout&, int d) {
    return 1 + (d > 0 ? O0 : 0) + (d > 1 ? O1 : 0) + (d > 2 ? O2 : 0);
  }
};

enum { LAY_DYN = 0, LAY_22 = 1, LAY_12 = 2, LAY_222 = 3, LAY_VALUE = 4 };
inline int pick_layout(const JetLayout& J, int act) {
  if (act != PPSCI_ACT_TANH) return LAY_DYN;
  auto is = [&](int n, int a, int b, int c) {
    return J.n_dir == n && (n < 1 || J.dir_order[0] == a) && (n < 2 || J.dir_order[1] == b) && (n < 3 || J.dir_order[2] == c);
  };
  if (is(2, 2, 2, 0)) return LAY_22;
  if (is(2, 1, 2, 0)) return LAY_12;
  if (is(3, 2, 2, 2)) return LAY_222;
  if (is(0, 0, 0, 0)) return LAY_VALUE;
  return LAY_DYN;
}

}  // namespace ppsci
