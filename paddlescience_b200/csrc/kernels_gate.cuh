// kernels_gate.cuh — the gating step of ModifiedMLP (ppsci/arch/mlp.py:488-506) on Taylor jets.
//
//   reference, per hidden layer:   y = act(linear(y));   y = y * u + (1 - y) * v
//   with u = act(embed_u(x)), v = act(embed_v(x)) computed once per batch.
//
// On jets the products are truncated Cauchy products along every direction (normalised Taylor coefficients:
// (a b)_k = sum_j a_j b_{k-j}); channel 0 (the value) is shared by all directions.  One thread owns one (point, unit)
// element with all of its C channels, so the adjoint runs in place and the U / V adjoints of successive layers add up
// without atomics (the launches of one chunk are ordered on the stream).
//
//   k_gate_fwd : G_l = V + act(Z_l) (U - V)                       (U, V re-derived from Zu, Zv: 2 x C loads, no stash)
//   k_gate_bwd : in  Gbar_l (adjoint of G_l)
//                out Zbar_l (in place), Zubar += , Zvbar +=       (adjoints of the PRE-activations: the activation's
//                adjoint is linear in its seed, so the per-layer contributions can be pushed through it one by one)
#pragma once

#include "kernels_simt.cuh"

namespace ppsci {

template <typename T>
struct GateArgs {
  JetLayout J;
  int act;
  const T* Z;   // [C][Np][ld] pre-activations of the hidden layer
  const T* Zu;  // [C][Np][ld] pre-activations of embed_u
  const T* Zv;
  T* G;         // fwd: gated jets out;  bwd: Gbar in -> Zbar out (in place)
  T* Zub;       // bwd: accumulated adjoint of Zu
  T* Zvb;
  int ld;
  long long plane;  // chunk points (allocated) * ld
  long long Np;     // valid points
  int H;
  int first;  // bwd: first gate of the chunk's adjoint pass -> Zub / Zvb are written, not accumulated
};

constexpr int GATE_MAXC = 32;

// z jets of one element -> y = act(z) jets (+ the activation's Taylor coefficients s[1..KMAX+1] at z0)
template <typename T, int KMAX>
__device__ __forceinline__ void gate_act_jet(int act, const JetLayout& J, const T* z, long long plane, T (&zj)[GATE_MAXC],
                                             T (&y)[GATE_MAXC], T (&s)[6]) {
  T y0;
  zj[0] = z[0];
  act_coef<T, KMAX + 1>(act, zj[0], y0, s);
  y[0] = y0;
  jet_fwd<T, DynLay<KMAX>>(J, s, [&](int c) { return zj[c] = z[(long long)c * plane]; }, [&](int c, T v) { y[c] = v; });
}

// adjoint of y = act(z): yb -> zb, stored (accumulate = false) or added (true) at out[c * plane]
template <typename T, int KMAX>
__device__ __forceinline__ void gate_act_adj(const JetLayout& J, const T (&s)[6], const T (&zj)[GATE_MAXC],
                                             const T (&yb)[GATE_MAXC], T* out, long long plane, bool accumulate) {
  auto put = [&](int c, T v) {
    T* o = out + (long long)c * plane;
    *o = accumulate ? *o + v : v;
  };
  put(0, jet_adj<T, DynLay<KMAX>>(J, s, [&](int c) { return zj[c]; }, [&](int c) { return yb[c]; }, put));
}

template <typename T, int KMAX>
__global__ void __launch_bounds__(128) k_gate_fwd(GateArgs<T> g) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= g.Np * g.H) return;
  const long long p = idx / g.H;
  const int h = (int)(idx % g.H);
  const long long e = p * g.ld + h;
  T zj[GATE_MAXC], y[GATE_MAXC], u[GATE_MAXC], v[GATE_MAXC], s[6];
  gate_act_jet<T, KMAX>(g.act, g.J, g.Z + e, g.plane, zj, y, s);
  gate_act_jet<T, KMAX>(g.act, g.J, g.Zu + e, g.plane, zj, u, s);
  gate_act_jet<T, KMAX>(g.act, g.J, g.Zv + e, g.plane, zj, v, s);
  T* out = g.G + e;
  const T y0 = y[0], d0 = u[0] - v[0];
  out[0] = v[0] + y0 * d0;
  for (int d = 0; d < g.J.n_dir; ++d) {
    const int K = g.J.dir_order[d];
    const int b = g.J.dir_base[d] - 1;  // channel of order k = b + k
    for (int k = 1; k <= K; ++k) {
      T acc = v[b + k] + y0 * (u[b + k] - v[b + k]) + y[b + k] * d0;
      for (int j = 1; j < k; ++j) acc += y[b + j] * (u[b + k - j] - v[b + k - j]);
      out[(long long)(b + k) * g.plane] = acc;
    }
  }
}

template <typename T, int KMAX>
__global__ void __launch_bounds__(128) k_gate_bwd(GateArgs<T> g) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= g.Np * g.H) return;
  const long long p = idx / g.H;
  const int h = (int)(idx % g.H);
  const long long e = p * g.ld + h;
  const int C = g.J.C;
  T zy[GATE_MAXC], zu[GATE_MAXC], zv[GATE_MAXC], y[GATE_MAXC], u[GATE_MAXC], v[GATE_MAXC], sy[6], su[6], sv[6];
  gate_act_jet<T, KMAX>(g.act, g.J, g.Z + e, g.plane, zy, y, sy);
  gate_act_jet<T, KMAX>(g.act, g.J, g.Zu + e, g.plane, zu, u, su);
  gate_act_jet<T, KMAX>(g.act, g.J, g.Zv + e, g.plane, zv, v, sv);
  T gb[GATE_MAXC], yb[GATE_MAXC], db[GATE_MAXC];
  T* io = g.G + e;
  for (int c = 0; c < C; ++c) {
    gb[c] = io[(long long)c * g.plane];
    yb[c] = T(0);
    db[c] = T(0);
    u[c] -= v[c];  // u now holds d = u - v
  }
  yb[0] = gb[0] * u[0];
  db[0] = gb[0] * y[0];
  for (int d = 0; d < g.J.n_dir; ++d) {
    const int K = g.J.dir_order[d];
    const int b = g.J.dir_base[d] - 1;
    for (int k = 1; k <= K; ++k) {
      const T gk = gb[b + k];
      yb[0] += gk * u[b + k];
      db[b + k] += gk * y[0];
      yb[b + k] += gk * u[0];
      db[0] += gk * y[b + k];
      for (int j = 1; j < k; ++j) {
        yb[b + j] += gk * u[b + k - j];
        db[b + k - j] += gk * y[b + j];
      }
    }
  }
  // g = v + y d:  vbar = gbar - dbar, ubar = dbar
  for (int c = 0; c < C; ++c) gb[c] -= db[c];
  gate_act_adj<T, KMAX>(g.J, sy, zy, yb, io, g.plane, false);
  gate_act_adj<T, KMAX>(g.J, su, zu, db, g.Zub + e, g.plane, !g.first);
  gate_act_adj<T, KMAX>(g.J, sv, zv, gb, g.Zvb + e, g.plane, !g.first);
}

// ---- PirateNet: adaptive residual of a block (mlp.py:617-624)  x <- alpha act(z3) + (1 - alpha) x ---------------------
// alpha == nullptr: plain activation, X = act(Z) (the Fourier embedding's output as a stored operand).
template <typename T>
struct MixArgs {
  JetLayout J;
  int act;
  const T* Z;      // [C][Np][ld] pre-activations (third layer of the block, or layer 1)
  const T* Xprev;  // block input jets (may be null: no residual path)
  const T* alpha;  // device scalar of the plan's dtype (may be null: alpha = 1)
  T* X;            // fwd: out.  bwd: Xbar in -> Zbar out (in place)
  T* Xres;         // bwd: adjoint carried by the residual path (read if use_res, written if write_res)
  T* alpha_grad;   // bwd: dLoss/dalpha (atomicAdd of one partial sum per CTA)
  int ld;
  long long plane;
  long long Np;
  int H;
  int use_res;
  int write_res;
};

template <typename T, int KMAX>
__global__ void __launch_bounds__(128) k_mix_fwd(MixArgs<T> g) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= g.Np * g.H) return;
  const long long p = idx / g.H;
  const int h = (int)(idx % g.H);
  const long long e = p * g.ld + h;
  T zj[GATE_MAXC], y[GATE_MAXC], s[6];
  gate_act_jet<T, KMAX>(g.act, g.J, g.Z + e, g.plane, zj, y, s);
  const T a = g.alpha ? g.alpha[0] : T(1);
  for (int c = 0; c < g.J.C; ++c) {
    T v = a * y[c];
    if (g.Xprev) v += (T(1) - a) * g.Xprev[e + (long long)c * g.plane];
    g.X[e + (long long)c * g.plane] = v;
  }
}

template <typename T, int KMAX>
__global__ void __launch_bounds__(128) k_mix_bwd(MixArgs<T> g) {
  __shared__ double red[128];
  const long long total = g.Np * g.H;
  const T a = g.alpha ? g.alpha[0] : T(1);
  double part = 0.0;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long p = idx / g.H;
    const int h = (int)(idx % g.H);
    const long long e = p * g.ld + h;
    T zj[GATE_MAXC], y[GATE_MAXC], xb[GATE_MAXC], s[6];
    gate_act_jet<T, KMAX>(g.act, g.J, g.Z + e, g.plane, zj, y, s);
    for (int c = 0; c < g.J.C; ++c) {
      T v = g.X[e + (long long)c * g.plane];
      if (g.use_res) v += g.Xres[e + (long long)c * g.plane];
      if (g.alpha_grad) part += (double)(v * (y[c] - (g.Xprev ? g.Xprev[e + (long long)c * g.plane] : T(0))));
      if (g.write_res) g.Xres[e + (long long)c * g.plane] = (T(1) - a) * v;
      xb[c] = a * v;
    }
    gate_act_adj<T, KMAX>(g.J, s, zj, xb, g.X + e, g.plane, false);
  }
  if (g.alpha_grad) {  // uniform across the grid
    red[threadIdx.x] = part;
    __syncthreads();
    for (int st = 64; st > 0; st >>= 1) {
      if ((int)threadIdx.x < st) red[threadIdx.x] += red[threadIdx.x + st];
      __syncthreads();
    }
    if (threadIdx.x == 0) atomicAdd(g.alpha_grad, (T)red[0]);
  }
}

}  // namespace ppsci
