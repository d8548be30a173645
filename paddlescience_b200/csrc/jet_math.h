// jet_math.h — per-element Taylor-mode (forward) jet propagation through an activation and
// its adjoint.  Host+device so the same arithmetic can be unit-tested on the CPU.
//
// What this replaces in the reference: the tanh / tanh_grad / tanh_double_grad (…) kernels
// that PaddlePaddle's autograd launches for every reverse sweep issued by
// ppsci/autodiff/ad.py:73-75,141-146 and by total_loss.backward() (ppsci/solver/train.py:158).
//
// Notation.  For one hidden unit and one direction v the pre-activation has the univariate
// Taylor expansion  z(t) = z0 + z1 t + z2 t^2 + z3 t^3 + z4 t^4  (NORMALISED coefficients,
// z_k = (1/k!) d^k z/dt^k).  With s_k = sigma^(k)(z0)/k!  the post-activation coefficients are
//   y1 = s1 z1
//   y2 = s1 z2 + s2 z1^2
//   y3 = s1 z3 + 2 s2 z1 z2 + s3 z1^3
//   y4 = s1 z4 + s2 (2 z1 z3 + z2^2) + 3 s3 z1^2 z2 + s4 z1^4
// (Faa di Bruno for univariate Taylor series).  The adjoint uses d s_k / d z0 = (k+1) s_{k+1}.
#pragma once

#include <math.h>

#if defined(__CUDACC__)
#define PPSCI_HD __host__ __device__ __forceinline__
#else
#define PPSCI_HD inline
#endif

namespace ppsci {

enum ActId {
  ACT_TANH = 0,
  ACT_SIN = 1,
  ACT_COS = 2,
  ACT_SIGMOID = 3,
  ACT_SILU = 4,
  ACT_IDENTITY = 5,
  ACT_RELU = 6,
  ACT_GELU = 7,
  ACT_ELU = 8,
  ACT_SELU = 9,
  ACT_LEAKY_RELU = 10,
  ACT_SIREN = 11,
  // activations with ONE trainable parameter per layer (scalar) or per unit (vector), handed in beside z0:
  ACT_STAN = 12,     // Stan (activation.py:28-46): tanh(z) (1 + beta z), beta per unit, 1 at start
  ACT_SWISH_B = 13,  // Swish (activation.py:49-58): z sigmoid(beta z), beta per layer, 1 at start
};
inline bool act_has_param(int act) { return act == ACT_STAN || act == ACT_SWISH_B; }

template <typename T>
PPSCI_HD T m_tanh(T x);
template <>
PPSCI_HD float m_tanh<float>(float x) { return tanhf(x); }
template <>
PPSCI_HD double m_tanh<double>(double x) { return tanh(x); }
template <typename T>
PPSCI_HD T m_exp(T x);
template <>
PPSCI_HD float m_exp<float>(float x) { return expf(x); }
template <>
PPSCI_HD double m_exp<double>(double x) { return exp(x); }
template <typename T>
PPSCI_HD void m_sincos(T x, T* s, T* c);
template <>
PPSCI_HD void m_sincos<float>(float x, float* s, float* c) {
  *s = sinf(x);
  *c = cosf(x);
}
template <>
PPSCI_HD void m_sincos<double>(double x, double* s, double* c) {
  *s = sin(x);
  *c = cos(x);
}
template <typename T>
PPSCI_HD T m_erf(T x);
template <>
PPSCI_HD float m_erf<float>(float x) { return erff(x); }
template <>
PPSCI_HD double m_erf<double>(double x) { return erf(x); }

// y0 = sigma(z0);  s[k] = sigma^(k)(z0)/k!  for k = 1..NS  (s[0] unused, entries > NS untouched).
template <typename T, int NS>
PPSCI_HD void act_coef(int act, T z0, T& y0, T (&s)[6]) {
  static_assert(NS >= 1 && NS <= 5, "NS in 1..5");
  T d[6];  // raw derivatives d[1..5]
  d[0] = T(0);
  switch (act) {
    case ACT_TANH: {
      const T t = m_tanh<T>(z0);
      const T u = T(1) - t * t;
      const T t2 = t * t;
      y0 = t;
      // normalised coefficients directly (derivation in DESIGN.md)
      s[1] = u;
      if (NS >= 2) s[2] = -t * u;
      if (NS >= 3) s[3] = u * (t2 - T(1) / T(3));
      if (NS >= 4) s[4] = t * u * (T(2) - T(3) * t2) / T(3);
      if (NS >= 5) s[5] = u * (T(2) / T(15) - t2 + t2 * t2);
      return;
    }
    case ACT_SIN: {
      T sn, cs;
      m_sincos<T>(z0, &sn, &cs);
      y0 = sn;
      d[1] = cs; d[2] = -sn; d[3] = -cs; d[4] = sn; d[5] = cs;
      break;
    }
    case ACT_COS: {
      T sn, cs;
      m_sincos<T>(z0, &sn, &cs);
      y0 = cs;
      d[1] = -sn; d[2] = -cs; d[3] = sn; d[4] = cs; d[5] = -sn;
      break;
    }
    case ACT_SIGMOID:
    case ACT_SILU: {
      const T g = T(1) / (T(1) + m_exp<T>(-z0));
      const T g1 = g * (T(1) - g);
      const T g2 = g1 * (T(1) - T(2) * g);
      const T g3 = g1 * (T(1) + g * (T(-6) + T(6) * g));
      const T g4 = g1 * (T(1) - T(2) * g) * (T(1) + g * (T(-12) + T(12) * g));
      const T g5 = g1 * (T(1) + g * (T(-30) + g * (T(150) + g * (T(-240) + T(120) * g))));
      if (act == ACT_SIGMOID) {
        y0 = g;
        d[1] = g1; d[2] = g2; d[3] = g3; d[4] = g4; d[5] = g5;
      } else {  // f = z g  ->  f^(k) = z g^(k) + k g^(k-1)
        y0 = z0 * g;
        d[1] = z0 * g1 + g;
        d[2] = z0 * g2 + T(2) * g1;
        d[3] = z0 * g3 + T(3) * g2;
        d[4] = z0 * g4 + T(4) * g3;
        d[5] = z0 * g5 + T(5) * g4;
      }
      break;
    }
    case ACT_RELU: {
      y0 = z0 > T(0) ? z0 : T(0);
      d[1] = z0 > T(0) ? T(1) : T(0);
      d[2] = d[3] = d[4] = d[5] = T(0);
      break;
    }
    case ACT_GELU: {  // z * Phi(z), erf form
      const T phi = m_exp<T>(T(-0.5) * z0 * z0) * T(0.3989422804014326779);
      const T Phi = T(0.5) * (T(1) + m_erf<T>(z0 * T(0.7071067811865475244)));
      const T z2 = z0 * z0;
      y0 = z0 * Phi;
      d[1] = Phi + z0 * phi;
      d[2] = phi * (T(2) - z2);
      d[3] = phi * z0 * (z2 - T(4));
      d[4] = phi * (T(-4) + z2 * (T(7) - z2));
      d[5] = phi * z0 * (T(18) + z2 * (T(-11) + z2));
      break;
    }
    case ACT_SIREN: {  // sin(w0 z), w0 = 30: d^k/dz^k = w0^k sin^(k)(w0 z)
      const T w0 = T(30);
      T sn, cs;
      m_sincos<T>(w0 * z0, &sn, &cs);
      y0 = sn;
      const T w2 = w0 * w0;
      d[1] = w0 * cs; d[2] = -w2 * sn; d[3] = -w2 * w0 * cs; d[4] = w2 * w2 * sn; d[5] = w2 * w2 * w0 * cs;
      break;
    }
    case ACT_ELU:
    case ACT_SELU: {  // scale * (x > 0 ? x : alpha (e^x - 1)): every derivative of the negative branch is scale alpha e^x
      const T scale = act == ACT_SELU ? T(1.0507009873554804934193349852946) : T(1);
      const T alpha = act == ACT_SELU ? T(1.6732632423543772848170429916717) : T(1);
      if (z0 > T(0)) {
        y0 = scale * z0;
        d[1] = scale;
        d[2] = d[3] = d[4] = d[5] = T(0);
      } else {
        const T e = scale * alpha * m_exp<T>(z0);
        y0 = e - scale * alpha;
        d[1] = d[2] = d[3] = d[4] = d[5] = e;
      }
      break;
    }
    case ACT_LEAKY_RELU: {
      const T sl = z0 > T(0) ? T(1) : T(0.01);
      y0 = sl * z0;
      d[1] = sl;
      d[2] = d[3] = d[4] = d[5] = T(0);
      break;
    }
    case ACT_IDENTITY:
    default: {
      y0 = z0;
      d[1] = T(1);
      d[2] = d[3] = d[4] = d[5] = T(0);
      break;
    }
  }
  const T inv_fact[6] = {T(1), T(1), T(0.5), T(1) / T(6), T(1) / T(24), T(1) / T(120)};
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int k = 1; k <= NS; ++k) s[k] = d[k] * inv_fact[k];
}

// Activations with a trainable parameter beta: same contract as act_coef (y0, s[1..NS] normalised), NS <= 5.
//   Stan     y = tanh(z) (1 + beta z):   s_k = t_k (1 + beta z0) + beta t_{k-1}
//   Swish    y = z f(z), f = sigmoid(beta z), f_k = beta^k sig_k(beta z0):   s_k = z0 f_k + f_{k-1}
template <typename T, int NS>
PPSCI_HD void act_coef_p(int act, T z0, T beta, T& y0, T (&s)[6]) {
  if (act == ACT_STAN) {
    T t[6], t0;
    act_coef<T, NS>(ACT_TANH, z0, t0, t);
    t[0] = t0;
    const T a = T(1) + beta * z0;
    y0 = t0 * a;
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int k = 1; k <= NS; ++k) s[k] = t[k] * a + beta * t[k - 1];
    return;
  }
  if (act == ACT_SWISH_B) {
    T g[6], g0;
    act_coef<T, NS>(ACT_SIGMOID, beta * z0, g0, g);
    g[0] = g0;
    T bp = T(1);
    y0 = z0 * g0;
    T fprev = g0;
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int k = 1; k <= NS; ++k) {
      bp *= beta;
      const T fk = bp * g[k];
      s[k] = z0 * fk + fprev;
      fprev = fk;
    }
    return;
  }
  act_coef<T, NS>(act, z0, y0, s);
}

// q[0..KMAX]: normalised Taylor coefficients (in z, at z0) of  d y / d beta  for the two activations above
//   Stan     z tanh(z):                 q_k = z0 t_k + t_{k-1}
//   Swish    z^2 sigmoid'(beta z):      r_k = beta^k (k+1) sig_{k+1}(beta z0),  q_k = z0^2 r_k + 2 z0 r_{k-1} + r_{k-2}
// The jets of dy/dbeta along a direction are jet_fwd_dir(q, z) (order >= 1) and q[0] (value).  KMAX <= 4.
template <typename T, int KMAX>
PPSCI_HD void act_dbeta_coef(int act, T z0, T beta, T (&q)[6]) {
  if (act == ACT_STAN) {
    T t[6], t0;
    act_coef<T, KMAX>(ACT_TANH, z0, t0, t);
    t[0] = t0;
    q[0] = z0 * t0;
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int k = 1; k <= KMAX; ++k) q[k] = z0 * t[k] + t[k - 1];
    return;
  }
  T g[6], g0;
  act_coef<T, KMAX + 1>(ACT_SIGMOID, beta * z0, g0, g);
  T r[6];
  T bp = T(1);
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int k = 0; k <= KMAX; ++k) {
    r[k] = bp * T(k + 1) * g[k + 1];
    bp *= beta;
  }
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int k = 0; k <= KMAX; ++k) {
    T v = z0 * z0 * r[k];
    if (k >= 1) v += T(2) * z0 * r[k - 1];
    if (k >= 2) v += r[k - 2];
    q[k] = v;
  }
}

// Forward for one direction: z[k-1], y[k-1] hold order k (k = 1..KMAX); entries of z past
// the direction's own order must be zero.  Uses s[1..KMAX].
template <typename T, int KMAX>
PPSCI_HD void jet_fwd_dir(const T (&s)[6], const T (&z)[4], T (&y)[4]) {
  const T z1 = z[0];
  y[0] = s[1] * z1;
  if (KMAX >= 2) y[1] = s[1] * z[1] + s[2] * z1 * z1;
  if (KMAX >= 3) y[2] = s[1] * z[2] + T(2) * s[2] * z1 * z[1] + s[3] * z1 * z1 * z1;
  if (KMAX >= 4)
    y[3] = s[1] * z[3] + s[2] * (T(2) * z1 * z[2] + z[1] * z[1]) + T(3) * s[3] * z1 * z1 * z[1] +
           s[4] * z1 * z1 * z1 * z1;
}

// Adjoint of jet_fwd_dir for one direction.
//   in : s[1..KMAX], z, yb (adjoint of y; zero past the direction's order)
//   out: zb (adjoint of z for this direction), sb[k] += adjoint of s_k   (k = 1..KMAX)
template <typename T, int KMAX>
PPSCI_HD void jet_adj_dir(const T (&s)[6], const T (&z)[4], const T (&yb)[4], T (&zb)[4],
                          T (&sb)[5]) {
  const T z1 = z[0];
  const T y1b = yb[0];
  if (KMAX == 1) {
    zb[0] = s[1] * y1b;
    sb[1] += z1 * y1b;
    return;
  }
  const T z2 = z[1], y2b = yb[1];
  if (KMAX == 2) {
    zb[1] = s[1] * y2b;
    zb[0] = s[1] * y1b + T(2) * s[2] * z1 * y2b;
    sb[1] += z1 * y1b + z2 * y2b;
    sb[2] += z1 * z1 * y2b;
    return;
  }
  const T z3 = z[2], y3b = yb[2];
  const T z4 = KMAX >= 4 ? z[3] : T(0);
  const T y4b = KMAX >= 4 ? yb[3] : T(0);
  const T s4 = KMAX >= 4 ? s[4] : T(0);
  const T a = T(2) * s[2] * z2 + T(3) * s[3] * z1 * z1;  // d y3/d z1 = d y4/d z2
  if (KMAX >= 4) zb[3] = s[1] * y4b;
  zb[2] = s[1] * y3b + T(2) * s[2] * z1 * y4b;
  zb[1] = s[1] * y2b + T(2) * s[2] * z1 * y3b + a * y4b;
  zb[0] = s[1] * y1b + T(2) * s[2] * z1 * y2b + a * y3b +
          (T(2) * s[2] * z3 + T(6) * s[3] * z1 * z2 + T(4) * s4 * z1 * z1 * z1) * y4b;
  sb[1] += z1 * y1b + z2 * y2b + z3 * y3b + z4 * y4b;
  sb[2] += z1 * z1 * y2b + T(2) * z1 * z2 * y3b + (T(2) * z1 * z3 + z2 * z2) * y4b;
  sb[3] += z1 * z1 * z1 * y3b + T(3) * z1 * z1 * z2 * y4b;
  if (KMAX >= 4) sb[4] += z1 * z1 * z1 * z1 * y4b;
}

// zb0 = s1 * y0b + sum_k (k+1) s_{k+1} sb_k      (uses s[1..KMAX+1])
template <typename T, int KMAX>
PPSCI_HD T jet_adj_z0(const T (&s)[6], T y0b, const T (&sb)[5]) {
  T r = s[1] * y0b;
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int k = 1; k <= KMAX; ++k) r += T(k + 1) * s[k + 1] * sb[k];
  return r;
}

// Taylor coefficients (normalised) of g(omega*(x + t*v)) for g in {identity, cos, sin}.
// out[0] = value, out[k] = order-k coefficient, k = 1..KMAX.
template <typename T, int KMAX>
PPSCI_HD void seed_coef(int kind, T omega, T x, T v, T (&out)[5]) {
  if (kind == 0) {
    out[0] = x;
    out[1] = v;
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int k = 2; k <= KMAX; ++k) out[k] = T(0);
    return;
  }
  T sn, cs;
  m_sincos<T>(omega * x, &sn, &cs);
  T g[5];  // derivative cycle of g at theta = omega*x
  if (kind == 1) { g[0] = cs; g[1] = -sn; g[2] = -cs; g[3] = sn; g[4] = cs; }
  else           { g[0] = sn; g[1] = cs; g[2] = -sn; g[3] = -cs; g[4] = sn; }
  const T h = omega * v;
  const T inv_fact[5] = {T(1), T(1), T(0.5), T(1) / T(6), T(1) / T(24)};
  T hp = T(1);
  out[0] = g[0];
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int k = 1; k <= KMAX; ++k) {
    hp *= h;
    out[k] = g[k] * hp * inv_fact[k];
  }
}

// d/d omega of seed_coef's coefficients (a trainable PeriodEmbedding frequency; kind 1 / 2, identity features have none).
// With G_k the k-th derivative of g at omega*x, the order-k coefficient G_k (omega v)^k / k! has the omega-derivative
//   G_{k+1} x (omega v)^k / k!  +  G_k k omega^{k-1} v^k / k!        (value channel, k = 0:  G_1 x)
template <typename T, int KMAX>
PPSCI_HD void seed_dcoef(int kind, T omega, T x, T v, T (&out)[5]) {
  if (kind == 0) {
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int k = 0; k <= KMAX; ++k) out[k] = T(0);
    return;
  }
  T sn, cs;
  m_sincos<T>(omega * x, &sn, &cs);
  T g[6];
  if (kind == 1) { g[0] = cs; g[1] = -sn; g[2] = -cs; g[3] = sn; g[4] = cs; g[5] = -sn; }
  else           { g[0] = sn; g[1] = cs; g[2] = -sn; g[3] = -cs; g[4] = sn; g[5] = cs; }
  const T h = omega * v;
  const T inv_fact[5] = {T(1), T(1), T(0.5), T(1) / T(6), T(1) / T(24)};
  T hp = T(1);  // h^(k-1)
  out[0] = g[1] * x;
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int k = 1; k <= KMAX; ++k) {
    out[k] = (g[k + 1] * x * hp * h + g[k] * T(k) * hp * v) * inv_fact[k];
    hp *= h;
  }
}

}  // namespace ppsci
