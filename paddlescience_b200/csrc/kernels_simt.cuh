// kernels_simt.cuh — generic (any width / activation / order<=4 / f32|f64) CUDA-core kernels
// of the jet engine: every hidden layer runs on them, and they are the correctness anchor for the
// vectorised fp32 thin-layer kernels (kernels_thin.cuh).
//
// Data layout (all in the caller's workspace; see DESIGN.md "HBM layout"):
//   jets of a layer are CHANNEL-MAJOR planes   Z[c][p][h] ,  c < C, p < Np, h < ld
//   channel 0 = value, channel (d,k) = k-th normalised Taylor coefficient along direction d.
// Row r of a tile = c*TP + pl  (TP points per tile, pl = point within tile).
//
// Reference functions replaced here:
//   k_gemm_fwd   : nn.Linear + activation per layer, evaluated for all jet channels at once
//                  (ppsci/arch/mlp.py:281-296) — no reverse sweeps (ppsci/autodiff/ad.py).
//   k_gemm_dx    : the "dX" half of total_loss.backward() (ppsci/solver/train.py:158)
//   k_gemm_dw    : the "dW/db" half of the same.
//   k_head       : ComposedNode.forward residual assembly (ppsci/utils/symbolic.py:498-504),
//                  MSELoss.forward (ppsci/loss/mse.py:82-106), mtl.Sum (loss/mtl/sum.py:45-60)
#pragma once

#include "jet_math.h"
#include "ppsci_b200.h"

#ifndef PPSCI_EMUL
#include <cuda_runtime.h>
#define PPSCI_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#define PPSCI_LAUNCH(kernel, grid, block, smem, stream, ...) \
  kernel<<<(grid), (block), (smem), (cudaStream_t)(stream)>>>(__VA_ARGS__)
#endif

namespace ppsci {

constexpr int TM = 128;      // tile rows (points x channels)
constexpr int TMS = TM + 4;  // padded smem row stride of the k-major A tile
constexpr int KC = 16;       // reduction chunk of the fwd / dx GEMMs
constexpr int RC = 32;       // reduction (row) chunk of the dW GEMM
constexpr int NTHREADS = 256;

struct JetLayout {
  int C;
  int n_dir;
  int dir_order[PPSCI_MAX_DIR];
  int dir_base[PPSCI_MAX_DIR];  // channel index of order-1 coefficient of direction d
};

struct SeedSpec {
  int n_in;
  int n_feat;
  int feat_src[PPSCI_MAX_FEAT];
  int feat_kind[PPSCI_MAX_FEAT];
  double feat_omega[PPSCI_MAX_FEAT];
  double dir_vec[PPSCI_MAX_DIR][PPSCI_MAX_IN];
  const void* x_cols[PPSCI_MAX_IN];
};

enum { A_SEED = 0, A_ACT = 1, A_PLAIN = 2 };

template <typename T>
struct AOperand {
  int mode;
  int act;
  const T* Z;  // [C][Np][ld]  (A_ACT: pre-activations of the previous layer, A_PLAIN: as is)
  int ld;
  long long plane;  // Np * ld
  SeedSpec seed;  // by value (kernel parameter space), used by A_SEED
  long long x_off;       // first point of this chunk inside the x columns
  // A_ACT with a trainable activation parameter (ACT_STAN: one beta per unit, stride 1; ACT_SWISH_B: one per layer, stride 0)
  const T* act_param;
  int act_pstride;
};

// Produce all C channel values of A[(c, p), k] and hand them to st(c, value).
template <typename T, int KMAX, typename St>
__device__ __forceinline__ void produce_a(const AOperand<T>& A, const JetLayout& J, long long p,
                                          int k, bool valid, St st) {
  if (!valid) {
    for (int c = 0; c < J.C; ++c) st(c, T(0));
    return;
  }
  if (A.mode == A_PLAIN) {
    const T* z = A.Z + p * A.ld + k;
    for (int c = 0; c < J.C; ++c) st(c, z[c * A.plane]);
    return;
  }
  if (A.mode == A_ACT) {
    const T* z = A.Z + p * A.ld + k;
    T s[6];
    T y0;
    if (A.act_param) act_coef_p<T, KMAX>(A.act, z[0], A.act_param[(long long)k * A.act_pstride], y0, s);
    else act_coef<T, KMAX>(A.act, z[0], y0, s);
    st(0, y0);
    for (int d = 0; d < J.n_dir; ++d) {
      const int K = J.dir_order[d];
      const int base = J.dir_base[d];
      T zz[4], yy[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) zz[q] = (q < KMAX && q < K) ? z[(long long)(base + q) * A.plane] : T(0);
      jet_fwd_dir<T, KMAX>(s, zz, yy);
#pragma unroll
      for (int q = 0; q < KMAX; ++q)
        if (q < K) st(base + q, yy[q]);
    }
    return;
  }
  // A_SEED: feature k of the (period-embedded) network input, Taylor-expanded along each direction
  const SeedSpec& S = A.seed;
  const int src = S.feat_src[k];
  const int kind = S.feat_kind[k];
  const T omega = T(S.feat_omega[k]);
  const T x = reinterpret_cast<const T*>(S.x_cols[src])[A.x_off + p];
  T co[5];
  seed_coef<T, KMAX>(kind, omega, x, T(0), co);
  st(0, co[0]);
  for (int d = 0; d < J.n_dir; ++d) {
    const int K = J.dir_order[d];
    const int base = J.dir_base[d];
    seed_coef<T, KMAX>(kind, omega, x, T(S.dir_vec[d][src]), co);
#pragma unroll
    for (int q = 0; q < KMAX; ++q)
      if (q < K) st(base + q, co[q + 1]);
  }
}

// Same arithmetic as produce_a's A_PLAIN / A_ACT branches, but the C channel values of the element
// come from a caller-supplied loader ld(c) (e.g. a shared-memory staging tile).
template <typename T, int KMAX, typename Ld, typename St>
__device__ __forceinline__ void produce_from(int mode, int act, const JetLayout& J, bool valid, Ld ld, St st) {
  if (!valid) {
    for (int c = 0; c < J.C; ++c) st(c, T(0));
    return;
  }
  if (mode == A_PLAIN) {
    for (int c = 0; c < J.C; ++c) st(c, ld(c));
    return;
  }
  T s[6];
  T y0;
  act_coef<T, KMAX>(act, ld(0), y0, s);
  st(0, y0);
  for (int d = 0; d < J.n_dir; ++d) {
    const int K = J.dir_order[d];
    const int base = J.dir_base[d];
    T zz[4], yy[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) zz[q] = (q < KMAX && q < K) ? ld(base + q) : T(0);
    jet_fwd_dir<T, KMAX>(s, zz, yy);
#pragma unroll
    for (int q = 0; q < KMAX; ++q)
      if (q < K) st(base + q, yy[q]);
  }
}

template <typename T>
__device__ __forceinline__ void ld4(const T* p, T* out);
template <>
__device__ __forceinline__ void ld4<float>(const float* p, float* out) {
  const float4 v = *reinterpret_cast<const float4*>(p);
  out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w;
}
template <>
__device__ __forceinline__ void ld4<double>(const double* p, double* out) {
  const double2 v0 = *reinterpret_cast<const double2*>(p);
  const double2 v1 = *reinterpret_cast<const double2*>(p + 2);
  out[0] = v0.x; out[1] = v0.y; out[2] = v1.x; out[3] = v1.y;
}

template <typename T>
struct GemmArgs {
  AOperand<T> A;
  JetLayout J;
  const T* B;  // row-major [Kdim][ldb]
  int Kdim;
  int Nout;
  int ldb;
  const T* bias;  // fwd: added to channel-0 rows (may be null)
  T* Out;         // fwd: Z_l [C][Np][ldo];  dx: Zbar_{l-1} [C][Np][ldo]
  int ldo;
  long long oplane;
  long long Np;  // valid points in this chunk
  int TP;        // points per tile = TM / C
  // dx epilogue: pre-activations of the layer whose activation is being back-propagated
  const T* Zprev;
  int ldz;
  long long zplane;
  int act;
  int accum;  // dx: add to Out instead of storing (a second consumer of the same operand)
  // dx epilogue of an activation with a trainable parameter: beta (stride 1 per unit / 0 per layer) and where
  // dLoss/dbeta accumulates (same stride)
  const T* act_param;
  T* act_param_grad;
  int act_pstride;
};

template <int TN>
struct MicroShape {
  static constexpr int NJ = TN / 16;  // columns per thread
  static constexpr int NG = TN / 64;  // groups of 4 columns
};

// acc[8][NJ] += A_tile[128 x K] * B[K x TN] ; A produced on the fly (k-major smem tile).
template <typename T, int TN, int KMAX>
__device__ __forceinline__ void gemm_mainloop(const GemmArgs<T>& g, T* As, T* Bs,
                                              T (&acc)[8][TN / 16], long long p0, int n0) {
  constexpr int NJ = TN / 16;
  constexpr int NG = TN / 64;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int TP = g.TP;
  const int rows_used = g.J.C * TP;
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[i][j] = T(0);
  for (int idx = tid; idx < KC * TMS; idx += NTHREADS) {
    const int r = idx % TMS;
    if (r >= rows_used) As[idx] = T(0);
  }
  for (int k0 = 0; k0 < g.Kdim; k0 += KC) {
    for (int item = tid; item < TP * KC; item += NTHREADS) {
      const int kk = item % KC, pl = item / KC;
      const long long p = p0 + pl;
      const int k = k0 + kk;
      T* dst = As + kk * TMS + pl;
      produce_a<T, KMAX>(g.A, g.J, p, k, (p < g.Np) && (k < g.Kdim),
                         [&](int c, T v) { dst[c * TP] = v; });
    }
    for (int idx = tid; idx < KC * TN; idx += NTHREADS) {
      const int kk = idx / TN, nn = idx % TN;
      const int k = k0 + kk, n = n0 + nn;
      Bs[idx] = (k < g.Kdim && n < g.Nout) ? g.B[(long long)k * g.ldb + n] : T(0);
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < KC; ++kk) {
      T a[8], b[NJ];
      ld4<T>(As + kk * TMS + ty * 4, a);
      ld4<T>(As + kk * TMS + 64 + ty * 4, a + 4);
#pragma unroll
      for (int gq = 0; gq < NG; ++gq) ld4<T>(Bs + kk * TN + gq * 64 + tx * 4, b + gq * 4);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc[i][j] += a[i] * b[j];
    }
    __syncthreads();
  }
}

__device__ __forceinline__ int micro_row(int ty, int i) { return (i < 4) ? ty * 4 + i : 64 + ty * 4 + (i - 4); }
__device__ __forceinline__ int micro_col(int tx, int j) { return (j >> 2) * 64 + tx * 4 + (j & 3); }

// ---- forward layer:  Z_l = A(Z_{l-1}) W_l + b_l ------------------------------------------------
template <typename T, int TN, int KMAX>
__global__ void __launch_bounds__(NTHREADS) k_gemm_fwd(GemmArgs<T> g) {
  PPSCI_DYN_SMEM(smem_raw);
  T* As = reinterpret_cast<T*>(smem_raw);
  T* Bs = As + KC * TMS;
  constexpr int NJ = TN / 16;
  const long long p0 = (long long)blockIdx.x * g.TP;
  const int n0 = blockIdx.y * TN;
  T acc[8][NJ];
  gemm_mainloop<T, TN, KMAX>(g, As, Bs, acc, p0, n0);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int rows_used = g.J.C * g.TP;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = micro_row(ty, i);
    if (r >= rows_used) continue;
    const int c = r / g.TP, pl = r % g.TP;
    const long long p = p0 + pl;
    if (p >= g.Np) continue;
    T* out = g.Out + (long long)c * g.oplane + p * g.ldo;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int n = n0 + micro_col(tx, j);
      if (n < g.Nout) out[n] = acc[i][j] + ((c == 0 && g.bias) ? g.bias[n] : T(0));
    }
  }
}

// ---- backward dx:  Abar = Zbar_l W_l^T ;  Zbar_{l-1} = act_adjoint(Abar, Z_{l-1}) -----------------
template <typename T, int TN, int KMAX>
__global__ void __launch_bounds__(NTHREADS) k_gemm_dx(GemmArgs<T> g) {
  PPSCI_DYN_SMEM(smem_raw);
  T* As = reinterpret_cast<T*>(smem_raw);
  T* Bs = As + KC * TMS;
  T* Cs = reinterpret_cast<T*>(smem_raw);  // aliases As/Bs after the main loop
  constexpr int NJ = TN / 16;
  const long long p0 = (long long)blockIdx.x * g.TP;
  const int n0 = blockIdx.y * TN;
  T acc[8][NJ];
  gemm_mainloop<T, TN, KMAX>(g, As, Bs, acc, p0, n0);  // ends with __syncthreads()
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = micro_row(ty, i);
#pragma unroll
    for (int j = 0; j < NJ; ++j) Cs[r * TN + micro_col(tx, j)] = acc[i][j];
  }
  __syncthreads();
  const int TP = g.TP;
  static_assert(NTHREADS % TN == 0, "a thread keeps one output column across its items (dLoss/dbeta partial sums)");
  T bsum = T(0);  // this thread's share of dLoss/dbeta of column n0 + threadIdx.x % TN
  for (int item = threadIdx.x; item < TP * TN; item += NTHREADS) {
    const int nn = item % TN, pl = item / TN;
    const long long p = p0 + pl;
    const int n = n0 + nn;
    if (p >= g.Np || n >= g.Nout) continue;
    const T* z = g.Zprev + p * g.ldz + n;
    T* zb_out = g.Out + p * g.ldo + n;
    T s[6];
    T y0;
    T qb[6];
    T bacc = T(0);
    const T beta = g.act_param ? g.act_param[(long long)n * g.act_pstride] : T(0);
    if (g.act_param) {
      act_coef_p<T, KMAX + 1>(g.act, z[0], beta, y0, s);
      act_dbeta_coef<T, KMAX>(g.act, z[0], beta, qb);
    } else {
      act_coef<T, KMAX + 1>(g.act, z[0], y0, s);
    }
    const T y0b = Cs[pl * TN + nn];
    if (g.act_param) bacc = y0b * qb[0];
    T sb[5] = {T(0), T(0), T(0), T(0), T(0)};
    for (int d = 0; d < g.J.n_dir; ++d) {
      const int K = g.J.dir_order[d];
      const int base = g.J.dir_base[d];
      T zz[4], yb[4], zb[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const bool on = (q < KMAX && q < K);
        zz[q] = on ? z[(long long)(base + q) * g.zplane] : T(0);
        yb[q] = on ? Cs[((base + q) * TP + pl) * TN + nn] : T(0);
        zb[q] = T(0);
      }
      jet_adj_dir<T, KMAX>(s, zz, yb, zb, sb);
      if (g.act_param) {  // dLoss/dbeta += <adjoint of the activation's output jets, jets of dy/dbeta>
        T wq[4] = {T(0), T(0), T(0), T(0)};
        jet_fwd_dir<T, KMAX>(qb, zz, wq);
#pragma unroll
        for (int qq = 0; qq < KMAX; ++qq) bacc += yb[qq] * wq[qq];
      }
#pragma unroll
      for (int q = 0; q < KMAX; ++q)
        if (q < K) {
          T* o = zb_out + (long long)(base + q) * g.oplane;
          *o = g.accum ? *o + zb[q] : zb[q];
        }
    }
    const T z0b = jet_adj_z0<T, KMAX>(s, y0b, sb);
    zb_out[0] = g.accum ? zb_out[0] + z0b : z0b;
    bsum += bacc;
  }
  if (g.act_param_grad) {
    const int n = n0 + (int)(threadIdx.x % TN);
    if (n < g.Nout && bsum != T(0)) atomicAdd(g.act_param_grad + (long long)n * g.act_pstride, bsum);
  }
}

// ---- backward dW:  dW_l += A(Z_{l-1})^T Zbar_l ,  db_l += colsum(Zbar_l[channel 0]) ---------------
template <typename T>
struct DwArgs {
  AOperand<T> A;
  JetLayout J;
  const T* Zbar;  // [C][Np][ldzb]
  int ldzb;
  long long zbplane;
  int Kdim;  // rows of dW (= fan-in of the layer)
  int Nout;  // cols of dW
  T* dW;     // [Kdim][Nout] (accumulated with atomics)
  T* db;     // [Nout]
  long long Np;
  int PT;  // points per reduction chunk = RC / C
  int chunks_per_split;
};

template <typename T, int TN, int KMAX>
__global__ void __launch_bounds__(NTHREADS) k_gemm_dw(DwArgs<T> g) {
  PPSCI_DYN_SMEM(smem_raw);
  T* As = reinterpret_cast<T*>(smem_raw);  // [RC][TMS]   (reduction-row major, k contiguous)
  T* Bs = As + RC * TMS;                   // [RC][TN]
  constexpr int NJ = TN / 16;
  constexpr int NG = TN / 64;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int k0 = blockIdx.x * TM;
  const int n0 = blockIdx.y * TN;
  const int PT = g.PT;
  const int rows_used = g.J.C * PT;
  const long long total_chunks = (g.Np + PT - 1) / PT;
  const long long ch_begin = (long long)blockIdx.z * g.chunks_per_split;
  long long ch_end = ch_begin + g.chunks_per_split;
  if (ch_end > total_chunks) ch_end = total_chunks;
  T acc[8][NJ];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[i][j] = T(0);
  T dbacc = T(0);
  for (int idx = tid; idx < RC * TMS; idx += NTHREADS) As[idx] = T(0);
  for (int idx = tid; idx < RC * TN; idx += NTHREADS) Bs[idx] = T(0);
  __syncthreads();
  for (long long ch = ch_begin; ch < ch_end; ++ch) {
    const long long p0 = ch * PT;
    for (int item = tid; item < PT * TM; item += NTHREADS) {
      const int kq = item % TM, pl = item / TM;
      const long long p = p0 + pl;
      const int k = k0 + kq;
      T* dst = As + pl * TMS + kq;
      produce_a<T, KMAX>(g.A, g.J, p, k, (p < g.Np) && (k < g.Kdim),
                         [&](int c, T v) { dst[c * PT * TMS] = v; });
    }
    for (int item = tid; item < rows_used * TN; item += NTHREADS) {
      const int nn = item % TN, r = item / TN;
      const int c = r / PT, pl = r % PT;
      const long long p = p0 + pl;
      const int n = n0 + nn;
      Bs[r * TN + nn] = (p < g.Np && n < g.Nout) ? g.Zbar[(long long)c * g.zbplane + p * g.ldzb + n] : T(0);
    }
    __syncthreads();
#pragma unroll 4
    for (int rr = 0; rr < RC; ++rr) {
      T a[8], b[NJ];
      ld4<T>(As + rr * TMS + ty * 4, a);
      ld4<T>(As + rr * TMS + 64 + ty * 4, a + 4);
#pragma unroll
      for (int gq = 0; gq < NG; ++gq) ld4<T>(Bs + rr * TN + gq * 64 + tx * 4, b + gq * 4);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc[i][j] += a[i] * b[j];
    }
    if (blockIdx.x == 0 && tid < TN) {
      for (int pl = 0; pl < PT; ++pl) dbacc += Bs[pl * TN + tid];  // channel-0 rows are rows [0, PT)
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int k = k0 + micro_row(ty, i);
    if (k >= g.Kdim) continue;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int n = n0 + micro_col(tx, j);
      if (n < g.Nout) atomicAdd(g.dW + (long long)k * g.Nout + n, acc[i][j]);
    }
  }
  if (blockIdx.x == 0 && tid < TN && (n0 + tid) < g.Nout && g.db) atomicAdd(g.db + n0 + tid, dbacc);
}

// =====================================================================================================
// Thin layers.  The input layer has K = n_feat (2..8) and the output layer N = n_out (1..8): a 128-wide
// GEMM tile wastes >95 % of its FMAs on them, and they are pure HBM streams (read or write one jet plane
// set).  Dedicated kernels: one pass over the planes, coalesced along the hidden dimension.
// =====================================================================================================
constexpr int THIN_MAXF = 8;    // input features handled by the thin first-layer kernels
constexpr int THIN_MAXM = 8;    // network outputs handled by the thin last-layer kernels
constexpr int THIN_MAXCM = 64;  // C * n_out bound of k_last_fwd

template <typename T>
struct FirstArgs {
  AOperand<T> A;  // A_SEED
  JetLayout J;
  const T* W;     // [nf][N]
  const T* bias;  // [N]
  int nf, N;
  T* Out;         // fwd: Z_1 [C][Np][ldo]
  int ldo;
  long long oplane;
  const T* Zbar;  // dW: Zbar_1 [C][Np][ldzb]
  int ldzb;
  long long zbplane;
  T* dW;          // [nf][N]
  T* db;          // [N]
  long long Np;
  int pts_per_block;
};

// Z_1[c][p][n] = sum_f seed_c[p][f] W[f][n] (+ b[n] on the value channel)
template <typename T, int KMAX>
__global__ void __launch_bounds__(256) k_first_fwd(FirstArgs<T> g) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.Np * g.N) return;
  const long long p = i / g.N;
  const int n = (int)(i % g.N);
  T acc[32];
  for (int c = 0; c < g.J.C; ++c) acc[c] = T(0);
  for (int f = 0; f < g.nf; ++f) {
    const T w = g.W[(long long)f * g.N + n];
    produce_a<T, KMAX>(g.A, g.J, p, f, true, [&](int c, T v) { acc[c] += v * w; });
  }
  T* out = g.Out + p * g.ldo + n;
  for (int c = 0; c < g.J.C; ++c) out[(long long)c * g.oplane] = acc[c] + (c == 0 ? g.bias[n] : T(0));
}

// dW_1[f][n] += sum_{c,p} seed_c[p][f] Zbar_1[c][p][n] ;  db_1[n] += sum_p Zbar_1[0][p][n]
template <typename T, int KMAX>
__global__ void __launch_bounds__(256) k_first_dw(FirstArgs<T> g) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= g.N) return;
  const long long p_begin = (long long)blockIdx.y * g.pts_per_block;
  long long p_end = p_begin + g.pts_per_block;
  if (p_end > g.Np) p_end = g.Np;
  T acc[THIN_MAXF];
#pragma unroll
  for (int f = 0; f < THIN_MAXF; ++f) acc[f] = T(0);
  T dbacc = T(0);
  for (long long p = p_begin; p < p_end; ++p) {
    const T* zb = g.Zbar + p * g.ldzb + n;
    dbacc += zb[0];
#pragma unroll
    for (int f = 0; f < THIN_MAXF; ++f) {
      if (f < g.nf) {
        T a = T(0);
        produce_a<T, KMAX>(g.A, g.J, p, f, true, [&](int c, T v) { a += v * zb[(long long)c * g.zbplane]; });
        acc[f] += a;
      }
    }
  }
#pragma unroll
  for (int f = 0; f < THIN_MAXF; ++f)
    if (f < g.nf) atomicAdd(g.dW + (long long)f * g.N + n, acc[f]);
  atomicAdd(g.db + n, dbacc);
}

template <typename T>
struct LastArgs {
  AOperand<T> A;  // A_ACT over Z_{L-1}  (pre-activations of the last hidden layer)
  JetLayout J;
  const T* W;     // [K][m]
  const T* bias;  // [m]
  int K, m;
  T* Y;           // fwd: output jets [C][Np][ldy]
  const T* Ybar;  // bwd: adjoints of the output jets, same layout
  int ldy;
  long long yplane;
  T* ZbarOut;     // bwd: Zbar_{L-1} [C][Np][ldo]
  int ldo;
  long long oplane;
  T* dW;          // [K][m]
  T* db;          // [m]
  long long Np;
  int pts_per_block;
};

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Y[c][p][j] = sum_k act_jets(Z_{L-1})[c][p][k] W[k][j] (+ b[j] on the value channel); one warp per point
template <typename T, int KMAX>
__global__ void __launch_bounds__(256) k_last_fwd(LastArgs<T> g) {
  const int lane = threadIdx.x & 31;
  const long long p = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (p >= g.Np) return;  // whole warp exits together
  T acc[THIN_MAXCM];
  const int CM = g.J.C * g.m;
  for (int i = 0; i < CM; ++i) acc[i] = T(0);
  for (int k = lane; k < g.K; k += 32) {
    T w[THIN_MAXM];
#pragma unroll
    for (int j = 0; j < THIN_MAXM; ++j) w[j] = j < g.m ? g.W[(long long)k * g.m + j] : T(0);
    produce_a<T, KMAX>(g.A, g.J, p, k, true, [&](int c, T v) {
#pragma unroll
      for (int j = 0; j < THIN_MAXM; ++j)
        if (j < g.m) acc[c * g.m + j] += v * w[j];
    });
  }
  for (int i = 0; i < CM; ++i) {
    const T v = warp_sum<T>(acc[i]);
    if (lane == 0) {
      const int c = i / g.m, j = i % g.m;
      g.Y[(long long)c * g.yplane + p * g.ldy + j] = v + (c == 0 ? g.bias[j] : T(0));
    }
  }
}

// Output layer backward, fused: for every (point, hidden unit k)
//   abar_c = sum_j Ybar[c][p][j] W[k][j];  Zbar_{L-1} = act_adjoint(abar, Z_{L-1});
//   dW[k][j] += sum_{c,p} a_c[p][k] Ybar[c][p][j];  db[j] += sum_p Ybar[0][p][j]
template <typename T, int KMAX>
__global__ void __launch_bounds__(256) k_last_bwd(LastArgs<T> g) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const bool k_ok = k < g.K;
  const long long p_begin = (long long)blockIdx.y * g.pts_per_block;
  long long p_end = p_begin + g.pts_per_block;
  if (p_end > g.Np) p_end = g.Np;
  T w[THIN_MAXM], dwacc[THIN_MAXM], dbacc[THIN_MAXM];
#pragma unroll
  for (int j = 0; j < THIN_MAXM; ++j) {
    w[j] = (k_ok && j < g.m) ? g.W[(long long)k * g.m + j] : T(0);
    dwacc[j] = T(0);
    dbacc[j] = T(0);
  }
  const bool do_db = (blockIdx.x == 0 && threadIdx.x == 0);
  if (k_ok) {
    for (long long p = p_begin; p < p_end; ++p) {
      const T* yb = g.Ybar + p * g.ldy;  // + c*yplane + j   (same address for the whole block: broadcast)
      const T* z = g.A.Z + p * g.A.ld + k;
      T* zb_out = g.ZbarOut + p * g.ldo + k;
      T s[6];
      T y0;
      act_coef<T, KMAX + 1>(g.A.act, z[0], y0, s);
      T y0b = T(0);
#pragma unroll
      for (int j = 0; j < THIN_MAXM; ++j)
        if (j < g.m) {
          const T ybj = yb[j];
          y0b += ybj * w[j];
          dwacc[j] += y0 * ybj;
          if (do_db) dbacc[j] += ybj;
        }
      T sb[5] = {T(0), T(0), T(0), T(0), T(0)};
      for (int d = 0; d < g.J.n_dir; ++d) {
        const int Kd = g.J.dir_order[d];
        const int cb = g.J.dir_base[d];
        T zz[4], yy[4], ybq[4], zbq[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          zz[q] = (q < KMAX && q < Kd) ? z[(long long)(cb + q) * g.A.plane] : T(0);
          ybq[q] = T(0);
          zbq[q] = T(0);
        }
        jet_fwd_dir<T, KMAX>(s, zz, yy);
#pragma unroll
        for (int q = 0; q < KMAX; ++q)
          if (q < Kd) {
            const T* ybc = yb + (long long)(cb + q) * g.yplane;
#pragma unroll
            for (int j = 0; j < THIN_MAXM; ++j)
              if (j < g.m) {
                const T ybj = ybc[j];
                ybq[q] += ybj * w[j];
                dwacc[j] += yy[q] * ybj;
              }
          }
        jet_adj_dir<T, KMAX>(s, zz, ybq, zbq, sb);
#pragma unroll
        for (int q = 0; q < KMAX; ++q)
          if (q < Kd) zb_out[(long long)(cb + q) * g.oplane] = zbq[q];
      }
      zb_out[0] = jet_adj_z0<T, KMAX>(s, y0b, sb);
    }
#pragma unroll
    for (int j = 0; j < THIN_MAXM; ++j)
      if (j < g.m) atomicAdd(g.dW + (long long)k * g.m + j, dwacc[j]);
  }
  if (do_db) {
#pragma unroll
    for (int j = 0; j < THIN_MAXM; ++j)
      if (j < g.m) atomicAdd(g.db + j, dbacc[j]);
  }
}

// Output adjoints supplied by the caller (ppsci_b200_values_fwd_bwd): value channel <- ybar[p][j], other channels 0.
template <typename T>
__global__ void k_seed_ybar(const T* __restrict__ ybar_in, long long x_off, long long Np, int n_out, int C, T* __restrict__ Ybar,
                            int ldy, long long yplane) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Np * ldy) return;
  const long long p = i / ldy;
  const int j = (int)(i - p * ldy);
  Ybar[i] = j < n_out ? ybar_in[(x_off + p) * n_out + j] : T(0);
  for (int c = 1; c < C; ++c) Ybar[(long long)c * yplane + i] = T(0);
}

// ---- small helpers ---------------------------------------------------------------------------
template <typename T>
__global__ void k_transpose(const T* W, T* WT, int K, int N) {  // WT[n][k] = W[k][n]
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)K * N) return;
  const int k = (int)(i / N), n = (int)(i % N);
  WT[(long long)n * K + k] = W[i];
}

// ---- residual program + MSE + output-jet adjoints ---------------------------------------------
struct HeadProgram {  // all pointers are device pointers owned by the plan
  const int* prog;    // n_ops * 4
  const double* consts;
  int n_ops;
  int n_reg;
  int n_res;
  int res_reg[PPSCI_MAX_RES];
  int n_grad;
  const int* grad_res;
  const int* grad_in;
  const int* grad_reg;
  // learnable equation parameters (ppsci_plan_spec.aux_bcast / pgrad_*): passed by value, at most PPSCI_MAX_PGRAD terms
  int n_pgrad;
  int pgrad_res[PPSCI_MAX_PGRAD];
  int pgrad_aux[PPSCI_MAX_PGRAD];
  int pgrad_reg[PPSCI_MAX_PGRAD];
};

template <typename T>
struct HeadArgs {
  HeadProgram P;
  int C, n_out, n_in, n_aux;
  const T* Y;  // [C][Np][ldy]
  int ldy;
  long long yplane;
  T* Ybar;  // same layout, may be null
  const void* x_cols[PPSCI_MAX_IN];
  const void* aux_cols[PPSCI_MAX_IN];
  int aux_bcast[PPSCI_MAX_IN];      // 1: aux_cols[a] is one scalar (a learnable parameter), not a column
  double* aux_grad[PPSCI_MAX_IN];   // fp64 accumulators of dLoss/d(parameter a), or null
  long long x_off;  // chunk offset into the caller's columns
  long long Np;
  const void* label_cols[PPSCI_MAX_RES];
  double label_const[PPSCI_MAX_RES];
  const void* weight_cols[PPSCI_MAX_RES];
  double coef[PPSCI_MAX_RES];  // loss_weight * (1/n_norm for mean)
  void* residual_out[PPSCI_MAX_RES];
  double* loss_acc;  // [n_res] fp64 accumulators (may be null for fwd-only)
};

template <typename T>
__device__ __forceinline__ T vm_powi(T a, int e) {
  if (e == 0) return T(1);
  bool neg = e < 0;
  unsigned u = neg ? (unsigned)(-e) : (unsigned)e;
  T r = T(1), b = a;
  while (u) {
    if (u & 1u) r *= b;
    b *= b;
    u >>= 1;
  }
  return neg ? T(1) / r : r;
}

template <typename T>
__device__ __forceinline__ void vm_run(const HeadProgram& P, T* r) {
  for (int i = 0; i < P.n_ops; ++i) {
    const int op = P.prog[4 * i], dst = P.prog[4 * i + 1], a = P.prog[4 * i + 2], b = P.prog[4 * i + 3];
    T v;
    switch (op) {
      case PPSCI_OP_CONST: v = T(P.consts[a]); break;
      case PPSCI_OP_MOV: v = r[a]; break;
      case PPSCI_OP_ADD: v = r[a] + r[b]; break;
      case PPSCI_OP_SUB: v = r[a] - r[b]; break;
      case PPSCI_OP_MUL: v = r[a] * r[b]; break;
      case PPSCI_OP_DIV: v = r[a] / r[b]; break;
      case PPSCI_OP_NEG: v = -r[a]; break;
      case PPSCI_OP_POWI: v = vm_powi<T>(r[a], b); break;
      case PPSCI_OP_POW: v = T(pow((double)r[a], (double)r[b])); break;
      case PPSCI_OP_SIN: v = T(sin((double)r[a])); break;
      case PPSCI_OP_COS: v = T(cos((double)r[a])); break;
      case PPSCI_OP_TANH: v = T(tanh((double)r[a])); break;
      case PPSCI_OP_EXP: v = T(exp((double)r[a])); break;
      case PPSCI_OP_LOG: v = T(log((double)r[a])); break;
      case PPSCI_OP_SQRT: v = T(sqrt((double)r[a])); break;
      case PPSCI_OP_ABS: v = r[a] < T(0) ? -r[a] : r[a]; break;
      case PPSCI_OP_MAX: v = r[a] > r[b] ? r[a] : r[b]; break;
      case PPSCI_OP_MIN: v = r[a] < r[b] ? r[a] : r[b]; break;
      case PPSCI_OP_SIGN: v = r[a] > T(0) ? T(1) : (r[a] < T(0) ? T(-1) : T(0)); break;
      case PPSCI_OP_FMA: v = r[a] * r[b] + r[dst]; break;
      case PPSCI_OP_SINH: v = T(sinh((double)r[a])); break;
      case PPSCI_OP_COSH: v = T(cosh((double)r[a])); break;
      case PPSCI_OP_HEAVISIDE: v = r[a] > T(0) ? T(1) : (r[a] < T(0) ? T(0) : T(0.5)); break;
      default: v = T(0); break;
    }
    r[dst] = v;
  }
}

constexpr int HEAD_THREADS = 128;

template <typename T>
__global__ void __launch_bounds__(HEAD_THREADS) k_head(HeadArgs<T> h) {
  __shared__ double red[HEAD_THREADS];
  const long long p = (long long)blockIdx.x * HEAD_THREADS + threadIdx.x;
  const bool valid = p < h.Np;
  T r[PPSCI_MAX_REG];
  T rb[PPSCI_MAX_RES];
  double part[PPSCI_MAX_RES];
  const int nY = h.C * h.n_out;
  if (valid) {
    for (int c = 0; c < h.C; ++c)
      for (int j = 0; j < h.n_out; ++j) r[c * h.n_out + j] = h.Y[(long long)c * h.yplane + p * h.ldy + j];
    for (int i = 0; i < h.n_in; ++i) r[nY + i] = reinterpret_cast<const T*>(h.x_cols[i])[h.x_off + p];
    for (int a = 0; a < h.n_aux; ++a)
      r[nY + h.n_in + a] = reinterpret_cast<const T*>(h.aux_cols[a])[h.aux_bcast[a] ? 0 : h.x_off + p];
    vm_run<T>(h.P, r);
  }
  for (int k = 0; k < h.P.n_res; ++k) {
    T res = T(0), e = T(0), w = T(1);
    if (valid) {
      res = r[h.P.res_reg[k]];
      if (h.residual_out[k]) reinterpret_cast<T*>(h.residual_out[k])[h.x_off + p] = res;
      const T label = h.label_cols[k] ? reinterpret_cast<const T*>(h.label_cols[k])[h.x_off + p]
                                      : T(h.label_const[k]);
      w = h.weight_cols[k] ? reinterpret_cast<const T*>(h.weight_cols[k])[h.x_off + p] : T(1);
      e = res - label;
    }
    const T coef = T(h.coef[k]);
    rb[k] = valid ? T(2) * e * w * coef : T(0);
    part[k] = valid ? (double)(w * e * e) * h.coef[k] : 0.0;
  }
  if (h.loss_acc) {
    for (int k = 0; k < h.P.n_res; ++k) {
      red[threadIdx.x] = part[k];
      __syncthreads();
      for (int s = HEAD_THREADS / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
      }
      if (threadIdx.x == 0) atomicAdd(h.loss_acc + k, red[0]);
      __syncthreads();
    }
  }
  // dLoss/d(learnable parameter a) = sum over points and residuals of (2 coef w e) * d residual / d parameter
  if (h.P.n_pgrad > 0 && h.Ybar) {
    for (int a = 0; a < h.n_aux; ++a) {
      if (!h.aux_grad[a]) continue;  // uniform across the block
      double acc = 0.0;
      if (valid)
        for (int g = 0; g < h.P.n_pgrad; ++g)
          if (h.P.pgrad_aux[g] == a) acc += (double)(rb[h.P.pgrad_res[g]] * r[h.P.pgrad_reg[g]]);
      red[threadIdx.x] = acc;
      __syncthreads();
      for (int s = HEAD_THREADS / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
      }
      if (threadIdx.x == 0) atomicAdd(h.aux_grad[a], red[0]);
      __syncthreads();
    }
  }
  if (h.Ybar && valid) {
    // grad list is sorted by grad_in; every output-jet register gets a value (zero if absent)
    int gi = 0;
    for (int idx = 0; idx < nY; ++idx) {
      T acc = T(0);
      while (gi < h.P.n_grad && h.P.grad_in[gi] == idx) {
        acc += rb[h.P.grad_res[gi]] * r[h.P.grad_reg[gi]];
        ++gi;
      }
      const int c = idx / h.n_out, j = idx % h.n_out;
      h.Ybar[(long long)c * h.yplane + p * h.ldy + j] = acc;
    }
  }
}

// DeepONet head (reference: ppsci/arch/deeponet.py:141-149 + ppsci/loss/mse.py:82-106 for the one output G):
//   G[p] = sum_i b[p][i] * sigma(t[p][i]) + bias ,  e = G - label ,  loss += coef * w[p] * e^2 ,
//   gbar = 2 coef w e ,  bbar[p][i] = gbar sigma(t_i) ,  tbar[p][i] = gbar b_i sigma'(t_i) ,  dbias += gbar.
// One warp per point and pass (lanes stride the feature dimension: coalesced rows); bbar / tbar may alias b / t.
template <typename T>
__global__ void __launch_bounds__(256) k_deeponet_head(const T* b, const T* t, const T* __restrict__ bias, int act,
                                                       const T* __restrict__ label, const T* __restrict__ weight, long long n, int F,
                                                       double coef, T* __restrict__ g_out, double* __restrict__ loss_acc, T* bbar,
                                                       T* tbar, T* __restrict__ dbias) {
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const T bias_v = bias ? bias[0] : T(0);
  double loss_part = 0.0;
  T db_part = T(0);
  for (long long p = (long long)blockIdx.x * wpb + wib; p < n; p += (long long)gridDim.x * wpb) {
    const T* bp = b + p * F;
    const T* tp = t + p * F;
    T acc = T(0);
    for (int i = lane; i < F; i += 32) {
      T y0, sc[6];
      act_coef<T, 1>(act, tp[i], y0, sc);
      acc += bp[i] * y0;
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    const T gval = acc + bias_v;
    if (g_out && lane == 0) g_out[p] = gval;
    if (!bbar) continue;
    const T e = gval - (label ? label[p] : T(0));
    const T w = weight ? weight[p] : T(1);
    const T gbar = (T)(2.0 * coef) * w * e;
    if (lane == 0) {
      loss_part += coef * (double)w * (double)e * (double)e;
      db_part += gbar;
    }
    for (int i = lane; i < F; i += 32) {
      T y0, sc[6];
      const T bv = bp[i];
      act_coef<T, 1>(act, tp[i], y0, sc);
      bbar[p * F + i] = gbar * y0;
      tbar[p * F + i] = gbar * bv * sc[1];
    }
  }
  if (bbar && lane == 0) {
    if (loss_acc) atomicAdd(loss_acc, loss_part);
    if (dbias) atomicAdd(dbias, db_part);
  }
}

// Device-side collocation sampling (SURVEY section 8(f) rank 4): uniform points in a box, Philox4x32-10 counter-based
// generator (Salmon et al., SC'11) keyed by `seed`, counter = (point index + offset, dimension group).  Replaces the
// per-step numpy RNG + H2D copy of ContinuousNamedArrayDataset (ppsci/data/dataset/array_dataset.py:208-228) for boxes;
// the stream is NOT numpy's (MT19937 cannot be reproduced on the device) — host sampling stays the bit-exact mode.
__host__ __device__ inline void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k0, n1 = (uint32_t)p1;
    const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k1, n3 = (uint32_t)p0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}
struct SampleArgs {
  void* cols[PPSCI_MAX_IN];
  double lo[PPSCI_MAX_IN], hi[PPSCI_MAX_IN];
  int ndim;
  long long n;
  unsigned long long seed, offset;
};
template <typename T>
__global__ void k_sample_uniform(SampleArgs a) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const unsigned long long ctr = a.offset + (unsigned long long)i;
  for (int d0 = 0; d0 < a.ndim; d0 += 2) {  // one Philox block = 4 words = two 53-bit (or four 24-bit) uniforms
    uint32_t c[4] = {(uint32_t)ctr, (uint32_t)(ctr >> 32), (uint32_t)(d0 >> 1), 0u};
    philox4x32_10(c, (uint32_t)a.seed, (uint32_t)(a.seed >> 32));
    for (int j = 0; j < 2 && d0 + j < a.ndim; ++j) {
      double u;
      if (sizeof(T) == 8) u = (double)((((unsigned long long)c[2 * j] << 32) | c[2 * j + 1]) >> 11) * (1.0 / 9007199254740992.0);
      else u = (double)(c[2 * j] >> 8) * (1.0 / 16777216.0);
      reinterpret_cast<T*>(a.cols[d0 + j])[i] = (T)(a.lo[d0 + j] + (a.hi[d0 + j] - a.lo[d0 + j]) * u);
    }
  }
}

template <typename T>
__global__ void k_finalize_loss(const double* acc, T* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = T(acc[i]);
}

// jets_out[c][x_off + p][j] (plane = n_total*n_out)  <-  Y[c][p][j]
template <typename T>
__global__ void k_copy_jets(const T* Y, int ldy, long long yplane, T* out, long long n_total,
                            long long x_off, long long Np, int C, int n_out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long tot = (long long)C * Np * n_out;
  if (i >= tot) return;
  const int j = (int)(i % n_out);
  const long long p = (i / n_out) % Np;
  const int c = (int)(i / (n_out * Np));
  out[((long long)c * n_total + x_off + p) * n_out + j] = Y[(long long)c * yplane + p * ldy + j];
}

// ---- fused Adam on flat buffers (paddle.optimizer.Adam semantics, no amsgrad) ------------------
template <typename T>
__global__ void k_adam(T* p, const T* g, T* m, T* v, long long n, double lr, double b1, double b2,
                       double eps, double wd, double bc1, double bc2, double gscale) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double gi = (double)g[i] * gscale;
  double pi = (double)p[i];
  if (wd > 0.0) gi += wd * pi;                 // Adam: L2 regularisation folded into the gradient
  else if (wd < 0.0) pi *= 1.0 + lr * wd;      // AdamW: decoupled decay, coefficient -wd (p <- p (1 - lr coeff) first)
  const double mi = b1 * (double)m[i] + (1.0 - b1) * gi;
  const double vi = b2 * (double)v[i] + (1.0 - b2) * gi * gi;
  m[i] = T(mi);
  v[i] = T(vi);
  const double denom = sqrt(vi) / sqrt(bc2) + eps;
  p[i] = T(pi - (lr / bc1) * mi / denom);
}

// Same update with the per-step scalars read from device memory (hyper = {lr, 1 - beta1^t, 1 - beta2^t, grad_scale}) so
// that the launch can sit inside a captured CUDA graph and be replayed with new values; optionally clears the gradient
// it consumed (the step's  clear_grad  without another launch).
template <typename T>
__global__ void k_adam_dev(T* p, T* g, T* m, T* v, long long n, const double* __restrict__ hyper, double b1, double b2,
                           double eps, double wd, int zero_grads) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double lr = hyper[0], bc1 = hyper[1], bc2 = hyper[2], gscale = hyper[3];
  double gi = (double)g[i] * gscale;
  double pi = (double)p[i];
  if (wd > 0.0) gi += wd * pi;                 // Adam: L2 regularisation folded into the gradient
  else if (wd < 0.0) pi *= 1.0 + lr * wd;      // AdamW: decoupled decay, coefficient -wd (p <- p (1 - lr coeff) first)
  const double mi = b1 * (double)m[i] + (1.0 - b1) * gi;
  const double vi = b2 * (double)v[i] + (1.0 - b2) * gi * gi;
  m[i] = T(mi);
  v[i] = T(vi);
  const double denom = sqrt(vi) / sqrt(bc2) + eps;
  p[i] = T(pi - (lr / bc1) * mi / denom);
  if (zero_grads) g[i] = T(0);
}

}  // namespace ppsci
