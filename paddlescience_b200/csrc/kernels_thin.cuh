// kernels_thin.cuh — fp32, compile-time-jet-layout versions of the thin first / last layer kernels.
//
// The input layer (K = n_feat = 2..8) and the output layer (N = n_out = 1..8) are pure HBM streams: one pass
// over a [C][Np][width] jet plane set.  The generic kernels in kernels_simt.cuh keep the channel structure at run
// time (channel-indexed accumulators end up in local memory) and move 4 bytes per thread and instruction; these
// specialisations fix the layout at compile time (ThinLays, jet_layout.cuh), move 16 bytes per thread and instruction along the
// hidden dimension, and evaluate the input seeds once per point into shared memory instead of once per thread.
// Same arithmetic (jet_math.h); the generic kernels remain the fallback (fp64, runtime layouts, odd widths) and
// the on-GPU cross-check (PPSCI_B200_NO_THINV=1).
#pragma once
#include "kernels_simt.cuh"

namespace ppsci {
namespace thin {

constexpr int PB = 32;  // points per seed tile

__device__ __forceinline__ float f4c(const float4& v, int t) { return t == 0 ? v.x : t == 1 ? v.y : t == 2 ? v.z : v.w; }

// seeds of PB points -> shared memory  sS[pt][f][c]
template <class L>
__device__ __forceinline__ void stage_seeds(const FirstArgs<float>& g, long long p0, float (*sS)[THIN_MAXF][L::CS]) {
  for (int idx = threadIdx.x; idx < PB * g.nf; idx += blockDim.x) {
    const int pt = idx / g.nf, f = idx - pt * g.nf;
    const long long p = p0 + pt;
    const bool ok = p < g.Np;
    produce_a<float, L::KM>(g.A, g.J, ok ? p : 0, f, ok, [&](int c, float v) {
      if (c < L::CS) sS[pt][f][c] = v;
    });
  }
}

// Z_1[c][p][n] = sum_f seed_c[p][f] W[f][n] (+ b[n] on the value channel).  Block = PB points x all columns.
template <class L>
__global__ void __launch_bounds__(256) k_first_fwd_v(FirstArgs<float> g) {
  constexpr int CS = L::CS;
  __shared__ float sS[PB][THIN_MAXF][CS];
  const int tid = threadIdx.x;
  const long long p0 = (long long)blockIdx.x * PB;
  stage_seeds<L>(g, p0, sS);
  __syncthreads();
  const int lane4 = tid >> 6;
  for (int nq = tid & 63; nq * 4 < g.N; nq += 64) {
    float w[THIN_MAXF][4], b[4];
#pragma unroll
    for (int f = 0; f < THIN_MAXF; ++f)
#pragma unroll
      for (int t = 0; t < 4; ++t) w[f][t] = f < g.nf ? __ldg(g.W + (long long)f * g.N + 4 * nq + t) : 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) b[t] = __ldg(g.bias + 4 * nq + t);
    for (int pt = lane4; pt < PB; pt += 4) {
      const long long p = p0 + pt;
      if (p >= g.Np) break;
      float* out = g.Out + p * g.ldo + 4 * nq;
#pragma unroll
      for (int c = 0; c < CS; ++c) {
        float acc[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) acc[t] = c == 0 ? b[t] : 0.f;
#pragma unroll
        for (int f = 0; f < THIN_MAXF; ++f)
          if (f < g.nf) {
            const float sv = sS[pt][f][c];
#pragma unroll
            for (int t = 0; t < 4; ++t) acc[t] += sv * w[f][t];
          }
        *reinterpret_cast<float4*>(out + (long long)c * g.oplane) = make_float4(acc[0], acc[1], acc[2], acc[3]);
      }
    }
  }
}

// dW_1[f][n] += sum_{c,p} seed_c[p][f] Zbar_1[c][p][n] ;  db_1[n] += sum_p Zbar_1[0][p][n]
// grid (ceil(N / 256), ceil(Np / pts_per_block)), pts_per_block a multiple of PB.
template <class L>
__global__ void __launch_bounds__(256) k_first_dw_v(FirstArgs<float> g) {
  constexpr int CS = L::CS;
  __shared__ float sS[PB][THIN_MAXF][CS];
  __shared__ float red[3][64][4];
  const int tid = threadIdx.x;
  const int nq = blockIdx.x * 64 + (tid & 63), lane4 = tid >> 6;
  const bool n_ok = nq * 4 < g.N;
  const long long p_begin = (long long)blockIdx.y * g.pts_per_block;
  long long p_end = p_begin + g.pts_per_block;
  if (p_end > g.Np) p_end = g.Np;
  float acc[THIN_MAXF + 1][4];  // [nf] = bias gradient
#pragma unroll
  for (int f = 0; f <= THIN_MAXF; ++f)
#pragma unroll
    for (int t = 0; t < 4; ++t) acc[f][t] = 0.f;
  for (long long p0 = p_begin; p0 < p_end; p0 += PB) {
    __syncthreads();
    stage_seeds<L>(g, p0, sS);
    __syncthreads();
    if (!n_ok) continue;
    for (int pt = lane4; pt < PB; pt += 4) {
      const long long p = p0 + pt;
      if (p >= p_end) break;
      const float* zb = g.Zbar + p * g.ldzb + 4 * nq;
      float4 z[CS];
#pragma unroll
      for (int c = 0; c < CS; ++c) z[c] = __ldg(reinterpret_cast<const float4*>(zb + (long long)c * g.zbplane));
#pragma unroll
      for (int t = 0; t < 4; ++t) acc[THIN_MAXF][t] += f4c(z[0], t);
#pragma unroll
      for (int f = 0; f < THIN_MAXF; ++f)
        if (f < g.nf) {
#pragma unroll
          for (int c = 0; c < CS; ++c) {
            const float sv = sS[pt][f][c];
#pragma unroll
            for (int t = 0; t < 4; ++t) acc[f][t] += sv * f4c(z[c], t);
          }
        }
    }
  }
  // reduce the four point lanes, then one atomic per (f, n)
  for (int f = 0; f <= THIN_MAXF; ++f) {
    if (f < THIN_MAXF && f >= g.nf) continue;
    __syncthreads();
    if (lane4 > 0)
#pragma unroll
      for (int t = 0; t < 4; ++t) red[lane4 - 1][tid & 63][t] = acc[f][t];
    __syncthreads();
    if (lane4 == 0 && n_ok) {
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float v = acc[f][t] + red[0][tid & 63][t] + red[1][tid & 63][t] + red[2][tid & 63][t];
        if (f < THIN_MAXF) atomicAdd(g.dW + (long long)f * g.N + 4 * nq + t, v);
        else atomicAdd(g.db + 4 * nq + t, v);
      }
    }
  }
}

// Y[c][p][j] = sum_k act_jets(Z_{L-1})[c][p][k] W[k][j] (+ b[j] on the value channel); one warp per point,
// lanes along k in quads.
template <class L, int M>
__global__ void __launch_bounds__(256) k_last_fwd_v(LastArgs<float> g) {
  constexpr int CS = L::CS;
  const int lane = threadIdx.x & 31;
  const long long p = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (p >= g.Np) return;  // whole warp exits together
  float acc[CS][M];
#pragma unroll
  for (int c = 0; c < CS; ++c)
#pragma unroll
    for (int j = 0; j < M; ++j) acc[c][j] = 0.f;
  for (int kq = lane; kq * 4 < g.K; kq += 32) {
    const float* zp = g.A.Z + p * g.A.ld + 4 * kq;
    float4 z[CS];
#pragma unroll
    for (int c = 0; c < CS; ++c) z[c] = __ldg(reinterpret_cast<const float4*>(zp + (long long)c * g.A.plane));
    float a[CS][4];  // activation jets of the 4 hidden units
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      float sc[6], y0;
      act_coef<float, L::KM>(g.A.act, f4c(z[0], t), y0, sc);
      a[0][t] = y0;
      jet_fwd<float, L>(g.J, sc, [&](int c) { return f4c(z[c], t); }, [&](int c, float v) { a[c][t] = v; });
    }
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      float w[M];
#pragma unroll
      for (int j = 0; j < M; ++j) w[j] = __ldg(g.W + (long long)(4 * kq + t) * M + j);
#pragma unroll
      for (int c = 0; c < CS; ++c)
#pragma unroll
        for (int j = 0; j < M; ++j) acc[c][j] += a[c][t] * w[j];
    }
  }
#pragma unroll
  for (int c = 0; c < CS; ++c)
#pragma unroll
    for (int j = 0; j < M; ++j) {
      const float v = warp_sum<float>(acc[c][j]);
      if (lane == 0) g.Y[(long long)c * g.yplane + p * g.ldy + j] = v + (c == 0 ? __ldg(g.bias + j) : 0.f);
    }
}

// Output layer backward, fused (see k_last_bwd).  Block = 64 k quads x 4 point lanes; grid (ceil(K/256), point blocks).
template <class L, int M>
__global__ void __launch_bounds__(256) k_last_bwd_v(LastArgs<float> g) {
  constexpr int CS = L::CS;
  __shared__ float red[3][64][4 * M];
  const int tid = threadIdx.x;
  const int kq = blockIdx.x * 64 + (tid & 63), lane4 = tid >> 6;
  const bool k_ok = kq * 4 < g.K;
  const long long p_begin = (long long)blockIdx.y * g.pts_per_block;
  long long p_end = p_begin + g.pts_per_block;
  if (p_end > g.Np) p_end = g.Np;
  float w[4][M], dwacc[4][M], dbacc[M];
#pragma unroll
  for (int t = 0; t < 4; ++t)
#pragma unroll
    for (int j = 0; j < M; ++j) {
      w[t][j] = k_ok ? __ldg(g.W + (long long)(4 * kq + t) * M + j) : 0.f;
      dwacc[t][j] = 0.f;
    }
#pragma unroll
  for (int j = 0; j < M; ++j) dbacc[j] = 0.f;
  const bool do_db = (blockIdx.x == 0 && (tid & 63) == 0);
  if (k_ok) {
    for (long long p = p_begin + lane4; p < p_end; p += 4) {
      const float* ybp = g.Ybar + p * g.ldy;
      float yb[CS][M];
#pragma unroll
      for (int c = 0; c < CS; ++c)
#pragma unroll
        for (int j = 0; j < M; ++j) yb[c][j] = __ldg(ybp + (long long)c * g.yplane + j);
      const float* zp = g.A.Z + p * g.A.ld + 4 * kq;
      float4 z[CS];
#pragma unroll
      for (int c = 0; c < CS; ++c) z[c] = __ldg(reinterpret_cast<const float4*>(zp + (long long)c * g.A.plane));
      if (do_db)
#pragma unroll
        for (int j = 0; j < M; ++j) dbacc[j] += yb[0][j];
      float ob[CS][4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        auto ldz = [&](int c) { return f4c(z[c], t); };
        auto abar = [&](int c) {  // adjoint of activation jet channel c of unit 4 kq + t
          float a = 0.f;
#pragma unroll
          for (int j = 0; j < M; ++j) a += yb[c][j] * w[t][j];
          return a;
        };
        float sc[6], y0;
        act_coef<float, L::KM + 1>(g.A.act, f4c(z[0], t), y0, sc);
#pragma unroll
        for (int j = 0; j < M; ++j) dwacc[t][j] += y0 * yb[0][j];
        jet_fwd<float, L>(g.J, sc, ldz, [&](int c, float v) {
#pragma unroll
          for (int j = 0; j < M; ++j) dwacc[t][j] += v * yb[c][j];
        });
        ob[0][t] = jet_adj<float, L>(g.J, sc, ldz, abar, [&](int c, float v) { ob[c][t] = v; });
      }
      float* out = g.ZbarOut + p * g.ldo + 4 * kq;
#pragma unroll
      for (int c = 0; c < CS; ++c)
        *reinterpret_cast<float4*>(out + (long long)c * g.oplane) = make_float4(ob[c][0], ob[c][1], ob[c][2], ob[c][3]);
    }
  }
  // reduce the four point lanes, then one atomic per (k, j)
  if (lane4 > 0)
#pragma unroll
    for (int t = 0; t < 4; ++t)
#pragma unroll
      for (int j = 0; j < M; ++j) red[lane4 - 1][tid & 63][t * M + j] = dwacc[t][j];
  __syncthreads();
  if (lane4 == 0 && k_ok) {
#pragma unroll
    for (int t = 0; t < 4; ++t)
#pragma unroll
      for (int j = 0; j < M; ++j) {
        const int i = t * M + j;
        atomicAdd(g.dW + (long long)(4 * kq + t) * M + j, dwacc[t][j] + red[0][tid & 63][i] + red[1][tid & 63][i] + red[2][tid & 63][i]);
      }
  }
  if (do_db) {
#pragma unroll
    for (int j = 0; j < M; ++j) atomicAdd(g.db + j, dbacc[j]);
  }
}

}  // namespace thin
}  // namespace ppsci
