// kernels_wgmma.cuh — Hopper (sm_90a) tensor-core kernels for the fp32 layers (K a multiple of 32 up to 1024, N a
// multiple of 32 up to 256) with one of the compile-time jet layouts: the forward  Z_l = act_jets(Z_{l-1}) W_l + b_l, the
// dx  Zbar_{l-1} = adj(Zbar_l W_l^T, Z_{l-1})  (k_wg_layer) and the weight gradient (k_wg_dw, further down).
//
// fp32-faithful contraction on TF32 tensor cores: every operand is split x = hi + lo with hi = rn_tf32(x), lo = x - hi
// (exact in fp32), and each K step computes  A_hi B_hi + A_lo B_hi + A_hi B_lo  (3xTF32; the dropped A_lo B_lo term is
// O(2^-22) relative).  The tensor cores round every accumulation into an fp32 accumulator at the accumulator's
// magnitude, so the exact-product term A_hi B_hi gets an accumulator of its own (one rounding per K step at the full
// magnitude of the result instead of three); the cross terms, 2^-11 of the result, share the second one.  Measured on
// an H100 80GB HBM3 (400 W power limit), cfg3 (6 x 256): one shared accumulator gave a residual error of 1.7e-5 against
// the fp64 oracle, above the 1e-5 bar.
//
// A CTA of two warpgroups owns a tile of 64 jet rows (TP = 64 / C points x C channels, row r = c TP + pl); both
// warpgroups issue wgmma.mma_async m64n64k8 over all 64 rows (N / 64 column blocks, and one m64n32k8 block when N is an
// odd multiple of 32): warpgroup 0 accumulates
// A_hi B_hi, warpgroup 1 A_lo B_hi + A_hi B_lo, both in registers; the epilogue adds the two through shared memory.  Per
// 32-wide K chunk all threads write the activation jets of the previous layer's pre-activations, split into hi / lo,
// into the chunk's A stage (K-major, 128-byte rows, 128-byte swizzle); one thread stages the chunk of the pre-swizzled
// weight image (prepared once per call by k_wg_prep_w) with a TMA bulk copy onto an mbarrier.  Two stages: the MMAs of
// chunk j run while the operands of chunk j + 1 are produced.  Persistent: CTA b handles tiles b, b + grid, ...
#pragma once

#include "kernels_thin.cuh"

#ifndef PPSCI_EMUL
#include <stdint.h>

namespace ppsci {
namespace wg {

constexpr int KCH = 32;                      // K elements per chunk = one 128-byte swizzle row of tf32
constexpr int THREADS = 256;                 // two warpgroups
constexpr int TM = 64;                       // jet rows per tile
constexpr int A_TILE_BYTES = TM * KCH * 4;   // 8 KB (one of hi / lo)
__host__ __device__ inline int tile_points(int C) { return TM / C; }

__host__ __device__ inline int stage_bytes(int N) { return 2 * A_TILE_BYTES + 2 * N * KCH * 4; }
// two stages, then an all-zero A tile (operand of warpgroup 0's second MMA per K step), then the mbarriers
__host__ __device__ inline int fwd_smem_bytes(int N) { return 2 * stage_bytes(N) + A_TILE_BYTES + 1024 + 64; }

// byte offset of element (row, kk) inside a [rows x 32 fp32] K-major 128-byte-swizzled tile
__host__ __device__ __forceinline__ uint32_t sw128(int row, int kk) {
  return (uint32_t)(row * 128 + ((((kk >> 2) ^ row) & 7) << 4) + ((kk & 3) << 2));
}
__device__ __forceinline__ uint32_t sw128_q(int row, int kq) { return (uint32_t)(row * 128 + (((kq ^ row) & 7) << 4)); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ float tf32_rn(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}

// ---- mbarrier + TMA bulk copy --------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (reported as a CUDA error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// generic-proxy shared-memory writes become visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma ------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor: K-major, 128-byte swizzle, 8-row groups 1024 B apart (stride byte offset), leading
// byte offset unused for swizzled K-major layouts.  The tile base must be 1024-byte aligned; a K step of 8 tf32 inside
// the swizzle row advances the start address by 32 bytes.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);  // start address, bits [0,14)
  d |= (uint64_t)1 << 16;                    // leading byte offset >> 4, bits [16,30)
  d |= (uint64_t)(1024 >> 4) << 32;          // stride byte offset >> 4, bits [32,46)
  d |= (uint64_t)1 << 62;                    // layout type: 128-byte swizzle, bits [62,64)
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// D[64 x 64] (+)= A[64 x 8] B[8 x 64], tf32 operands from shared memory, fp32 accumulators in registers
__device__ __forceinline__ void wgmma_tf32_m64n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate));
}

// D[64 x 32] (+)= A[64 x 8] B[8 x 32]
__device__ __forceinline__ void wgmma_tf32_m64n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(accumulate));
}

// ---- weight image: img[j][part][sw128(n, kk)] = split(B[n][32 j + kk]), part 0 = hi, 1 = lo ----------------------
// transposed = 0: B[n][k] = W[k N + n]   (forward: W is [K = in][N = out] row-major)
// transposed = 1: B[n][k] = W[n K + k]   (dx: contraction over the layer's outputs)
__global__ void k_wg_prep_w(const float* __restrict__ W, float* __restrict__ img, int K, int N, int transposed) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)K * N) return;
  const int n = (int)(i / K), k = (int)(i % K);
  const float w = transposed ? W[(long long)n * K + k] : W[(long long)k * N + n];
  const float hi = tf32_rn(w);
  float* blk = img + (long long)(k / KCH) * 2 * N * KCH;
  const uint32_t off = sw128(n, k % KCH) >> 2;
  blk[off] = hi;
  blk[(long long)N * KCH + off] = w - hi;
}

struct WgArgs {
  AOperand<float> A;    // forward: A_ACT over Z_{l-1}; dx: A_PLAIN over Zbar_l
  JetLayout J;
  const float* Wimg;    // [K/32][2][N*32] swizzled hi / lo images
  int Kdim;
  int Kvalid;           // operand columns that exist (0 = Kdim): a dense first-layer operand [Np][100] is read as [Np][128]
  int Nout;
  const float* bias;    // forward only
  float* Out;           // forward: Z_l; dx: Zbar_{l-1}
  int ldo;
  long long oplane;
  long long Np;
  int num_tiles;
  const float* Zprev;   // dx: Z_{l-1} [C][Np][ldz] and the activation applied to it
  int ldz;
  long long zplane;
  int act;
};

// Epilogue scratch, free once every MMA of the tile has retired: the B region of stage 0 takes warpgroup 1's accumulators
// (fragment order), the B region of stage 1 the dx exchange tile [64 rows][N] (16-byte chunks XOR-swizzled by r & 7).
__device__ __forceinline__ unsigned char* xchg(unsigned char* base_ptr, int sbytes, int N, int r, int col) {
  return base_ptr + sbytes + 2 * A_TILE_BYTES + r * N * 4 + ((((col >> 2) ^ r) & 7) << 4) + (((col >> 2) & ~7) << 4) +
         (col & 3) * 4;
}

// DX = false: forward  Z_l = act_jets(Z_{l-1}) W_l + b_l.
// DX = true:  Abar = Zbar_l W_l^T on the tensor cores, then the activation adjoint  Zbar_{l-1} = adj(Abar, Z_{l-1}); the
// C channels of one point sit in different accumulator rows, so the accumulators go through a shared-memory exchange tile.
template <class L, int NQ, bool DX>
__global__ void __launch_bounds__(THREADS, 1) k_wg_layer(WgArgs g) {
  PPSCI_DYN_SMEM(smem_dyn);
  const uint32_t base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  unsigned char* base_ptr = smem_dyn + (base - smem_u32(smem_dyn));
  constexpr int CS = L::CS;
  constexpr int TP = TM / CS;
  constexpr int rows_used = CS * TP;
  constexpr int PPR = (THREADS / 32) * 4;  // points per pass of the producers
  constexpr int MAXI = (TP + PPR - 1) / PPR;
  constexpr int N = NQ * 32;  // output columns: NB blocks of 64, then a block of 32 if TAIL
  constexpr int NB = NQ / 2, TAIL = NQ & 1;
  const int sbytes = stage_bytes(N);
  const uint32_t bar0 = base + 2 * sbytes + A_TILE_BYTES;  // two mbarriers: weight chunk of stage 0 / 1 landed
  const uint32_t b_bytes = (uint32_t)(2 * N * KCH * 4);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = tid >> 7;
  const int kq = lane & 7, psub = lane >> 3;
  const int nchunks = g.Kdim / KCH;
  const int act = g.A.act;

  if (tid == 0) {
    mbar_init(bar0, 1);
    mbar_init(bar0 + 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int s = 0; s < 3; ++s) {  // A pad rows (>= rows_used) stay zero operands for good; s = 2: the zero tile
    float4* az = reinterpret_cast<float4*>(base_ptr + s * sbytes);
    for (int i = tid; i < (s < 2 ? 2 : 1) * A_TILE_BYTES / 16; i += THREADS) az[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  fence_proxy_async();
  __syncthreads();

  float acc[NB > 0 ? NB : 1][32], acct[TAIL ? 16 : 1];
  // registers of accumulator fragment (row group h, columns 8 j + 2 (lane & 3) + b): element 2 h + b of n8 block j
  auto frag = [&](int j, int i) -> float& { return j < 8 * NB ? acc[j >> 3][4 * (j & 7) + i] : acct[4 * (j - 8 * NB) + i]; };
  uint32_t it = 0;  // running chunk counter: stage it & 1, use (it >> 1) of that stage
  for (int tile = blockIdx.x; tile < g.num_tiles; tile += gridDim.x) {
    const long long p0 = (long long)tile * TP;
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) frag(j, i) = 0.f;
    for (int j = 0; j < nchunks; ++j, ++it) {
      const uint32_t s = it & 1u;
      wgmma_wait<1>();  // this warpgroup's MMAs of chunk it - 2 (the last reader of stage s) have retired
      __syncthreads();  // ... and the other warpgroup's
      const uint32_t st_addr = base + s * sbytes;
      unsigned char* st_ptr = base_ptr + s * sbytes;
      if (tid == 0) {
        mbar_expect_tx(bar0 + 8 * s, b_bytes);
        bulk_g2s(st_addr + 2 * A_TILE_BYTES, g.Wimg + (long long)j * 2 * N * KCH, b_bytes, bar0 + 8 * s);
      }
      // A operand of this chunk: item = (point, 4 consecutive k); a quarter warp writes the 8 chunks of one row
#pragma unroll
      for (int i = 0; i < MAXI; ++i) {
        const int pl = warp * 4 + psub + i * PPR;
        if (pl >= TP) continue;
        const long long p = p0 + pl;
        bool valid = p < g.Np;
        const float* src = g.A.Z + p * g.A.ld + j * KCH + 4 * kq;
        if (g.Kvalid && j * KCH + 4 * kq >= g.Kvalid) valid = false;  // zero columns beyond a padded contraction length
        float4 z[CS];
#pragma unroll
        for (int c = 0; c < CS; ++c)
          z[c] = valid ? __ldg(reinterpret_cast<const float4*>(src + (long long)c * g.A.plane)) : make_float4(0.f, 0.f, 0.f, 0.f);
        float yout[CS][4];
        if constexpr (DX) {  // plain operand
#pragma unroll
          for (int c = 0; c < CS; ++c) {
            yout[c][0] = z[c].x; yout[c][1] = z[c].y; yout[c][2] = z[c].z; yout[c][3] = z[c].w;
          }
        } else {
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            auto comp = [&](const float4& v) { return t == 0 ? v.x : t == 1 ? v.y : t == 2 ? v.z : v.w; };
            float sc[6];
            float y0;
            act_coef<float, L::KM>(act, comp(z[0]), y0, sc);
            yout[0][t] = valid ? y0 : 0.f;
#pragma unroll
            for (int d = 0; d < L::ND; ++d) {
              const int K = L::order(g.J, d), cb = L::cbase(g.J, d);
              float zz[4], yy[4];
#pragma unroll
              for (int o = 0; o < 4; ++o) zz[o] = (o < L::KM && o < K) ? comp(z[(cb + o) < CS ? (cb + o) : 0]) : 0.f;
              jet_fwd_dir<float, L::KM>(sc, zz, yy);
#pragma unroll
              for (int o = 0; o < L::KM; ++o)
                if (o < K && cb + o < CS) yout[cb + o][t] = valid ? yy[o] : 0.f;
            }
          }
        }
#pragma unroll
        for (int c = 0; c < CS; ++c) {
          float4 h, l;
          h.x = tf32_rn(yout[c][0]); h.y = tf32_rn(yout[c][1]); h.z = tf32_rn(yout[c][2]); h.w = tf32_rn(yout[c][3]);
          l.x = yout[c][0] - h.x; l.y = yout[c][1] - h.y; l.z = yout[c][2] - h.z; l.w = yout[c][3] - h.w;
          const uint32_t off = sw128_q(c * TP + pl, kq);
          *reinterpret_cast<float4*>(st_ptr + off) = h;
          *reinterpret_cast<float4*>(st_ptr + A_TILE_BYTES + off) = l;
        }
      }
      fence_proxy_async();
      __syncthreads();
      mbar_wait(bar0 + 8 * s, (it >> 1) & 1u);
      // MMAs of this chunk: warpgroup 0 the exact-product term, warpgroup 1 the two cross terms
      const uint64_t a_hi = make_desc(st_addr), a_lo = make_desc(st_addr + A_TILE_BYTES);
      const uint64_t b_hi = make_desc(st_addr + 2 * A_TILE_BYTES), b_lo = make_desc(st_addr + 2 * A_TILE_BYTES + N * 128);
      // Both warpgroups issue the same instruction sequence (the compiler serialises wgmma issued on divergent paths):
      // warpgroup 0 A_hi B_hi + 0 B_lo (the zero tile adds an exact 0), warpgroup 1 A_lo B_hi + A_hi B_lo
      const uint64_t a1 = wgi ? a_lo : a_hi, a2 = wgi ? a_hi : make_desc(base + 2 * sbytes);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < KCH / 8; ++ks) {
        const uint64_t inc = (uint64_t)(2 * ks);  // 32 bytes in units of 16
        const uint32_t first = (j == 0 && ks == 0) ? 0u : 1u;
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) {
          const uint64_t bo = inc + (uint64_t)(nb * 64 * 128 / 16);  // column block nb = B rows 64 nb ..
          wgmma_tf32_m64n64(acc[nb], a1 + inc, b_hi + bo, first);
          wgmma_tf32_m64n64(acc[nb], a2 + inc, b_lo + bo, 1u);
        }
        if constexpr (TAIL) {
          const uint64_t bo = inc + (uint64_t)(NB * 64 * 128 / 16);  // the last 32 columns
          wgmma_tf32_m64n32(acct, a1 + inc, b_hi + bo, first);
          wgmma_tf32_m64n32(acct, a2 + inc, b_lo + bo, 1u);
        }
      }
      wgmma_commit();
    }
    wgmma_wait<0>();
    __syncthreads();  // every MMA of the tile has retired in both warpgroups: the B regions are free
    {  // warpgroup 0 adds warpgroup 1's accumulators (fragment order, conflict-free)
      float* xs = reinterpret_cast<float*>(base_ptr + 2 * A_TILE_BYTES);
      const int lt = tid & 127;
      if (wgi == 1) {
#pragma unroll
        for (int j = 0; j < N / 8; ++j)
#pragma unroll
          for (int i = 0; i < 4; ++i) xs[(4 * j + i) * 128 + lt] = frag(j, i);
      }
      __syncthreads();
      if (wgi == 0) {
#pragma unroll
        for (int j = 0; j < N / 8; ++j)
#pragma unroll
          for (int i = 0; i < 4; ++i) frag(j, i) += xs[(4 * j + i) * 128 + lt];
      }
    }
    const int rbase = (warp & 3) * 16 + (lane >> 2);  // warpgroup 0: accumulator rows rbase, rbase + 8 of this thread
    if constexpr (!DX) {
      // ---- forward epilogue: accumulator fragments (+ bias) -> Z_l; row r = c TP + pl of the tile ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = rbase + 8 * h;
        if (wgi != 0) break;
        const int c = r / TP, pl = r - c * TP;
        const long long p = p0 + pl;
        if (r >= rows_used || p >= g.Np) continue;
        float* out_row = g.Out + (long long)c * g.oplane + p * g.ldo;
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
          const int col = j * 8 + 2 * (lane & 3);
          float2 v = make_float2(frag(j, 2 * h), frag(j, 2 * h + 1));
          if (c == 0 && g.bias) {
            v.x += __ldg(g.bias + col);
            v.y += __ldg(g.bias + col + 1);
          }
          *reinterpret_cast<float2*>(out_row + col) = v;
        }
      }
      fence_proxy_async();  // warpgroup 1's scratch writes are ordered before the next tile's bulk copies
    } else {
      // ---- dx epilogue: Abar (registers) -> exchange tile -> activation adjoint with Z_{l-1} -> Zbar_{l-1} ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = rbase + 8 * h;
        if (wgi != 0) break;
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
          const int col = j * 8 + 2 * (lane & 3);
          *reinterpret_cast<float2*>(xchg(base_ptr, sbytes, N, r, col)) = make_float2(frag(j, 2 * h), frag(j, 2 * h + 1));
        }
      }
      __syncthreads();
      constexpr int N4 = N / 4;
      for (int item = tid; item < TP * N4; item += THREADS) {  // item = (point, 4 consecutive columns)
        const int pl = item / N4, q = item - pl * N4;
        const long long p = p0 + pl;
        if (p >= g.Np) continue;
        float4 zc[CS], xc[CS];
#pragma unroll
        for (int c = 0; c < CS; ++c) {
          zc[c] = __ldg(reinterpret_cast<const float4*>(g.Zprev + (long long)c * g.zplane + p * g.ldz + 4 * q));
          xc[c] = *reinterpret_cast<const float4*>(xchg(base_ptr, sbytes, N, c * TP + pl, 4 * q));
        }
        float ob[CS][4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          auto comp = [&](const float4& v) { return t == 0 ? v.x : t == 1 ? v.y : t == 2 ? v.z : v.w; };
          float sc[6];
          float y0;
          act_coef<float, L::KM + 1>(g.act, comp(zc[0]), y0, sc);
          float sb[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int d = 0; d < L::ND; ++d) {
            const int K = L::order(g.J, d), cbs = L::cbase(g.J, d);
            float zz[4], yb[4], zbv[4];
#pragma unroll
            for (int o = 0; o < 4; ++o) {
              const bool on = (o < L::KM && o < K && cbs + o < CS);
              zz[o] = on ? comp(zc[on ? cbs + o : 0]) : 0.f;
              yb[o] = on ? comp(xc[on ? cbs + o : 0]) : 0.f;
              zbv[o] = 0.f;
            }
            jet_adj_dir<float, L::KM>(sc, zz, yb, zbv, sb);
#pragma unroll
            for (int o = 0; o < L::KM; ++o)
              if (o < K && cbs + o < CS) ob[cbs + o][t] = zbv[o];
          }
          ob[0][t] = jet_adj_z0<float, L::KM>(sc, comp(xc[0]), sb);
        }
        float* out = g.Out + p * g.ldo + 4 * q;
#pragma unroll
        for (int c = 0; c < CS; ++c)
          *reinterpret_cast<float4*>(out + (long long)c * g.oplane) = make_float4(ob[c][0], ob[c][1], ob[c][2], ob[c][3]);
      }
      fence_proxy_async();  // the exchange writes are ordered before the next tile's bulk copies into the B regions
      __syncthreads();
    }
  }
}

// ---- weight gradient  dW_l[k][n] += sum over jet rows  a_{l-1}[row][k] Zbar_l[row][n] ------------------------------
// The contraction runs over jet rows, so both operands are transposes of the row-major jet planes: the A tile holds 64
// fan-in rows k x 32 jet rows (PT = 32 / C points x C channels per chunk, the activation jets of Z_{l-1} recomputed on
// the fly), the B tile N output columns x the same 32 jet rows (Zbar_l); both split hi / lo into the same K-major
// 128-byte-swizzled stages as k_wg_layer, and the same two warpgroups accumulate A_hi B_hi and the cross terms.  CTA
// (kb, split) owns dW rows [64 kb, +64) and a contiguous range of chunks; it flushes once with atomicAdd.
struct WgDwArgs {
  AOperand<float> A;   // A_ACT over Z_{l-1}
  JetLayout J;
  const float* Zbar;   // [C][Np][ldzb]
  int ldzb;
  long long zbplane;
  int Kdim;            // fan-in (rows of dW), a multiple of 4
  float* dW;           // [Kdim][N]
  long long Np;
  int chunks_per_split;
};

template <class L, int NQ>
__global__ void __launch_bounds__(THREADS, 1) k_wg_dw(WgDwArgs g) {
  PPSCI_DYN_SMEM(smem_dyn);
  const uint32_t base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  unsigned char* base_ptr = smem_dyn + (base - smem_u32(smem_dyn));
  constexpr int CS = L::CS;
  constexpr int PT = KCH / CS;  // points per chunk of 32 jet rows
  constexpr int N = NQ * 32;
  constexpr int NB = NQ / 2, TAIL = NQ & 1;
  const int sbytes = stage_bytes(N);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = tid >> 7;
  const int k0 = blockIdx.x * TM;
  const long long total_chunks = (g.Np + PT - 1) / PT;
  const long long ch_begin = (long long)blockIdx.y * g.chunks_per_split;
  const long long ch_end = ch_begin + g.chunks_per_split < total_chunks ? ch_begin + g.chunks_per_split : total_chunks;
  const int act = g.A.act;

  for (int i = tid; i < (2 * sbytes + A_TILE_BYTES) / 16; i += THREADS)  // pad jet rows (>= C PT), the zero tile
    reinterpret_cast<float4*>(base_ptr)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  fence_proxy_async();
  __syncthreads();

  float acc[NB > 0 ? NB : 1][32], acct[TAIL ? 16 : 1];
  auto frag = [&](int j, int i) -> float& { return j < 8 * NB ? acc[j >> 3][4 * (j & 7) + i] : acct[4 * (j - 8 * NB) + i]; };
#pragma unroll
  for (int j = 0; j < N / 8; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) frag(j, i) = 0.f;
  auto put = [&](unsigned char* tile_hi, int tile_lo_off, int row, int col, float v) {
    const float h = tf32_rn(v);
    *reinterpret_cast<float*>(tile_hi + sw128(row, col)) = h;
    *reinterpret_cast<float*>(tile_hi + tile_lo_off + sw128(row, col)) = v - h;
  };
  uint32_t it = 0;
  for (long long ch = ch_begin; ch < ch_end; ++ch, ++it) {
    const uint32_t s = it & 1u;
    wgmma_wait<1>();
    __syncthreads();
    const uint32_t st_addr = base + s * sbytes;
    unsigned char* st_ptr = base_ptr + s * sbytes;
    const long long p0 = ch * PT;
    // A: item = (point, 4 consecutive fan-in rows)
    for (int item = tid; item < PT * (TM / 4); item += THREADS) {
      const int pl = item / (TM / 4), kq = item - pl * (TM / 4);
      const long long p = p0 + pl;
      const bool valid = p < g.Np && k0 + 4 * kq < g.Kdim;
      const float* src = g.A.Z + p * g.A.ld + k0 + 4 * kq;
      float4 z[CS];
#pragma unroll
      for (int c = 0; c < CS; ++c)
        z[c] = valid ? __ldg(reinterpret_cast<const float4*>(src + (long long)c * g.A.plane)) : make_float4(0.f, 0.f, 0.f, 0.f);
      float yout[CS][4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        auto comp = [&](const float4& v) { return t == 0 ? v.x : t == 1 ? v.y : t == 2 ? v.z : v.w; };
        float sc[6];
        float y0;
        act_coef<float, L::KM>(act, comp(z[0]), y0, sc);
        yout[0][t] = valid ? y0 : 0.f;
#pragma unroll
        for (int d = 0; d < L::ND; ++d) {
          const int K = L::order(g.J, d), cb = L::cbase(g.J, d);
          float zz[4], yy[4];
#pragma unroll
          for (int o = 0; o < 4; ++o) zz[o] = (o < L::KM && o < K) ? comp(z[(cb + o) < CS ? (cb + o) : 0]) : 0.f;
          jet_fwd_dir<float, L::KM>(sc, zz, yy);
#pragma unroll
          for (int o = 0; o < L::KM; ++o)
            if (o < K && cb + o < CS) yout[cb + o][t] = valid ? yy[o] : 0.f;
        }
      }
#pragma unroll
      for (int c = 0; c < CS; ++c)
#pragma unroll
        for (int t = 0; t < 4; ++t) put(st_ptr, A_TILE_BYTES, 4 * kq + t, c * PT + pl, yout[c][t]);
    }
    // B: item = (point, 4 consecutive output columns)
    for (int item = tid; item < PT * (N / 4); item += THREADS) {
      const int pl = item / (N / 4), nq = item - pl * (N / 4);
      const long long p = p0 + pl;
      const bool valid = p < g.Np;
#pragma unroll
      for (int c = 0; c < CS; ++c) {
        const float4 v = valid ? __ldg(reinterpret_cast<const float4*>(g.Zbar + (long long)c * g.zbplane + p * g.ldzb + 4 * nq))
                               : make_float4(0.f, 0.f, 0.f, 0.f);
        put(st_ptr + 2 * A_TILE_BYTES, N * 128, 4 * nq, c * PT + pl, v.x);
        put(st_ptr + 2 * A_TILE_BYTES, N * 128, 4 * nq + 1, c * PT + pl, v.y);
        put(st_ptr + 2 * A_TILE_BYTES, N * 128, 4 * nq + 2, c * PT + pl, v.z);
        put(st_ptr + 2 * A_TILE_BYTES, N * 128, 4 * nq + 3, c * PT + pl, v.w);
      }
    }
    fence_proxy_async();
    __syncthreads();
    const uint64_t a_hi = make_desc(st_addr), a_lo = make_desc(st_addr + A_TILE_BYTES);
    const uint64_t b_hi = make_desc(st_addr + 2 * A_TILE_BYTES), b_lo = make_desc(st_addr + 2 * A_TILE_BYTES + N * 128);
    const uint64_t a1 = wgi ? a_lo : a_hi, a2 = wgi ? a_hi : make_desc(base + 2 * sbytes);  // as in k_wg_layer
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < KCH / 8; ++ks) {
      const uint64_t inc = (uint64_t)(2 * ks);
      const uint32_t first = (it == 0 && ks == 0) ? 0u : 1u;
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) {
        const uint64_t bo = inc + (uint64_t)(nb * 64 * 128 / 16);
        wgmma_tf32_m64n64(acc[nb], a1 + inc, b_hi + bo, first);
        wgmma_tf32_m64n64(acc[nb], a2 + inc, b_lo + bo, 1u);
      }
      if constexpr (TAIL) {
        const uint64_t bo = inc + (uint64_t)(NB * 64 * 128 / 16);
        wgmma_tf32_m64n32(acct, a1 + inc, b_hi + bo, first);
        wgmma_tf32_m64n32(acct, a2 + inc, b_lo + bo, 1u);
      }
    }
    wgmma_commit();
  }
  wgmma_wait<0>();
  __syncthreads();
  if (it == 0) return;
  float* xs = reinterpret_cast<float*>(base_ptr + 2 * A_TILE_BYTES);
  const int lt = tid & 127;
  if (wgi == 1) {
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) xs[(4 * j + i) * 128 + lt] = frag(j, i);
  }
  __syncthreads();
  if (wgi != 0) return;
  const int rbase = (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int k = k0 + rbase + 8 * h;
    if (k >= g.Kdim) continue;
    float* row = g.dW + (long long)k * N;
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      const int col = j * 8 + 2 * (lane & 3);
      atomicAdd(row + col, frag(j, 2 * h) + xs[(4 * j + 2 * h) * 128 + lt]);
      atomicAdd(row + col + 1, frag(j, 2 * h + 1) + xs[(4 * j + 2 * h + 1) * 128 + lt]);
    }
  }
}

// db_l[n] += sum over points of Zbar_l[channel 0][p][n]   (tiny, HBM-bound)
__global__ void k_wg_bias_grad(const float* __restrict__ Zbar0, int ld, long long Np, int N, float* __restrict__ db,
                               int pts_per_block) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const long long p_begin = (long long)blockIdx.y * pts_per_block;
  const long long p_end = p_begin + pts_per_block < Np ? p_begin + pts_per_block : Np;
  float acc = 0.f;
  for (long long p = p_begin; p < p_end; ++p) acc += Zbar0[p * ld + n];
  atomicAdd(db + n, acc);
}

}  // namespace wg

// jet layouts of the wgmma kernels: the thin kernels' compile-time layouts and four fourth-order directions (the
// polarised biharmonic operator)
enum { WG_LAY_4444 = 16 };
inline int wg_layout(const JetLayout& J) {
  const int lay = pick_layout(J, PPSCI_ACT_TANH);
  if (lay != LAY_DYN) return lay;
  bool o4 = J.n_dir == 4;
  for (int d = 0; d < J.n_dir; ++d) o4 = o4 && J.dir_order[d] == 4;
  return o4 ? (int)WG_LAY_4444 : (int)LAY_DYN;
}
// a GEMM of contraction length K and N output columns on k_wg_layer
inline int wg_kpad(int K) { return (K + wg::KCH - 1) / wg::KCH * wg::KCH; }
inline bool wg_shape_ok(int K, int N) { return K % wg::KCH == 0 && K >= 32 && K <= 1024 && N % 32 == 0 && N >= 32 && N <= 256; }
// fp32 layer l whose forward runs on k_wg_layer: one of the wgmma jet layouts, an activation without a trainable
// parameter; layer 1 only as a dense first layer (its operand the caller's matrix, contraction padded to 32)
inline bool wg_fwd_ok(const ppsci_plan_spec& s, int l, const JetLayout& J) {
  if (s.dtype != PPSCI_F32 || s.gated) return false;
  if (s.act == PPSCI_ACT_STAN || s.act == PPSCI_ACT_SWISH_B) return false;
  if (wg_layout(J) == LAY_DYN) return false;
  if (l == 1) return s.dense_in && s.n_layers >= 2 && s.widths[0] % 4 == 0 && wg_shape_ok(wg_kpad(s.widths[0]), s.widths[1]);
  if (l < 2 || l > s.n_layers) return false;  // l == n_layers: a wide output layer
  return wg_shape_ok(s.widths[l - 1], s.widths[l]);
}
// dx through layer l (produces Zbar_{l-1} of hidden layer l - 1): gemm K = width of layer l, gemm N = width of layer l - 1
inline bool wg_dx_ok(const ppsci_plan_spec& s, int l, const JetLayout& J) {
  if (s.dtype != PPSCI_F32 || s.gated) return false;
  if (s.act == PPSCI_ACT_STAN || s.act == PPSCI_ACT_SWISH_B) return false;
  if (l < 2 || l > s.n_layers || wg_layout(J) == LAY_DYN) return false;
  return wg_shape_ok(s.widths[l], s.widths[l - 1]);
}

// dW of layer l: fan-in a multiple of 4, fan-out a multiple of 32 up to 256; the A operand is the activation jets of the
// hidden layer below, or for a dense first layer the caller's matrix
inline bool wg_dw_ok(const ppsci_plan_spec& s, int l, const JetLayout& J) {
  if (s.dtype != PPSCI_F32 || s.gated) return false;
  if (s.act == PPSCI_ACT_STAN || s.act == PPSCI_ACT_SWISH_B) return false;
  if (l < 1 || (l == 1 && !s.dense_in) || l > s.n_layers || wg_layout(J) == LAY_DYN) return false;
  const int K = s.widths[l - 1], N = s.widths[l];
  return K % 4 == 0 && N % 32 == 0 && N >= 32 && N <= 256;
}

#define PPSCI_WG_DW_PICK_(LAY, n)                                                                                \
  ((n) == 256   ? wg::k_wg_dw<LAY, 8>                                                                           \
   : (n) == 224 ? wg::k_wg_dw<LAY, 7>                                                                           \
   : (n) == 192 ? wg::k_wg_dw<LAY, 6>                                                                           \
   : (n) == 160 ? wg::k_wg_dw<LAY, 5>                                                                           \
   : (n) == 128 ? wg::k_wg_dw<LAY, 4>                                                                           \
   : (n) == 96  ? wg::k_wg_dw<LAY, 3>                                                                           \
   : (n) == 64  ? wg::k_wg_dw<LAY, 2>                                                                           \
                : wg::k_wg_dw<LAY, 1>)
#define PPSCI_WG_DW_LAUNCH(lay, n, grid, smem, stream, args, err_expr)                                            \
  do {                                                                                                           \
    void (*kfn_)(decltype(args)) = nullptr;                                                                      \
    switch (lay) {                                                                                               \
      case LAY_22: kfn_ = PPSCI_WG_DW_PICK_(thin::Lay22, n); break;                                              \
      case LAY_12: kfn_ = PPSCI_WG_DW_PICK_(thin::Lay12, n); break;                                              \
      case LAY_222: kfn_ = PPSCI_WG_DW_PICK_(thin::Lay222, n); break;                                            \
      case WG_LAY_4444: kfn_ = PPSCI_WG_DW_PICK_(wg::Lay4444, n); break;                                         \
      default: kfn_ = PPSCI_WG_DW_PICK_(thin::LayV, n);                                                          \
    }                                                                                                            \
    cudaError_t e_ = cudaFuncSetAttribute(kfn_, cudaFuncAttributeMaxDynamicSharedMemorySize, (smem));            \
    if (e_ != cudaSuccess) { err_expr; }                                                                         \
    PPSCI_KLAUNCH(kfn_, (grid), dim3(wg::THREADS), (smem), (stream), 1, args);                                    \
  } while (0)

#define PPSCI_WG_PICK_(DX, LAY, n)                                                                               \
  ((n) == 256   ? wg::k_wg_layer<LAY, 8, DX>                                                                    \
   : (n) == 224 ? wg::k_wg_layer<LAY, 7, DX>                                                                    \
   : (n) == 192 ? wg::k_wg_layer<LAY, 6, DX>                                                                    \
   : (n) == 160 ? wg::k_wg_layer<LAY, 5, DX>                                                                    \
   : (n) == 128 ? wg::k_wg_layer<LAY, 4, DX>                                                                    \
   : (n) == 96  ? wg::k_wg_layer<LAY, 3, DX>                                                                    \
   : (n) == 64  ? wg::k_wg_layer<LAY, 2, DX>                                                                    \
                : wg::k_wg_layer<LAY, 1, DX>)
namespace wg {
using Lay4444 = SLay<4, 4, 4, 4>;
}
#define PPSCI_WG_LAUNCH(DX, lay, n, grid, smem, stream, args, err_expr)                                           \
  do {                                                                                                           \
    void (*kfn_)(decltype(args)) = nullptr;                                                                      \
    switch (lay) {                                                                                               \
      case LAY_22: kfn_ = PPSCI_WG_PICK_(DX, thin::Lay22, n); break;                                             \
      case LAY_12: kfn_ = PPSCI_WG_PICK_(DX, thin::Lay12, n); break;                                             \
      case LAY_222: kfn_ = PPSCI_WG_PICK_(DX, thin::Lay222, n); break;                                           \
      case WG_LAY_4444: kfn_ = PPSCI_WG_PICK_(DX, wg::Lay4444, n); break;                                        \
      default: kfn_ = PPSCI_WG_PICK_(DX, thin::LayV, n);                                                         \
    }                                                                                                            \
    cudaError_t e_ = cudaFuncSetAttribute(kfn_, cudaFuncAttributeMaxDynamicSharedMemorySize, (smem));            \
    if (e_ != cudaSuccess) { err_expr; }                                                                         \
    PPSCI_KLAUNCH(kfn_, (grid), dim3(wg::THREADS), (smem), (stream), 1, args);                                    \
  } while (0)

}  // namespace ppsci
#endif  // PPSCI_EMUL
