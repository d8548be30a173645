// kernels_wgmma.cuh — Hopper (sm_90a) tensor-core kernels for the fp32 layers (K a multiple of 32 up to 1024, N a
// multiple of 32 up to 256) with a jet layout of WgLays (jet_layout.cuh): the forward  Z_l = act_jets(Z_{l-1}) W_l + b_l, the
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
            jet_fwd<float, L>(g.J, sc, [&](int c) { return comp(z[c]); }, [&](int c, float v) { yout[c][t] = valid ? v : 0.f; });
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
          ob[0][t] = jet_adj<float, L>(g.J, sc, [&](int c) { return comp(zc[c]); }, [&](int c) { return comp(xc[c]); },
                                       [&](int c, float v) { ob[c][t] = v; });
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

// ---- weight gradient  dW_l[k][n] += sum over jet rows  a_{l-1}[row][k] Zbar_l[row][n],  db_l[n] += sum_p Zbar_l[0][p][n] ----
// The contraction runs over jet rows, in any order both operands share.  K index 4 j + u is point 4 q + u of channel c,
// j = c + C q (point quads, channels within a quad), so every aligned group of 4 K elements is 4 consecutive points of
// one channel and no jet row is left unused, for any C.  A chunk is dw_pch(C) points = dw_groups(C) groups, issued as dw_ksteps(C) K steps
// of 8 (an odd group count is padded with one zero group).
//
// A = act_jets(Z_{l-1})^T comes from registers: the tf32 A fragment gives lane t = lane % 4 of warp w the K elements
// 8 s + t and 8 s + t + 4 of rows 16 w + lane / 4 (+ 8), i.e. only points = t (mod 4).  Each thread computes the jets of
// its own (point, fan-in row) pairs once per CTA and splits them hi / lo in registers.
// B = Zbar_l^T is staged per chunk, K-major with the 128-byte swizzle: thread <-> output column, 32 lanes read 128
// contiguous bytes of one row, and each (column, group) is one float4 of hi and one of lo at sw128_q(column, group), so
// eight consecutive columns land in eight distinct 16-byte bank groups.
//
// CTA (fan-in block of 128 rows, column block of BN <= 128 columns, range of chunks): warpgroup i owns fan-in rows
// 64 i .. 64 i + 63 and issues  A_hi B_hi -> exact accumulator,  A_lo B_hi + A_hi B_lo -> cross accumulator  per K step
// (the 3xTF32 scheme of k_wg_layer, with the exact-product term in an accumulator of its own).  While the MMAs of chunk j
// run, the Zbar_l values of chunk j + 1 are loaded into registers and written to the other B stage, and its Z_{l-1}
// values are copied into per-thread shared-memory slots by cp.async (they would not fit in registers beside the two
// accumulators and the in-flight A fragments); the jets are computed once those MMAs have retired.  Every dw_flush(C)
// chunks each thread adds its accumulators to partial sums of its own in shared memory (fp32, round to nearest) and
// restarts them at zero.  The CTA adds partial sums and accumulators to dW_l once, with atomicAdd; the CTAs of fan-in
// block 0 also add their columns' channel-0 sums (summed in shared memory) to db_l.
//
// Why the periodic flush: the tensor cores do not round each accumulation to nearest, so the error of a wgmma
// accumulator grows linearly with the number of K steps added into it, not like a random walk.  Accumulated over a
// whole split (up to ~10^5 jet rows at 70,001 points), dW_l was off by up to ~8,000 units of 2^-24 sum |A| |Zbar|
// against ~50 for the CUDA-core kernel (measured on an H100 80GB HBM3, 700 W power limit; tests/test_gpu_tc_layers.py).
// Restarting the accumulators every ~512 jet rows bounds that error independently of the point count.
__host__ __device__ constexpr int dw_pch(int C) { return C >= 8 ? 4 : C >= 3 ? 8 : 32 / C; }  // points per chunk
__host__ __device__ constexpr int dw_groups(int C) { return dw_pch(C) / 4 * C; }
__host__ __device__ constexpr int dw_ksteps(int C) { return (dw_groups(C) + 1) / 2; }
__host__ __device__ constexpr int dw_atoms(int C) { return (dw_ksteps(C) + 3) / 4; }  // 32-wide K atoms per B stage
// widest column block in units of 32: two accumulators of BN / 2 registers each, beside the A fragments and the B
// prefetch of a chunk, must fit in 255 registers without spilling
__host__ __device__ constexpr int dw_maxq(int C) { return C <= 5 ? 4 : C <= 8 ? 2 : 1; }
// two stages of [hi | lo][atoms][BN rows x 128 bytes], 1024-byte aligned, then the db_l column sums, the A operand's
// per-thread Z_{l-1} slots and the per-thread partial sums of the flushed accumulators (BN / 2 per thread)
__host__ __device__ constexpr int dw_smem_bytes(int C, int bnq) {
  return 2 * 2 * dw_atoms(C) * bnq * 32 * 128 + bnq * 32 * 4 + dw_pch(C) / 4 * 2 * C * 256 * 4 + bnq * 32 * 2 * 256 + 1024;
}
constexpr int DW_TK = 128;  // fan-in rows per CTA
constexpr int DW_FLUSH_ROWS = 512;  // jet rows accumulated by the tensor cores between two flushes to dW_l
__host__ __device__ constexpr int dw_flush(int C) {  // chunks per flush
  return DW_FLUSH_ROWS / (dw_pch(C) * C) > 1 ? DW_FLUSH_ROWS / (dw_pch(C) * C) : 1;
}

struct WgDwArgs {
  AOperand<float> A;   // A_ACT over Z_{l-1}
  JetLayout J;
  const float* Zbar;   // [C][Np][ldzb]
  int ldzb;
  long long zbplane;
  int Kdim;            // fan-in (rows of dW)
  int Nout;            // fan-out (columns of dW)
  int col_blocks;      // column blocks per fan-in block (blockIdx.x = fan-in block * col_blocks + column block)
  float* dW;           // [Kdim][Nout]
  float* db;           // [Nout]
  long long Np;
  int chunks_per_split;
};

// D[64 x 64] += A[64 x 8] B[8 x 64], A tf32 fragments in registers, B from shared memory
__device__ __forceinline__ void wgmma_tf32_rA_m64n64(float (&d)[32], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1u));
}
// D[64 x 32] += A[64 x 8] B[8 x 32]
__device__ __forceinline__ void wgmma_tf32_rA_m64n32(float (&d)[16], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1u));
}

template <class L, int BNQ>
__global__ void __launch_bounds__(THREADS, 1) k_wg_dw(WgDwArgs g) {
  PPSCI_DYN_SMEM(smem_dyn);
  const uint32_t base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  unsigned char* base_ptr = smem_dyn + (base - smem_u32(smem_dyn));
  constexpr int CS = L::CS, PCH = dw_pch(CS), QPC = PCH / 4, G = dw_groups(CS), KS = dw_ksteps(CS), NA = dw_atoms(CS);
  constexpr int BN = BNQ * 32, NB = BNQ / 2, TAIL = BNQ & 1;
  constexpr int ATOM = BN * 128;                            // bytes of one K atom of B (hi or lo)
  constexpr int STAGE = 2 * NA * ATOM;
  constexpr int BI = (G * BN + THREADS - 1) / THREADS;     // B items (group, column) per thread and chunk
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = tid >> 7, t = lane & 3;
  const int kb = blockIdx.x / g.col_blocks, n0 = (blockIdx.x - kb * g.col_blocks) * BN;
  const int Np = (int)g.Np;  // points per call < 2^31 (the workspace chunk)
  const int total_chunks = (Np + PCH - 1) / PCH;
  const int ch_begin = blockIdx.y * g.chunks_per_split;
  const int ch_end = ch_begin + g.chunks_per_split < total_chunks ? ch_begin + g.chunks_per_split : total_chunks;
  if (ch_begin >= ch_end) return;
  const int act = g.A.act;
  const int krow = kb * DW_TK + wgi * 64 + (warp & 3) * 16 + (lane >> 2);  // A fragment rows krow, krow + 8

  float* bsum = reinterpret_cast<float*>(base_ptr + 2 * STAGE);  // [BN] channel-0 column sums (fan-in block 0)
  for (int i = tid; i < (2 * STAGE + BN * 4) / 16; i += THREADS)  // the pad group and the K atoms past the last group stay zero
    reinterpret_cast<float4*>(base_ptr)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();  // ... before the first chunk's B writes

  float ex[NB > 0 ? NB : 1][32], ext[TAIL ? 16 : 1], cr[NB > 0 ? NB : 1][32], crt[TAIL ? 16 : 1];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb)
#pragma unroll
    for (int i = 0; i < 32; ++i) ex[nb][i] = cr[nb][i] = 0.f;
#pragma unroll
  for (int i = 0; i < (TAIL ? 16 : 1); ++i) ext[i] = crt[i] = 0.f;

  // element e of this thread's accumulator fragments (exact + cross term): e = 4 j + 2 h + b is row krow + 8 h, column
  // 8 j + 2 t + b of the n8 block j
  auto acc_at = [&](int e) -> float {
    return e < 32 * NB ? ex[e >> 5][e & 31] + cr[e >> 5][e & 31] : ext[e - 32 * NB] + crt[e - 32 * NB];
  };
  // partial sums of the flushed accumulators: float4 q of this thread (elements 4 q .. 4 q + 3) at part[q THREADS + tid]
  float4* part = reinterpret_cast<float4*>(base_ptr + 2 * STAGE + BN * 4 + QPC * 2 * CS * THREADS * 4);
#pragma unroll
  for (int q = 0; q < BN / 8; ++q) part[q * THREADS + tid] = make_float4(0.f, 0.f, 0.f, 0.f);
  auto flush = [&]() {
#pragma unroll
    for (int q = 0; q < BN / 8; ++q) {
      float4 p = part[q * THREADS + tid];
      p.x += acc_at(4 * q); p.y += acc_at(4 * q + 1); p.z += acc_at(4 * q + 2); p.w += acc_at(4 * q + 3);
      part[q * THREADS + tid] = p;
    }
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int i = 0; i < 32; ++i) ex[nb][i] = cr[nb][i] = 0.f;
#pragma unroll
    for (int i = 0; i < (TAIL ? 16 : 1); ++i) ext[i] = crt[i] = 0.f;
  };

  // Z_{l-1} at point 4 qq + t of the chunk, fan-in row krow + 8 h, channel c: thread-private slots, filled by cp.async
  // (zero past Np and Kdim) while the previous chunk's MMAs run
  float* za = reinterpret_cast<float*>(base_ptr + 2 * STAGE + BN * 4);
  auto za_at = [&](int qq, int h, int c) -> float* { return za + ((qq * 2 + h) * CS + c) * THREADS + tid; };
  float4 zb[BI];         // Zbar_l at the 4 points of group gi, column n0 + n, for item tid + THREADS i = gi BN + n
  auto load_a = [&](int ch) {
    const int p0 = ch * PCH;
#pragma unroll
    for (int qq = 0; qq < QPC; ++qq)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int p = p0 + 4 * qq + t;
        const int k = krow + 8 * h;
        const bool ok = p < Np && k < g.Kdim;
        const float* src = g.A.Z + (ok ? (long long)p * g.A.ld + k : 0);
#pragma unroll
        for (int c = 0; c < CS; ++c)
          asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(za_at(qq, h, c))),
                       "l"(src + (ok ? (long long)c * g.A.plane : 0)), "r"(ok ? 4 : 0)
                       : "memory");
      }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  auto load_b = [&](int ch) {
    const int p0 = ch * PCH;
#pragma unroll
    for (int i = 0; i < BI; ++i) {
      const int item = tid + THREADS * i;
      const int gi = item / BN, n = item - gi * BN;
      const int qq = gi / CS, c = gi - qq * CS;
      const int p = p0 + 4 * qq;
      const bool ok = item < G * BN && n0 + n < g.Nout;
      const float* src = g.Zbar + (long long)c * g.zbplane + (long long)p * g.ldzb + n0 + n;
      zb[i].x = ok && p < Np ? __ldg(src) : 0.f;
      zb[i].y = ok && p + 1 < Np ? __ldg(src + g.ldzb) : 0.f;
      zb[i].z = ok && p + 2 < Np ? __ldg(src + 2 * g.ldzb) : 0.f;
      zb[i].w = ok && p + 3 < Np ? __ldg(src + 3 * g.ldzb) : 0.f;
    }
  };

  load_a(ch_begin);
  load_b(ch_begin);
  uint32_t ahi[KS][4], alo[KS][4];
  for (int ch = ch_begin; ch < ch_end; ++ch) {
    const int sidx = (ch - ch_begin) & 1;
    const uint32_t st_addr = base + sidx * STAGE;
    unsigned char* st = base_ptr + sidx * STAGE;
    // B of this chunk -> stage sidx; its last reader, chunk ch - 2, retired before the previous chunk's barrier
#pragma unroll
    for (int i = 0; i < BI; ++i) {
      const int item = tid + THREADS * i;
      if (item >= G * BN) continue;
      const int gi = item / BN, n = item - gi * BN;
      const float4 v = zb[i];
      float4 hi, lo;
      hi.x = tf32_rn(v.x); hi.y = tf32_rn(v.y); hi.z = tf32_rn(v.z); hi.w = tf32_rn(v.w);
      lo.x = v.x - hi.x; lo.y = v.y - hi.y; lo.z = v.z - hi.z; lo.w = v.w - hi.w;
      const uint32_t off = (gi >> 3) * ATOM + sw128_q(n, gi & 7);
      *reinterpret_cast<float4*>(st + off) = hi;
      *reinterpret_cast<float4*>(st + NA * ATOM + off) = lo;
      if (kb == 0 && gi % CS == 0) atomicAdd(bsum + n, (v.x + v.y) + (v.z + v.w));
    }
    wgmma_wait<0>();  // the MMAs of chunk ch - 1 have retired: the fragment registers are free
    if (ch > ch_begin && (ch - ch_begin) % dw_flush(CS) == 0) flush();
    // activation jets of this thread's A elements (points past Np give finite jets of 0 against zero B values)
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    float av[QPC][2][CS];
#pragma unroll
    for (int qq = 0; qq < QPC; ++qq)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float z[CS], sc[6];
#pragma unroll
        for (int c = 0; c < CS; ++c) z[c] = *za_at(qq, h, c);
        act_coef<float, L::KM>(act, z[0], av[qq][h][0], sc);
        jet_fwd<float, L>(g.J, sc, [&](int c) { return z[c]; }, [&](int c, float v) { av[qq][h][c] = v; });
      }
    if (ch + 1 < ch_end) load_a(ch + 1);
    fence_proxy_async();
    __syncthreads();  // this chunk's B stage is complete
    // K step s: a0 / a1 = group 2 s (rows krow / krow + 8), a2 / a3 = group 2 s + 1; group gi = channel gi % C of quad
    // gi / C
#pragma unroll
    for (int s = 0; s < KS; ++s)
#pragma unroll
      for (int e = 0; e < 2; ++e)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int gi = 2 * s + e;
          const float v = gi < G ? av[gi / CS][h][gi % CS] : 0.f;
          const float vh = tf32_rn(v);
          ahi[s][2 * e + h] = __float_as_uint(vh);
          alo[s][2 * e + h] = __float_as_uint(v - vh);
        }
    wgmma_fence();
#pragma unroll
    for (int s = 0; s < KS; ++s) {
      const uint64_t b_hi = make_desc(st_addr + (s >> 2) * ATOM + (s & 3) * 32);
      const uint64_t b_lo = b_hi + (uint64_t)(NA * ATOM / 16);
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) {
        const uint64_t bo = (uint64_t)(nb * 64 * 128 / 16);  // column block nb = B rows 64 nb ..
        wgmma_tf32_rA_m64n64(ex[nb], ahi[s], b_hi + bo);
        wgmma_tf32_rA_m64n64(cr[nb], alo[s], b_hi + bo);
        wgmma_tf32_rA_m64n64(cr[nb], ahi[s], b_lo + bo);
      }
      if constexpr (TAIL) {
        const uint64_t bo = (uint64_t)(NB * 64 * 128 / 16);  // the last 32 columns
        wgmma_tf32_rA_m64n32(ext, ahi[s], b_hi + bo);
        wgmma_tf32_rA_m64n32(crt, alo[s], b_hi + bo);
        wgmma_tf32_rA_m64n32(crt, ahi[s], b_lo + bo);
      }
    }
    wgmma_commit();
    if (ch + 1 < ch_end) load_b(ch + 1);
  }
  wgmma_wait<0>();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int k = krow + 8 * h;
    if (k >= g.Kdim) continue;
    float* row = g.dW + (long long)k * g.Nout + n0;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      if (n0 + 8 * j >= g.Nout) break;
      const int col = 8 * j + 2 * t;
      const float4 p = part[j * THREADS + tid];
      atomicAdd(row + col, (h ? p.z : p.x) + acc_at(4 * j + 2 * h));
      atomicAdd(row + col + 1, (h ? p.w : p.y) + acc_at(4 * j + 2 * h + 1));
    }
  }
  if (kb == 0) {
    __syncthreads();
    if (tid < BN && n0 + tid < g.Nout) atomicAdd(g.db + n0 + tid, bsum[tid]);
  }
}

}  // namespace wg

// a GEMM of contraction length K and N output columns on k_wg_layer
inline int wg_kpad(int K) { return (K + wg::KCH - 1) / wg::KCH * wg::KCH; }
inline bool wg_shape_ok(int K, int N) { return K % wg::KCH == 0 && K >= 32 && K <= 1024 && N % 32 == 0 && N >= 32 && N <= 256; }
// the plans whose layers may run on the wgmma kernels: fp32, not gated, an activation without a trainable parameter and
// a jet layout of WgLays; which passes of which layers do is up to wg_fwd_ok / wg_dx_ok / wg_dw_ok
inline bool wg_plan_ok(const ppsci_plan_spec& s, const JetLayout& J) {
  return s.dtype == PPSCI_F32 && !s.gated && !act_has_param(s.act) && with_lay(WgLays{}, J, [](auto) {});
}
// forward of layer l on k_wg_layer; layer 1 only as a dense first layer (its operand the caller's matrix, contraction
// padded to 32)
inline bool wg_fwd_ok(const ppsci_plan_spec& s, int l) {
  if (l == 1) return s.dense_in && s.n_layers >= 2 && s.widths[0] % 4 == 0 && wg_shape_ok(wg_kpad(s.widths[0]), s.widths[1]);
  if (l < 2 || l > s.n_layers) return false;  // l == n_layers: a wide output layer
  return wg_shape_ok(s.widths[l - 1], s.widths[l]);
}
// dx through layer l (produces Zbar_{l-1} of hidden layer l - 1): gemm K = width of layer l, gemm N = width of layer l - 1
inline bool wg_dx_ok(const ppsci_plan_spec& s, int l) {
  if (l < 2 || l > s.n_layers) return false;
  return wg_shape_ok(s.widths[l], s.widths[l - 1]);
}

// dW of layer l: fan-in a multiple of 4, fan-out a multiple of 32 up to 256; the A operand is the activation jets of the
// hidden layer below, or for a dense first layer the caller's matrix
inline bool wg_dw_ok(const ppsci_plan_spec& s, int l) {
  if (l < 1 || (l == 1 && !s.dense_in) || l > s.n_layers) return false;
  const int K = s.widths[l - 1], N = s.widths[l];
  return K % 4 == 0 && N % 32 == 0 && N >= 32 && N <= 256;
}

}  // namespace ppsci
#endif  // PPSCI_EMUL
