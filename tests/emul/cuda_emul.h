// cuda_emul.h — TEST INFRASTRUCTURE ONLY.
//
// A CPU shim that lets the kernel sources (paddlescience_b200/csrc/*.cuh, *.cu) be compiled with g++ (-DPPSCI_EMUL)
// and executed with one OS thread per CUDA thread.  Blocks run one at a time; the CTAs of a thread-block cluster run
// concurrently.  It exists so that indexing / tiling / barrier-protocol / descriptor logic can be checked against the
// oracle on a box without a GPU.  It is never linked into the product library and the package never loads it
// (tests/emul/build_emul.py builds tests/emul/_build/libppsci_b200_emul.so, loaded only by tests/).
#pragma once
#ifndef PPSCI_EMUL
#error "cuda_emul.h is only for -DPPSCI_EMUL builds"
#endif

#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <functional>
#include <map>
#include <mutex>
#include <thread>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __cluster_dims__(...)
#define __restrict__
#define __shared__ static  // non-cluster kernels: one block runs at a time, so a function-static IS block-shared
#define __align__(n) __attribute__((aligned(n)))

struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};

namespace emul {

constexpr uint32_t SMEM_BASE = 1024;  // shared-window address of arena offset 0 (non-zero, 1024-aligned)

// reusable counting barrier (generation based)
struct Barrier {
  std::mutex m;
  std::condition_variable cv;
  unsigned count = 0, waiting = 0;
  unsigned long gen = 0;
  void init(unsigned n) { count = n; waiting = 0; }
  void wait() {
    std::unique_lock<std::mutex> lk(m);
    const unsigned long g = gen;
    if (++waiting == count) {
      waiting = 0;
      ++gen;
      cv.notify_all();
    } else {
      cv.wait(lk, [&] { return gen != g; });
    }
  }
  // barrier among `n` threads where n is only known at the call (bar.sync id, n)
  void wait_n(unsigned n) {
    std::unique_lock<std::mutex> lk(m);
    const unsigned long g = gen;
    if (++waiting == n) {
      waiting = 0;
      ++gen;
      cv.notify_all();
    } else {
      cv.wait(lk, [&] { return gen != g; });
    }
  }
};

struct Cluster;
struct Cta {
  std::vector<unsigned char> smem_store;
  unsigned char* smem = nullptr;  // 1024-aligned arena
  size_t smem_bytes = 0;
  Barrier sync_all;
  Barrier warp_bar[64];
  double warp_scratch[64][32];
  dim3 block_idx;
  unsigned rank = 0;
  Cluster* cluster = nullptr;
};
struct Cluster {
  std::vector<Cta> ctas;
  Barrier sync;  // barrier.cluster
};

inline thread_local dim3 t_threadIdx, t_blockIdx;
inline thread_local Cta* t_cta = nullptr;
inline dim3 g_blockDim, g_gridDim;

inline unsigned linear_tid() {
  return t_threadIdx.x + g_blockDim.x * (t_threadIdx.y + g_blockDim.y * t_threadIdx.z);
}
[[noreturn]] inline void die(const char* msg) {
  fprintf(stderr, "[cuda_emul] FATAL: %s (block %u, thread %u)\n", msg, t_blockIdx.x, linear_tid());
  fflush(stderr);
  abort();
}

}  // namespace emul

#define threadIdx (emul::t_threadIdx)
#define blockIdx (emul::t_blockIdx)
#define blockDim (emul::g_blockDim)
#define gridDim (emul::g_gridDim)

inline void __syncthreads() { emul::t_cta->sync_all.wait(); }
inline void __syncwarp(unsigned = 0xffffffffu) {
  const unsigned t = emul::linear_tid();
  emul::t_cta->warp_bar[t >> 5].wait();
}
inline void __trap() { emul::die("__trap()"); }
inline long long clock64() { return 0; }
template <typename T>
inline T __ldg(const T* p) { return *p; }
inline float __uint_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
inline uint32_t __float_as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

// warp shuffles: lanes of a warp rendezvous on a per-warp barrier and exchange through scratch
template <typename T>
inline T __shfl_xor_sync(unsigned, T v, int lane_mask) {
  const unsigned t = emul::linear_tid();
  const unsigned w = t >> 5, l = t & 31;
  emul::t_cta->warp_scratch[w][l] = (double)v;
  emul::t_cta->warp_bar[w].wait();
  const T r = (T)emul::t_cta->warp_scratch[w][l ^ (unsigned)lane_mask];
  emul::t_cta->warp_bar[w].wait();
  return r;
}

inline float atomicAdd(float* addr, float v) {
  uint32_t* ia = reinterpret_cast<uint32_t*>(addr);
  uint32_t old = __atomic_load_n(ia, __ATOMIC_RELAXED);
  for (;;) {
    float f;
    memcpy(&f, &old, 4);
    float nf = f + v;
    uint32_t ni;
    memcpy(&ni, &nf, 4);
    if (__atomic_compare_exchange_n(ia, &old, ni, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) return f;
  }
}
inline unsigned atomicMax(unsigned* addr, unsigned v) {
  unsigned old = __atomic_load_n(addr, __ATOMIC_RELAXED);
  while (old < v && !__atomic_compare_exchange_n(addr, &old, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
  return old;
}
inline unsigned long long atomicMax(unsigned long long* addr, unsigned long long v) {
  unsigned long long old = __atomic_load_n(addr, __ATOMIC_RELAXED);
  while (old < v && !__atomic_compare_exchange_n(addr, &old, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
  return old;
}
inline double atomicAdd(double* addr, double v) {
  uint64_t* ia = reinterpret_cast<uint64_t*>(addr);
  uint64_t old = __atomic_load_n(ia, __ATOMIC_RELAXED);
  for (;;) {
    double f;
    memcpy(&f, &old, 8);
    double nf = f + v;
    uint64_t ni;
    memcpy(&ni, &nf, 8);
    if (__atomic_compare_exchange_n(ia, &old, ni, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) return f;
  }
}

// ---- runtime API stubs -------------------------------------------------------------------
typedef int cudaError_t;
typedef void* cudaStream_t;
enum { cudaSuccess = 0 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
inline const char* cudaGetErrorString(cudaError_t) { return "emul"; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaPeekAtLastError() { return cudaSuccess; }
inline cudaError_t cudaMalloc(void** p, size_t n) { *p = malloc(n ? n : 1); return cudaSuccess; }
inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { memset(d, v, n); return cudaSuccess; }
template <typename F>
inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
struct cudaDeviceProp { int multiProcessorCount; int major; int minor; };
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) { p->multiProcessorCount = 4; p->major = 9; p->minor = 0; return cudaSuccess; }

typedef void* cudaEvent_t;
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = nullptr; return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* t, cudaEvent_t, cudaEvent_t) { *t = 0.f; return cudaSuccess; }

namespace emul {
// Run `body` once per (block, thread).  Clusters (groups of `cluster_x` consecutive blocks along x) run one after
// the other; the threads of a cluster's CTAs are real OS threads, so __syncthreads semantics are honest.
inline void launch(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()>& body, unsigned cluster_x = 1) {
  g_blockDim = block;
  g_gridDim = grid;
  const unsigned nthr = block.x * block.y * block.z;
  if (grid.x % cluster_x != 0) { fprintf(stderr, "[cuda_emul] grid.x not a multiple of the cluster size\n"); abort(); }
  for (unsigned bz = 0; bz < grid.z; ++bz)
    for (unsigned by = 0; by < grid.y; ++by)
      for (unsigned bx0 = 0; bx0 < grid.x; bx0 += cluster_x) {
        Cluster cl;
        cl.ctas = std::vector<Cta>(cluster_x);
        cl.sync.init(nthr * cluster_x);
        for (unsigned r = 0; r < cluster_x; ++r) {
          Cta& c = cl.ctas[r];
          c.smem_store.assign(smem_bytes + 2048, 0xCD);
          c.smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(c.smem_store.data()) + 1023) & ~uintptr_t(1023));
          c.smem_bytes = smem_bytes;
          c.sync_all.init(nthr);
          for (unsigned w = 0; w < (nthr + 31) / 32 && w < 64; ++w) c.warp_bar[w].init(std::min(32u, nthr - 32 * w));
          c.block_idx = dim3(bx0 + r, by, bz);
          c.rank = r;
          c.cluster = &cl;
        }
        std::vector<std::thread> th;
        th.reserve(nthr * cluster_x);
        for (unsigned r = 0; r < cluster_x; ++r)
          for (unsigned t = 0; t < nthr; ++t) {
            th.emplace_back([=, &body, &cl]() {
              t_cta = &cl.ctas[r];
              t_blockIdx = cl.ctas[r].block_idx;
              t_threadIdx = dim3(t % block.x, (t / block.x) % block.y, t / (block.x * block.y));
              body();
            });
          }
        for (auto& x : th) x.join();
      }
}
inline unsigned char* dyn_smem() { return t_cta->smem; }
}  // namespace emul

#define PPSCI_DYN_SMEM(name) unsigned char* name = emul::dyn_smem()
#define PPSCI_LAUNCH(kernel, grid, block, smem, stream, ...) \
  emul::launch((grid), (block), (smem), [&]() { kernel(__VA_ARGS__); })

struct __attribute__((aligned(16))) float4 { float x, y, z, w; };
struct __attribute__((aligned(16))) double2 { double x, y; };
struct __attribute__((aligned(16))) uint4 { uint32_t x, y, z, w; };
struct __attribute__((aligned(8))) float2 { float x, y; };
struct __attribute__((aligned(8))) uint2 { uint32_t x, y; };
inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
inline float2 make_float2(float x, float y) { return float2{x, y}; }
inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }
inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
