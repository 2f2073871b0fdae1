// simt_shim.h -- TEST INFRASTRUCTURE: just enough of the CUDA vocabulary to compile ONE
// warp-sized kernel for the host and run it as 32 OS threads, one per lane.
//
// The model is the one CUDA itself gives since independent thread scheduling: lanes run
// freely and only meet where the kernel says so (__syncwarp, __ballot_sync, __shfl_sync).
// Those become pthread barriers here, `__shared__` variables become function-local statics
// (one copy for the single CTA), dynamic shared memory is simt::dynamic_smem (FMB_SIMT_HOST),
// shared-memory atomics become __atomic builtins.  Everything else -- the arithmetic, the
// indexing, the order of memory operations -- is the kernel's own source.
// Because the barriers are real synchronisation, ThreadSanitizer can check that every
// cross-lane hand-off through "shared" or "global" memory is ordered by one.
#pragma once
#include <cuda_runtime.h>  // vector types, and the annotation macros we are about to replace

#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <string.h>

#define FMB_SIMT_HOST 1

#undef __global__
#undef __device__
#undef __host__
#undef __shared__
#undef __forceinline__
#undef __launch_bounds__
#undef __align__
#define __global__
#define __device__
#define __host__
#define __shared__ static
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))

namespace simt {

constexpr int kLanes = 32;
struct Dim {
  unsigned x;
};
extern thread_local Dim tid;
extern pthread_barrier_t warp_barrier;
extern unsigned ballot_in[kLanes];
extern uint64_t shfl_in[kLanes];
extern double dynamic_smem[];  // the kernel's `extern __shared__` memory

inline void sync() { pthread_barrier_wait(&warp_barrier); }

}  // namespace simt

#define threadIdx (simt::tid)

#ifdef SIMT_NO_SYNCWARP  // negative control: the harness must notice when the kernel's barriers are gone
inline void __syncwarp(unsigned = 0xffffffffu) {}
#else
inline void __syncwarp(unsigned = 0xffffffffu) { simt::sync(); }
#endif

inline unsigned __ballot_sync(unsigned, bool pred) {
  __atomic_store_n(&simt::ballot_in[simt::tid.x], pred ? 1u : 0u, __ATOMIC_RELAXED);
  simt::sync();
  unsigned m = 0;
  for (int l = 0; l < simt::kLanes; l++)
    if (__atomic_load_n(&simt::ballot_in[l], __ATOMIC_RELAXED)) m |= 1u << l;
  simt::sync();  // nobody overwrites its slot for the next ballot before all have read
  return m;
}

template <class T>
inline T __shfl_sync(unsigned, T v, int src) {
  static_assert(sizeof(T) <= sizeof(uint64_t), "one word per lane");
  uint64_t bits = 0;
  memcpy(&bits, &v, sizeof(T));
  __atomic_store_n(&simt::shfl_in[simt::tid.x], bits, __ATOMIC_RELAXED);
  simt::sync();
  bits = __atomic_load_n(&simt::shfl_in[src & (simt::kLanes - 1)], __ATOMIC_RELAXED);
  simt::sync();  // nobody overwrites its slot for the next exchange before all have read
  memcpy(&v, &bits, sizeof(T));
  return v;
}

inline int __ffs(unsigned v) { return __builtin_ffs((int)v); }

inline unsigned atomicMax(unsigned* addr, unsigned val) {
  unsigned old = __atomic_load_n(addr, __ATOMIC_RELAXED);
  while (old < val && !__atomic_compare_exchange_n(addr, &old, val, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {
  }
  return old;
}
