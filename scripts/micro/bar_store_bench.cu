// Microbenchmark: what does a block barrier cost when global stores (or cp.async fetches) issued by
// the CTA are still in flight?  The ORDERED epoch kernel (one CTA, a few warps, a barrier every few
// hundred cycles) showed half of its stall samples on barriers; this isolates the cause.
//   one CTA of `threads`; per iteration: `nst` 16-byte global stores per thread to scattered rows, then a
//   barrier; cycles per iteration by clock64.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o bar_store_bench bar_store_bench.cu
#include <cstdio>
#include <cuda_runtime.h>
#include <stdint.h>

__device__ __forceinline__ uint32_t hash(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x;
}

// MODE 0: __syncthreads; 1: bar.sync 1 (named); 2: no barrier (store issue cost alone);
// 3: stores then __threadfence_block then __syncthreads; 4: st.global.cg; 5: loads (ld.cg) instead of stores
template <int MODE>
__global__ void k(double2* tab, uint32_t rows, int nst, int iters, long long* out, double* sink) {
  const int tid = threadIdx.x;
  double acc = 0;
  long long t0 = clock64();
  for (int i = 0; i < iters; i++) {
    for (int s = 0; s < nst; s++) {
      const uint32_t r = hash(tid * 7919u + i * 104729u + s * 31u) % rows;
      if (MODE == 5) {
        double2 v = __ldcg(tab + (size_t)r * 5 + (s % 5));
        acc += v.x;
      } else if (MODE == 4) {
        __stcg(tab + (size_t)r * 5 + (s % 5), make_double2(1.0, 2.0));
      } else {
        tab[(size_t)r * 5 + (s % 5)] = make_double2(1.0, 2.0);
      }
    }
    if (MODE == 3) __threadfence_block();
    if (MODE == 0 || MODE == 3 || MODE == 4 || MODE == 5) __syncthreads();
    if (MODE == 1) asm volatile("bar.sync 1, %0;" ::"r"((int)blockDim.x) : "memory");
  }
  long long t1 = clock64();
  if (tid == 0) out[0] = t1 - t0;
  if (acc == 1.2345) *sink = acc;
}

template <int MODE>
void run(const char* name, double2* tab, int threads, int nst) {
  long long* out;
  double* sink;
  cudaMalloc(&out, 8);
  cudaMalloc(&sink, 8);
  const int iters = 2000;
  k<MODE><<<1, threads>>>(tab, 9746, nst, iters, out, sink);
  k<MODE><<<1, threads>>>(tab, 9746, nst, iters, out, sink);
  cudaDeviceSynchronize();
  long long h;
  cudaMemcpy(&h, out, 8, cudaMemcpyDeviceToHost);
  printf("%-46s threads=%4d stores/thread=%2d : %8.1f cycles/iteration\n", name, threads, nst, (double)h / iters);
  cudaFree(out);
  cudaFree(sink);
}

int main() {
  double2* tab;
  cudaMalloc(&tab, 9746 * 5 * sizeof(double2));
  for (int threads : {128, 512}) {
    for (int nst : {0, 1, 4, 10}) {
      run<0>("stores + __syncthreads", tab, threads, nst);
      run<1>("stores + named barrier", tab, threads, nst);
      run<2>("stores, no barrier", tab, threads, nst);
      run<3>("stores + fence.cta + __syncthreads", tab, threads, nst);
      run<4>("st.cg + __syncthreads", tab, threads, nst);
      run<5>("ld.cg (consumed) + __syncthreads", tab, threads, nst);
    }
  }
  return 0;
}
