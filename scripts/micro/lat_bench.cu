// Latency microbenchmark for the ordered (sequentially-consistent) epoch kernel design:
// dependent-chain latencies of the operations its per-run critical path is made of.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o lat_bench lat_bench.cu
#include <cstdio>
#include <cuda_runtime.h>
#include <stdint.h>

__device__ __forceinline__ long long clk() {
  long long t;
  asm volatile("mov.u64 %0, %%clock64;" : "=l"(t)::"memory");
  return t;
}

template <int OP>
__global__ void chain(double* out, long long* cyc, int iters, double a, double b, const double* g, double* sm_src) {
  __shared__ double s[1024];
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) s[i] = (double)((i * 17 + 1) & 1023);
  __syncthreads();
  double x = a + threadIdx.x;
  float xf = (float)x;
  uint32_t idx = threadIdx.x & 1023;
  uint64_t gi = threadIdx.x;
  long long t0 = clk();
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int u = 0; u < 8; u++) {
      if (OP == 0) x = x + b;                       // DADD
      if (OP == 1) x = fma(x, b, a);                // DFMA
      if (OP == 2) x = x * b;                       // DMUL
      if (OP == 3) xf = fmaf(xf, (float)b, (float)a);  // FFMA
      if (OP == 4) x = __shfl_xor_sync(0xffffffffu, x, 1);  // 2x SHFL (fp64)
      if (OP == 5) xf = __shfl_xor_sync(0xffffffffu, xf, 1);
      if (OP == 6) { idx = (uint32_t)s[idx]; }      // LDS.64 pointer chase (+F2I)
      if (OP == 7) { __syncthreads(); }
      if (OP == 8) x = fmin(fmax(x, a), b);         // clamp
      if (OP == 9) x = exp(-x * 1e-9);              // fp64 exp
      if (OP == 10) { gi = (uint64_t)__ldcg(g + (gi & 0xfffff)); }  // L2 pointer chase
      if (OP == 11) { x = (x < a) ? b : x + 1.0; }  // DSETP + select + DADD
      if (OP == 12) { x = 1.0 / (1.0 + x); }        // fp64 div
      if (OP == 13) { gi = (uint64_t)(*(volatile const double*)(g + (gi & 0xfff))); }  // L1 chase
    }
  }
  long long t1 = clk();
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
  out[blockIdx.x * blockDim.x + threadIdx.x] = x + xf + idx + gi;
}

template <int OP>
void run(const char* name, int threads, double* out, long long* cyc, const double* g) {
  const int iters = 512;
  chain<OP><<<1, threads>>>(out, cyc, iters, 1.0000001, 0.9999999, g, nullptr);
  chain<OP><<<1, threads>>>(out, cyc, iters, 1.0000001, 0.9999999, g, nullptr);
  cudaDeviceSynchronize();
  long long h;
  cudaMemcpy(&h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
  printf("%-28s threads=%4d  %.1f cycles/op\n", name, threads, (double)h / (iters * 8));
}

int main() {
  double* out;
  long long* cyc;
  double* g;
  cudaMalloc(&out, 1024 * sizeof(double));
  cudaMalloc(&cyc, 8 * sizeof(long long));
  const size_t gn = 1 << 20;
  cudaMalloc(&g, gn * sizeof(double));
  double* hg = (double*)malloc(gn * sizeof(double));
  for (size_t i = 0; i < gn; i++) hg[i] = (double)((i * 1103515245ull + 12345ull) % gn);
  cudaMemcpy(g, hg, gn * sizeof(double), cudaMemcpyHostToDevice);
  for (int th : {32, 512}) {
    run<0>("DADD chain", th, out, cyc, g);
    run<1>("DFMA chain", th, out, cyc, g);
    run<2>("DMUL chain", th, out, cyc, g);
    run<3>("FFMA chain", th, out, cyc, g);
    run<4>("SHFL fp64 chain", th, out, cyc, g);
    run<5>("SHFL fp32 chain", th, out, cyc, g);
    run<6>("LDS.64 chase (+F2I)", th, out, cyc, g);
    run<7>("__syncthreads", th, out, cyc, g);
    run<8>("fp64 clamp (min,max)", th, out, cyc, g);
    run<9>("fp64 exp", th, out, cyc, g);
    run<11>("DSETP+sel+DADD", th, out, cyc, g);
    run<12>("fp64 1/(1+x)", th, out, cyc, g);
  }
  run<10>("ld.cg L2 chase (8MB)", 32, out, cyc, g);
  run<13>("ld L1 chase (32KB)", 32, out, cyc, g);
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  printf("clock %d kHz\n", p.clockRate);
  return 0;
}
