// Microbenchmark: can the TMA unit carry the Hogwild write-back (and gather) of small factor rows?
// Compares, with all SMs busy and pseudo-random rows of a 9746 x 32 B (or 64 B) table:
//   A  red.global.add.v4.f32, lane pairs share a 32 B row          (today's V write-back)
//   B  cp.reduce.async.bulk.global.shared::cta.add.f32, 32 B per lane (one TMA reduction per row)
//   C  same, 48 B per lane into 64 B records [V(8) | w pad3]       (V and w in one operation)
//   D  cp.async.bulk global -> shared, 32 B per lane               (one TMA load per row)
//   E  ld.global.cg.v4 lane pairs                                  (today's V gather)
//   F  E and B interleaved (LSU gathers + TMA reductions: do they overlap?)
//   G  E and A interleaved (today's mix)
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tma_red_bench tma_red_bench.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <stdint.h>

// the device's SM count and maximum SM clock, read in main(): the per-SM cycle figures are
// wall time x clock x SMs / instructions
static int g_sms = 0;
static double g_hz = 0;
static void read_device() {
  int khz = 0;
  cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
  g_hz = khz * 1e3;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t hash(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x;
}
__device__ __forceinline__ void red4(float* p, float a) {
  asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1,%1,%1,%1};" ::"l"(p), "f"(a) : "memory");
}
__device__ __forceinline__ void bulk_red(float* g, const void* s, uint32_t bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(g),
               "r"(smem_u32(s)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(c) : "memory");
}
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok)
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0,1,0,p;\n}\n"
                 : "=r"(ok) : "r"(smem_u32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_load(void* s, const void* g, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(s)), "l"(g), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

template <int MODE>
__global__ void __launch_bounds__(256) k(float* tab, uint32_t rows, int niter, float* sink) {
  __shared__ __align__(128) float stage[256 * 16];  // 64 B per thread
  __shared__ uint64_t bars[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t gw = (blockIdx.x * blockDim.x + tid) >> 5;
  for (int i = 0; i < 16; i++) stage[tid * 16 + i] = 1e-9f;
  if (lane == 0) mbar_init(bars + warp, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  float acc = 0.f;
  uint32_t par = 0;
  for (int i = 0; i < niter; i++) {
    const uint32_t base = hash(gw * 7919u + i * 104729u);
    const uint32_t rp = hash(base + (lane >> 1)) % rows;  // lane pairs share a row
    const uint32_t rl = hash(base + lane) % rows;         // one row per lane
    if (MODE == 0) red4(tab + (size_t)rp * 8 + (lane & 1) * 4, 1e-9f);
    if (MODE == 1 || MODE == 5) {
      bulk_red(tab + (size_t)rl * 8, stage + tid * 16, 32);
      bulk_commit();
      if ((i & 7) == 7) bulk_wait_read0();
    }
    if (MODE == 2) {
      bulk_red(tab + (size_t)rl * 16, stage + tid * 16, 48);
      bulk_commit();
      if ((i & 7) == 7) bulk_wait_read0();
    }
    if (MODE == 3) {
      if (lane == 0) mbar_expect(bars + warp, 32 * 32);
      __syncwarp();
      bulk_load(stage + tid * 16, tab + (size_t)rl * 8, 32, bars + warp);
      mbar_wait(bars + warp, par);
      par ^= 1;
      acc += stage[tid * 16];
    }
    if (MODE == 4 || MODE == 5 || MODE == 6) {
      float4 v = __ldcg(reinterpret_cast<const float4*>(tab + (size_t)rp * 8 + (lane & 1) * 4));
      acc += v.x + v.w;
    }
    if (MODE == 6) red4(tab + (size_t)rp * 8 + (lane & 1) * 4, 1e-9f);
  }
  if (MODE == 1 || MODE == 2 || MODE == 5) bulk_wait0();
  if (acc == 123.456f) *sink = acc;
}

template <int MODE>
void run(const char* name, float* tab, uint32_t rows, int rows_per_instr) {
  const int grid = g_sms * 4, block = 256, niter = 256;
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  float* sink;
  cudaMalloc(&sink, 4);
  k<MODE><<<grid, block>>>(tab, rows, niter, sink);
  cudaEventRecord(a);
  k<MODE><<<grid, block>>>(tab, rows, niter, sink);
  cudaEventRecord(b);
  cudaEventSynchronize(b);
  float ms;
  cudaEventElapsedTime(&ms, a, b);
  const cudaError_t e = cudaGetLastError();
  const double instr = (double)grid * (block / 32) * niter;
  printf("%-58s %8.1f us  %6.1f cyc/warp-instr/SM  %5.2f cyc/row/SM  %s\n", name, ms * 1e3,
         ms * 1e-3 * g_hz * g_sms / instr, ms * 1e-3 * g_hz * g_sms / instr / rows_per_instr,
         e == cudaSuccess ? "" : cudaGetErrorString(e));
  cudaFree(sink);
}

int main() {
  read_device();
  float* tab;
  const size_t bytes = 64ull << 20;
  cudaMalloc(&tab, bytes);
  cudaMemset(tab, 0, bytes);
  const uint32_t rows = 9746;
  run<0>("A red.v4 lane pairs, 32 B rows (16 rows/instr)", tab, rows, 16);
  run<1>("B TMA bulk reduce 32 B per lane (32 rows/instr)", tab, rows, 32);
  run<2>("C TMA bulk reduce 48 B per lane, 64 B records (32 rows)", tab, rows, 32);
  run<3>("D TMA bulk load 32 B per lane + mbarrier wait (32 rows)", tab, rows, 32);
  run<4>("E ld.cg.v4 lane pairs (16 rows/instr)", tab, rows, 16);
  run<5>("F E + B interleaved (16 loads + 32 reductions / iter)", tab, rows, 16);
  run<6>("G E + A interleaved (16 loads + 16 reductions / iter)", tab, rows, 16);
  return 0;
}
