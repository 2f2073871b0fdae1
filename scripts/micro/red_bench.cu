// Microbenchmark: cost model of fire-and-forget fp32 reductions (REDG), and of the write-back forms of a
// k=8 fixed-point record: 64 bytes of 64-bit integers (REDG.E.ADD.64 scattered or sector-coalesced, UBLKRED,
// on or off a 64-byte boundary) or 32 bytes of 32-bit integers (UBLKRED), and of a paired 32-byte row
// gather on or off a sector boundary.
// Each warp issues NITER reduction instructions (or record write-backs) to pseudo-random rows of a table.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o red_bench red_bench.cu
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
__device__ __forceinline__ void red4(float* p, float a) {
  asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1,%1,%1,%1};" ::"l"(p), "f"(a) : "memory");
}
__device__ __forceinline__ void red2(float* p, float a) {
  asm volatile("red.relaxed.gpu.global.add.v2.f32 [%0], {%1,%1};" ::"l"(p), "f"(a) : "memory");
}
__device__ __forceinline__ void red1(float* p, float a) {
  asm volatile("red.relaxed.gpu.global.add.f32 [%0], %1;" ::"l"(p), "f"(a) : "memory");
}
__device__ __forceinline__ uint32_t hash(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x;
}
// mode 0: v4, lane pairs share a 32B row (16 sectors / instr)
// mode 1: scalar, 16 active lanes, 16 sectors
// mode 2: scalar, 32 lanes, 32 sectors
// mode 3: v4, 32 lanes, 32 distinct sectors (16B each)
// mode 4: v4, 8 lanes cover one 128B line (4 lines / instr)
// mode 5: v4, 4 lanes cover 64B (8 half-lines / instr)
// mode 6: v2, 4 lanes share a 32B row (8 sectors)
// mode 7: loads instead (ld.cg v4 paired, 16 sectors) for comparison
// mode 12: mode 7 with every 32-byte row 16 bytes into a sector (each row straddles two sectors)
template <int MODE>
__global__ void k(float* tab, uint32_t rows32 /*number of 32B rows*/, int niter, float* sink) {
  const int lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  float acc = 0.f;
  for (int i = 0; i < niter; i++) {
    const uint32_t base = hash(gw * 7919u + i * 104729u);
    if (MODE == 0) { uint32_t r = hash(base + (lane >> 1)) % rows32; red4(tab + (size_t)r * 8 + (lane & 1) * 4, 1e-9f); }
    if (MODE == 1) { if (lane < 16) { uint32_t r = hash(base + lane) % rows32; red1(tab + (size_t)r * 8, 1e-9f); } }
    if (MODE == 2) { uint32_t r = hash(base + lane) % rows32; red1(tab + (size_t)r * 8, 1e-9f); }
    if (MODE == 3) { uint32_t r = hash(base + lane) % rows32; red4(tab + (size_t)r * 8, 1e-9f); }
    if (MODE == 4) { uint32_t r = hash(base + (lane >> 3)) % (rows32 / 4); red4(tab + (size_t)r * 32 + (lane & 7) * 4, 1e-9f); }
    if (MODE == 5) { uint32_t r = hash(base + (lane >> 2)) % (rows32 / 2); red4(tab + (size_t)r * 16 + (lane & 3) * 4, 1e-9f); }
    if (MODE == 6) { uint32_t r = hash(base + (lane >> 2)) % rows32; red2(tab + (size_t)r * 8 + (lane & 3) * 2, 1e-9f); }
    if (MODE == 8) { uint32_t r = hash(base + lane) % rows32; red1(tab + r, 1e-9f); }
    if (MODE == 9) { uint32_t r = hash(base + lane) % rows32; acc += __ldcg(tab + r); }
    if (MODE == 10) { uint32_t r = hash(base + lane) % rows32; acc += __ldcg(tab + r); red1(tab + r, 1e-9f); }
    if (MODE == 11) { uint32_t r = hash(base + lane) % rows32; acc += __ldcg(tab + (size_t)r * 8); red1(tab + (size_t)r * 8, 1e-9f); }
    if (MODE == 12) { uint32_t r = hash(base + (lane >> 1)) % rows32; float4 v = __ldcg(reinterpret_cast<const float4*>(tab + 4 + (size_t)r * 8 + (lane & 1) * 4)); acc += v.x + v.w; }
    if (MODE == 7) { uint32_t r = hash(base + (lane >> 1)) % rows32; float4 v = __ldcg(reinterpret_cast<const float4*>(tab + (size_t)r * 8 + (lane & 1) * 4)); acc += v.x + v.w; }
  }
  if (acc == 123.456f) *sink = acc;
}
// ---- 64-bit integer reductions into 64-byte records (8 x u64: a k=8 factor row of a fixed-point
// accumulator).  Every lane writes back one record per iteration; the three forms differ in how:
// mode 0: scattered, as after a lane-pair half swap: lanes 2j, 2j+1 share a record, lane 2j owns its
//         low 32-byte sector, 2j+1 the high one; 4 scalar REDs per sector, 8 instructions for 2 records
//         per lane pair, and every instruction touches 32 sectors with 8 bytes each
// mode 1: sector-coalesced: the 4 lanes of a quad cover one 32-byte sector (4 x 8 B contiguous); the
//         same 8 instructions per 32 records, each touching 8 full sectors
// mode 2: bulk: one cp.reduce.async.bulk .add.u64 of the lane's 64-byte record from shared memory
// mode 3: bulk, narrow: one cp.reduce.async.bulk .add.s32 of a 32-byte record (8 x s32), one sector
// mode 4: mode 2 with every record 32 bytes off a 64-byte boundary (every other one straddles a line)
__device__ __forceinline__ void red_u64(unsigned long long* p, unsigned long long a) {
  asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(p), "l"(a) : "memory");
}
__device__ __forceinline__ void bulk_red_s32(void* g, const void* s, uint32_t bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.s32 [%0], [%1], %2;" ::"l"(g),
               "r"((uint32_t)__cvta_generic_to_shared(s)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_red_u64(unsigned long long* g, const void* s, uint32_t bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.u64 [%0], [%1], %2;" ::"l"(g),
               "r"((uint32_t)__cvta_generic_to_shared(s)), "r"(bytes) : "memory");
}
template <int MODE>
__global__ void __launch_bounds__(256) k64(unsigned long long* tab, uint32_t recs, int niter) {
  __shared__ __align__(128) unsigned long long stage[256 * 8];  // 64 B per thread (mode 2)
  const int tid = threadIdx.x, lane = tid & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + tid) >> 5;
  for (int i = 0; i < 8; i++) stage[tid * 8 + i] = 1ull;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> bulk reads
  __syncthreads();
  for (int i = 0; i < niter; i++) {
    const uint32_t base = hash(gw * 7919u + i * 104729u);
    if (MODE == 0) {
      const uint32_t ra = hash(base + (lane & ~1)) % recs, rb = hash(base + (lane | 1)) % recs;
      unsigned long long* pa = tab + (size_t)ra * 8 + (lane & 1) * 4;
      unsigned long long* pb = tab + (size_t)rb * 8 + (lane & 1) * 4;
#pragma unroll
      for (int e = 0; e < 4; e++) red_u64(pa + e, 1ull);
#pragma unroll
      for (int e = 0; e < 4; e++) red_u64(pb + e, 1ull);
    }
    if (MODE == 1) {
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const uint32_t rec = hash(base + ((lane & ~3) | r)) % recs;
#pragma unroll
        for (int h = 0; h < 2; h++) red_u64(tab + (size_t)rec * 8 + h * 4 + (lane & 3), 1ull);
      }
    }
    if (MODE >= 2) {
      const size_t rec = hash(base + lane) % recs;
      if (MODE == 2) bulk_red_u64(tab + rec * 8, stage + tid * 8, 64);
      if (MODE == 3) bulk_red_s32(tab + rec * 4, stage + tid * 8, 32);
      if (MODE == 4) bulk_red_u64(tab + 4 + rec * 8, stage + tid * 8, 64);
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      if ((i & 7) == 7) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    }
  }
  if (MODE >= 2) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
template <int MODE>
void run64(const char* name, unsigned long long* tab, uint32_t recs, int grid, int block, int niter) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  k64<MODE><<<grid, block>>>(tab, recs, niter);
  cudaEventRecord(a);
  k64<MODE><<<grid, block>>>(tab, recs, niter);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  const cudaError_t e = cudaGetLastError();
  const double records = (double)grid * block * niter;
  printf("%-44s recs=%6u grid=%4d: %8.1f us  %6.2f G records/s  %7.2f ps/record  %6.2f cyc/record/SM  %s\n", name,
         recs, grid, ms * 1e3, records / ms / 1e6, ms * 1e9 / records, ms * 1e-3 * g_hz * g_sms / records,
         e == cudaSuccess ? "" : cudaGetErrorString(e));
}
template <int MODE>
void run(const char* name, float* tab, uint32_t rows32, int grid, int block, int niter, float* sink) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  k<MODE><<<grid, block>>>(tab, rows32, niter, sink);
  cudaEventRecord(a);
  k<MODE><<<grid, block>>>(tab, rows32, niter, sink);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  double instr = (double)grid * (block / 32) * niter;
  int sms = grid < g_sms ? grid : g_sms;
  printf("%-44s rows=%8u grid=%4d: %8.1f us  %7.2f G instr/s  %6.1f cyc/instr/SM\n", name, rows32, grid, ms * 1e3,
         instr / ms / 1e6, ms * 1e-3 * g_hz * sms / instr);
}
int main() {
  read_device();
  float *tab, *sink; size_t bytes = 512ull << 20;
  cudaMalloc(&tab, bytes); cudaMemset(tab, 0, bytes); cudaMalloc(&sink, 4);
  const int niter = 256, block = 256;
  for (uint32_t rows32 : {9746u, 82248u}) {
    int grid = g_sms * 4;
    run<2>("scalar RED 32 lanes, 32B stride", tab, rows32, grid, block, niter, sink);
    run<8>("scalar RED 32 lanes, contiguous 4B", tab, rows32, grid, block, niter, sink);
    run<9>("scalar LD  32 lanes, contiguous 4B", tab, rows32, grid, block, niter, sink);
    run<10>("LD+RED same word, contiguous 4B", tab, rows32, grid, block, niter, sink);
    run<11>("LD+RED same word, 32B stride", tab, rows32, grid, block, niter, sink);
    run<0>("v4 paired RED (16 sectors)", tab, rows32, grid, block, niter, sink);
    run<7>("v4 paired LD (16 sectors)", tab, rows32, grid, block, niter, sink);
    run<12>("(f) v4 paired LD, rows 16 B into a sector", tab, rows32, grid, block, niter, sink);
  }
  // 64-byte u64 records of the k=8 accumulator; 9746 = the C2 feature count
  unsigned long long* tab64 = reinterpret_cast<unsigned long long*>(tab);
  for (uint32_t recs : {9746u, 82248u}) {
    const int grid = g_sms * 4;
    run64<0>("u64 (a) scattered, 8 REDs/record, 32 sectors", tab64, recs, grid, block, niter);
    run64<1>("u64 (b) quad per sector, 8 REDs/record, 8 sec", tab64, recs, grid, block, niter);
    run64<2>("u64 (c) bulk reduce, 64 B/record", tab64, recs, grid, block, niter);
    run64<3>("s32 (d) bulk reduce, 32 B/record", tab64, recs, grid, block, niter);
    run64<4>("u64 (e) bulk reduce, 64 B at 32 mod 64", tab64, recs, grid, block, niter);
  }
  return 0;
}
