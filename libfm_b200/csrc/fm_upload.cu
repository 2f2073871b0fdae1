// fm_upload.cu -- device side of the data-set uploads that do not arrive as SoA CSR:
//
//  * the reference's own containers (util/fmatrix.h:34-42, Data.h:238,260): an array of
//    sparse_row{sparse_entry* data; uint size;} (16 B per row) pointing into ONE contiguous
//    sparse_entry{uint id; float value;}[] block (8 B per entry).  Both arrays cross PCIe as they
//    are; the row offsets are an exclusive scan of the sizes and the AoS -> SoA split is a
//    coalesced pass, both on the device (bit-exact index work; tests/test_upload_gpu.py copies the
//    device CSR back and compares it word for word).  The scan also verifies that every row
//    pointer is where a contiguous block puts it; if not, the caller falls back to gathering the
//    rows on the host.
//  * one-hot rows of a fixed width (every value 1, e.g. (user, item) pairs): only the ids and the
//    targets cross PCIe (4*z + 4 bytes per row instead of 12*z + 12); row offsets and values are
//    materialised here.
#include "fmb200_internal.h"

namespace fmb {

namespace {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 4;  // per thread
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

struct AosRow {  // sparse_row<float> on LP64
  unsigned long long data;
  unsigned int size;
  unsigned int pad;
};

__device__ __forceinline__ unsigned long long block_exclusive_scan(unsigned long long v, unsigned long long* total) {
  // exclusive scan of one value per thread over the block (SCAN_THREADS threads)
  __shared__ unsigned long long s_warp[SCAN_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    unsigned long long w = lane < SCAN_THREADS / 32 ? s_warp[lane] : 0ull;
#pragma unroll
    for (int o = 1; o < SCAN_THREADS / 32; o <<= 1) {
      const unsigned long long t = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += t;
    }
    if (lane < SCAN_THREADS / 32) s_warp[lane] = w;  // inclusive over warps
  }
  __syncthreads();
  const unsigned long long base = warp ? s_warp[warp - 1] : 0ull;
  *total = s_warp[SCAN_THREADS / 32 - 1];
  __syncthreads();
  return base + inc - v;
}

// pass 1: per-tile sum of the row sizes
__global__ void __launch_bounds__(SCAN_THREADS) aos_tile_sums_kernel(const AosRow* __restrict__ rows, uint64_t n_rows,
                                                                     unsigned long long* __restrict__ tile_sum) {
  const uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE;
  unsigned long long v = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++) {
    const uint64_t r = base + (uint64_t)threadIdx.x * SCAN_ITEMS + i;
    if (r < n_rows) v += rows[r].size;
  }
  unsigned long long total;
  block_exclusive_scan(v, &total);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// pass 2 (one block): exclusive scan of the tile sums in place
__global__ void __launch_bounds__(SCAN_THREADS) scan_tile_sums_kernel(unsigned long long* tile_sum, uint64_t n_tiles) {
  unsigned long long carry = 0;
  for (uint64_t b = 0; b < n_tiles; b += SCAN_THREADS) {
    const uint64_t i = b + threadIdx.x;
    const unsigned long long v = i < n_tiles ? tile_sum[i] : 0ull;
    unsigned long long total;
    const unsigned long long ex = block_exclusive_scan(v, &total);
    if (i < n_tiles) tile_sum[i] = carry + ex;
    carry += total;
  }
}

// pass 3: row offsets + the contiguity check.  flag[0] |= 1 when a row's pointer is not
// base + 8 * offset (rows not laid out back to back in one block).
__global__ void __launch_bounds__(SCAN_THREADS) aos_row_ptr_kernel(const AosRow* __restrict__ rows, uint64_t n_rows,
                                                                   const unsigned long long* __restrict__ tile_off,
                                                                   unsigned long long base_ptr,
                                                                   uint64_t* __restrict__ row_ptr,
                                                                   unsigned int* __restrict__ flag) {
  const uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE;
  unsigned int sz[SCAN_ITEMS];
  unsigned long long ptr[SCAN_ITEMS];
  unsigned long long v = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++) {
    const uint64_t r = base + (uint64_t)threadIdx.x * SCAN_ITEMS + i;
    sz[i] = 0;
    ptr[i] = 0;
    if (r < n_rows) {
      sz[i] = rows[r].size;
      ptr[i] = rows[r].data;
    }
    v += sz[i];
  }
  unsigned long long total;
  unsigned long long off = tile_off[blockIdx.x] + block_exclusive_scan(v, &total);
  bool bad = false;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++) {
    const uint64_t r = base + (uint64_t)threadIdx.x * SCAN_ITEMS + i;
    if (r < n_rows) {
      row_ptr[r] = off;
      if (sz[i] != 0 && ptr[i] != base_ptr + 8ull * off) bad = true;
      off += sz[i];
      if (r + 1 == n_rows) row_ptr[n_rows] = off;
    }
  }
  if (bad) atomicOr(flag, 1u);
  if (n_rows == 0 && blockIdx.x == 0 && threadIdx.x == 0) row_ptr[0] = 0;
}

// sparse_entry{uint id; float value}[] -> col[], val[]
__global__ void aos_split_kernel(const uint2* __restrict__ ent, uint64_t nnz, uint32_t* __restrict__ col,
                                 float* __restrict__ val) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < nnz; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint2 e = ent[i];
    col[i] = e.x;
    val[i] = __uint_as_float(e.y);
  }
}

__global__ void onehot_fill_kernel(uint64_t n_rows, uint32_t z, uint64_t* __restrict__ row_ptr,
                                   float* __restrict__ val) {
  const uint64_t nnz = n_rows * z;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < nnz + n_rows + 1;
       i += (uint64_t)gridDim.x * blockDim.x) {
    if (i < nnz) val[i] = 1.f;
    else row_ptr[i - nnz] = (i - nnz) * z;
  }
}

}  // namespace

// d_rows: device copy of the sparse_row array; scratch: aos_scan_tiles(n_rows)+1 u64.
// Writes row_ptr[0..n_rows]; flag[0] bit 0 = rows are not one contiguous block.
// (d_entries / nnz / col / val: when given, the split runs in the same call.)
cudaError_t launch_aos_to_csr(fmb200_ctx* c, cudaStream_t st, const void* d_rows, const void* d_entries, uint64_t n_rows,
                              uint64_t nnz, unsigned long long host_base_ptr, unsigned long long* scratch,
                              uint64_t* row_ptr, uint32_t* col, float* val, unsigned int* flag) {
  const uint64_t n_tiles = (n_rows + SCAN_TILE - 1) / SCAN_TILE;
  const AosRow* rows = static_cast<const AosRow*>(d_rows);
  if (n_tiles > 0) {
    aos_tile_sums_kernel<<<(unsigned)n_tiles, SCAN_THREADS, 0, st>>>(rows, n_rows, scratch);
    scan_tile_sums_kernel<<<1, SCAN_THREADS, 0, st>>>(scratch, n_tiles);
    aos_row_ptr_kernel<<<(unsigned)n_tiles, SCAN_THREADS, 0, st>>>(rows, n_rows, scratch, host_base_ptr,
                                                                         row_ptr, flag);
    c->launches += 3;
  } else {
    aos_row_ptr_kernel<<<1, SCAN_THREADS, 0, st>>>(rows, 0, scratch, host_base_ptr, row_ptr, flag);
    c->launches++;
  }
  if (nnz > 0 && d_entries != nullptr) return launch_aos_split(c, st, d_entries, nnz, col, val);
  return cudaGetLastError();
}

cudaError_t launch_aos_split(fmb200_ctx* c, cudaStream_t st, const void* d_entries, uint64_t nnz, uint32_t* col, float* val) {
  if (nnz > 0) {
    aos_split_kernel<<<grid_for(c, nnz), 256, 0, st>>>(static_cast<const uint2*>(d_entries), nnz, col, val);
    c->launches++;
  }
  return cudaGetLastError();
}

uint64_t aos_scan_tiles(uint64_t n_rows) { return (n_rows + SCAN_TILE - 1) / SCAN_TILE; }

cudaError_t launch_onehot_fill(fmb200_ctx* c, cudaStream_t st, uint64_t n_rows, uint32_t z, uint64_t* row_ptr, float* val) {
  onehot_fill_kernel<<<grid_for(c, n_rows * z + n_rows + 1), 256, 0, st>>>(n_rows, z, row_ptr, val);
  c->launches++;
  return cudaGetLastError();
}

}  // namespace fmb
