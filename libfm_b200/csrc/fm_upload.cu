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
//  * blocks of a binary .x file as the file stores them (per row {uint size; size x {uint id; float
//    value}}): the rows' sizes cross PCIe beside the block; the same offset scan builds the row offsets and
//    checks every row's header word against its size, and a split pass writes the ids and values.
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

// The offset scan reads each row's size, and checks each row against the offset the scan gives it,
// through a row source:
//   AosRows:    sparse_row records; a row must point where one contiguous entry block puts it
//   XblockRows: sizes beside a .x block; the block's header word of the row must equal its size
struct AosRows {
  const AosRow* rows;
  unsigned long long base_ptr;
  __device__ unsigned int size(uint64_t r) const { return rows[r].size; }
  __device__ bool ok(uint64_t r, unsigned int sz, unsigned long long off) const {
    return sz == 0 || rows[r].data == base_ptr + 8ull * off;
  }
};
struct XblockRows {
  const unsigned int* row_size;
  const unsigned int* words;  // the block: row r's header is word r + 2 * row_ptr[r]
  uint64_t n_words;
  __device__ unsigned int size(uint64_t r) const { return row_size[r]; }
  __device__ bool ok(uint64_t r, unsigned int sz, unsigned long long off) const {
    const unsigned long long w = r + 2ull * off;
    return w < n_words && words[w] == sz;
  }
};

// pass 1: per-tile sum of the row sizes
template <class Rows>
__global__ void __launch_bounds__(SCAN_THREADS) row_tile_sums_kernel(Rows rows, uint64_t n_rows,
                                                                     unsigned long long* __restrict__ tile_sum) {
  const uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE;
  unsigned long long v = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++) {
    const uint64_t r = base + (uint64_t)threadIdx.x * SCAN_ITEMS + i;
    if (r < n_rows) v += rows.size(r);
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

// pass 3: row offsets + the row source's check.  *flag := max over the failing rows r of n_rows - r, so
// 0 means every row passed and otherwise n_rows - *flag is the first failing row (n_rows < 2^32).
template <class Rows>
__global__ void __launch_bounds__(SCAN_THREADS) row_ptr_kernel(Rows rows, uint64_t n_rows,
                                                               const unsigned long long* __restrict__ tile_off,
                                                               uint64_t* __restrict__ row_ptr,
                                                               unsigned int* __restrict__ flag) {
  const uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE;
  unsigned int sz[SCAN_ITEMS];
  unsigned long long v = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++) {
    const uint64_t r = base + (uint64_t)threadIdx.x * SCAN_ITEMS + i;
    sz[i] = r < n_rows ? rows.size(r) : 0u;
    v += sz[i];
  }
  unsigned long long total;
  unsigned long long off = tile_off[blockIdx.x] + block_exclusive_scan(v, &total);
  unsigned int bad = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++) {
    const uint64_t r = base + (uint64_t)threadIdx.x * SCAN_ITEMS + i;
    if (r < n_rows) {
      row_ptr[r] = off;
      if (!bad && !rows.ok(r, sz[i], off)) bad = (unsigned int)(n_rows - r);
      off += sz[i];
      if (r + 1 == n_rows) row_ptr[n_rows] = off;
    }
  }
  if (bad) atomicMax(flag, bad);
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

// .x block -> col[], val[].  One CTA per XSPLIT_ROWS rows: their offsets go to shared memory, then the
// CTA's threads walk the rows' entries e in order (coalesced writes) and find each entry's row r by a
// binary search there; entry e of row r is word (r + 1) + 2e of the block.  Entries at or past nnz are
// never written (a header that disagrees with row_size fails the upload, but must not overrun col / val).
constexpr int XSPLIT_ROWS = 256;
__global__ void __launch_bounds__(XSPLIT_ROWS) xblock_split_kernel(const unsigned int* __restrict__ words,
                                                                   const uint64_t* __restrict__ row_ptr,
                                                                   uint64_t n_rows, uint64_t nnz,
                                                                   uint32_t* __restrict__ col,
                                                                   float* __restrict__ val) {
  __shared__ unsigned long long s_rp[XSPLIT_ROWS + 1];
  const uint64_t r0 = (uint64_t)blockIdx.x * XSPLIT_ROWS;
  const int nr = (int)min((uint64_t)XSPLIT_ROWS, n_rows - r0);
  for (int i = threadIdx.x; i <= nr; i += blockDim.x) s_rp[i] = row_ptr[r0 + i];
  __syncthreads();
  const unsigned long long e_end = min((unsigned long long)nnz, s_rp[nr]);
  for (unsigned long long e = s_rp[0] + threadIdx.x; e < e_end; e += blockDim.x) {
    int lo = 0, hi = nr - 1;  // the last row starting at or before e
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (s_rp[mid] <= e) lo = mid;
      else hi = mid - 1;
    }
    const unsigned long long w = r0 + (unsigned long long)lo + 1ull + 2ull * e;
    col[e] = words[w];
    val[e] = __uint_as_float(words[w + 1]);
  }
}

template <class Rows>
void launch_row_offsets(fmb200_ctx* c, cudaStream_t st, Rows rows, uint64_t n_rows, unsigned long long* scratch,
                        uint64_t* row_ptr, unsigned int* flag) {
  const uint64_t n_tiles = (n_rows + SCAN_TILE - 1) / SCAN_TILE;
  if (n_tiles > 0) {
    row_tile_sums_kernel<<<(unsigned)n_tiles, SCAN_THREADS, 0, st>>>(rows, n_rows, scratch);
    scan_tile_sums_kernel<<<1, SCAN_THREADS, 0, st>>>(scratch, n_tiles);
    row_ptr_kernel<<<(unsigned)n_tiles, SCAN_THREADS, 0, st>>>(rows, n_rows, scratch, row_ptr, flag);
    c->launches += 3;
  } else {
    row_ptr_kernel<<<1, SCAN_THREADS, 0, st>>>(rows, 0, scratch, row_ptr, flag);
    c->launches++;
  }
}

// *out := the largest id of col[0..nnz) (atomicMax; *out starts at 0)
__global__ void max_id_kernel(const uint32_t* __restrict__ col, uint64_t nnz, unsigned int* out) {
  unsigned int m = 0;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < nnz; i += (uint64_t)gridDim.x * blockDim.x)
    m = max(m, col[i]);
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
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
// Writes row_ptr[0..n_rows]; flag[0] != 0: the rows are not one contiguous block.
// (d_entries / nnz / col / val: when given, the split runs in the same call.)
cudaError_t launch_aos_to_csr(fmb200_ctx* c, cudaStream_t st, const void* d_rows, const void* d_entries, uint64_t n_rows,
                              uint64_t nnz, unsigned long long host_base_ptr, unsigned long long* scratch,
                              uint64_t* row_ptr, uint32_t* col, float* val, unsigned int* flag) {
  launch_row_offsets(c, st, AosRows{static_cast<const AosRow*>(d_rows), host_base_ptr}, n_rows, scratch, row_ptr, flag);
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

cudaError_t launch_xblock_to_csr(fmb200_ctx* c, cudaStream_t st, const unsigned int* d_words, const unsigned int* d_row_size,
                                 uint64_t n_rows, uint64_t nnz, unsigned long long* scratch, uint64_t* row_ptr,
                                 uint32_t* col, float* val, unsigned int* flag) {
  launch_row_offsets(c, st, XblockRows{d_row_size, d_words, n_rows + 2 * nnz}, n_rows, scratch, row_ptr, flag);
  if (n_rows > 0 && nnz > 0) {
    const uint64_t grid = (n_rows + XSPLIT_ROWS - 1) / XSPLIT_ROWS;
    xblock_split_kernel<<<(unsigned)grid, XSPLIT_ROWS, 0, st>>>(d_words, row_ptr, n_rows, nnz, col, val);
    c->launches++;
  }
  return cudaGetLastError();
}

cudaError_t launch_max_id(fmb200_ctx* c, cudaStream_t st, const uint32_t* col, uint64_t nnz, unsigned int* out) {
  if (nnz > 0) {
    max_id_kernel<<<grid_for(c, nnz), 256, 0, st>>>(col, nnz, out);
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
