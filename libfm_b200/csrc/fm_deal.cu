// fm_deal.cu -- the dealt row order of the reproducible row-lane epoch (fm_rowlane.cu, DEALT).
//
// The epoch runs windows of G tiles of TR rows, and every row of a window reads the state the previous
// window left, whichever CTA runs it: its steps are summed as integers and the bias step is formed from
// the rows' (mult, hjoint) in file order.  So the rows of a window may be dealt to the CTAs in any order
// without changing a bit of the result.  Dealing them sorted by the id of their last entry (the item of a
// (user, item) row) puts the rows that share that feature on adjacent lanes, where one lane gathers the
// feature's parameters and one reduction carries the summed steps (DESIGN.md section 3.3).
//
// Built on the device once per data set and geometry: a stable radix sort of the rows by (window, key),
// then a copy of the CSR in that order and each row's position inside its window in file order.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "fmb200_internal.h"

namespace fmb {

namespace {

// key of row r: window * (n + 1) + the id of its last entry (n: an empty row, dealt behind the others)
__global__ void deal_key_kernel(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col, uint64_t n_rows,
                                uint64_t win_rows, uint32_t n, uint64_t* __restrict__ key, uint32_t* __restrict__ row) {
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rows; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t b = rp[r], e = rp[r + 1];
    key[r] = (r / win_rows) * ((uint64_t)n + 1) + (e > b ? col[e - 1] : n);
    row[r] = (uint32_t)r;
  }
}

// dealt row i is file row perm[i]: its length (scanned into offsets), target and position in its window
__global__ void deal_rows_kernel(const uint64_t* __restrict__ rp, const float* __restrict__ tgt,
                                 const uint32_t* __restrict__ perm, uint64_t n_rows, uint64_t win_rows,
                                 uint64_t* __restrict__ len, float* __restrict__ dtgt, uint32_t* __restrict__ pos) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i <= n_rows; i += (uint64_t)gridDim.x * blockDim.x) {
    if (i == n_rows) {
      len[i] = 0;
      continue;
    }
    const uint32_t r = perm[i];
    len[i] = rp[r + 1] - rp[r];
    dtgt[i] = tgt[r];
    pos[i] = (uint32_t)(r % win_rows);
  }
}

__global__ void deal_entries_kernel(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col,
                                    const float* __restrict__ val, const uint32_t* __restrict__ perm, uint64_t n_rows,
                                    const uint64_t* __restrict__ drp, uint32_t* __restrict__ dcol,
                                    float* __restrict__ dval) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_rows; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t r = perm[i];
    const uint64_t b = rp[r], n = rp[r + 1] - b, o = drp[i];
    for (uint64_t k = 0; k < n; k++) {
      dcol[o + k] = col[b + k];
      dval[o + k] = val[b + k];
    }
  }
}

}  // namespace

cudaError_t build_rowlane_deal(fmb200_ctx* c, DataSlot& d, int TR, uint32_t G) {
  RowlaneDeal& dl = d.deal;
  if (dl.matches(d.upload_gen, TR, G)) return cudaSuccess;
  if (d.n_rows >= 0xffffffffull) return cudaErrorInvalidValue;  // row indices are u32
  const uint64_t n_rows = d.n_rows, win_rows = (uint64_t)G * TR;
  const uint64_t n_win = (n_rows + win_rows - 1) / win_rows;
  int bits = 1;
  while (bits < 64 && ((n_win * ((uint64_t)c->n + 1)) >> bits) != 0) bits++;
  cudaError_t e;
  const uint64_t cap_r = d.cap_rows + kRowSlack, cap_e = d.cap_nnz + kEntrySlack;
  if (dl.rows_cap < cap_r || dl.nnz_cap < cap_e) {
    // the slack behind the arrays is read by the last tile's bulk copies and never used: zero it once
    if ((e = alloc(dl.row_ptr, cap_r + 1)) != cudaSuccess) return e;
    if ((e = alloc(dl.target, cap_r)) != cudaSuccess) return e;
    if ((e = alloc(dl.pos, cap_r)) != cudaSuccess) return e;
    if ((e = alloc(dl.col, cap_e)) != cudaSuccess) return e;
    if ((e = alloc(dl.val, cap_e)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(dl.row_ptr.get(), 0, (cap_r + 1) * sizeof(uint64_t), c->stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(dl.target.get(), 0, cap_r * sizeof(float), c->stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(dl.col.get(), 0, cap_e * sizeof(uint32_t), c->stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(dl.val.get(), 0, cap_e * sizeof(float), c->stream)) != cudaSuccess) return e;
    dl.rows_cap = cap_r;
    dl.nnz_cap = cap_e;
  }
  // scratch: [key in | key out | len (n_rows + 1) : u64][row in | perm : u32][sort / scan temp]
  size_t sort_bytes = 0, scan_bytes = 0;
  if ((e = cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                           (const uint32_t*)nullptr, (uint32_t*)nullptr, n_rows, 0, bits,
                                           c->stream)) != cudaSuccess)
    return e;
  if ((e = cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                         n_rows + 1, c->stream)) != cudaSuccess)
    return e;
  const size_t words = (n_rows + 1 + 63) & ~(uint64_t)63;
  const size_t need = 3 * words * 8 + 2 * words * 4 + std::max(sort_bytes, scan_bytes) + 256;
  if ((e = grow(dl.scratch, dl.scratch_bytes, need)) != cudaSuccess) return e;
  uint64_t* key_in = reinterpret_cast<uint64_t*>(dl.scratch.get());
  uint64_t* key_out = key_in + words;
  uint64_t* len = key_out + words;
  uint32_t* row_in = reinterpret_cast<uint32_t*>(len + words);
  uint32_t* perm = row_in + words;
  void* tmp = perm + words;
  const int grid = grid_for(c, n_rows + 1);
  deal_key_kernel<<<grid, 256, 0, c->stream>>>(d.row_ptr.get(), d.col.get(), n_rows, win_rows, c->n, key_in, row_in);
  if ((e = cub::DeviceRadixSort::SortPairs(tmp, sort_bytes, key_in, key_out, row_in, perm, n_rows, 0, bits,
                                           c->stream)) != cudaSuccess)
    return e;
  deal_rows_kernel<<<grid, 256, 0, c->stream>>>(d.row_ptr.get(), d.target.get(), perm, n_rows, win_rows, len,
                                                dl.target.get(), dl.pos.get());
  if ((e = cub::DeviceScan::ExclusiveSum(tmp, scan_bytes, len, dl.row_ptr.get(), n_rows + 1, c->stream)) !=
      cudaSuccess)
    return e;
  deal_entries_kernel<<<grid, 256, 0, c->stream>>>(d.row_ptr.get(), d.col.get(), d.val.get(), perm, n_rows,
                                                   dl.row_ptr.get(), dl.col.get(), dl.val.get());
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  c->launches += 5;  // keys, rows, entries + the library's sort and scan passes counted as one each
  dl.gen = d.upload_gen;
  dl.tr = TR;
  dl.grid = G;
  return cudaSuccess;
}

}  // namespace fmb
