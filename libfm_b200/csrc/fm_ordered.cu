// fm_ordered.cu -- launcher of the sequentially consistent epoch (fm_ordered.cuh) and the
// index work it needs per uploaded data set: for every entry the distance to the previous
// entry naming the same feature, for every row the distance to the nearest earlier row it
// depends on.  Both are pure functions of col[] / row_ptr[] (bit-exact ordering work) and
// are built once per upload, on the device, the first time an ORDERED epoch needs them.
#include <algorithm>

#include <cub/device/device_radix_sort.cuh>

#include "fm_ordered.cuh"
#include "fm_roworder.cuh"
#include "fmb200_internal.h"

namespace fmb {

namespace {

__global__ void ord_iota_kernel(uint32_t* p, uint64_t n) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    p[i] = (uint32_t)i;
}

// `ids` / `ent`: the entries stably sorted by feature id, i.e. each feature's occurrences in
// file order.  Neighbours with equal id are consecutive occurrences of one feature.
__global__ void ord_link_kernel(const uint32_t* __restrict__ ids, const uint32_t* __restrict__ ent,
                                uint64_t nnz, const uint64_t* __restrict__ rp, uint64_t n_rows,
                                uint32_t* __restrict__ link, uint32_t* __restrict__ rowdep) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < nnz;
       i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t e = ent[i];
    uint32_t L = ORD_NONE;
    if (i > 0 && ids[i - 1] == ids[i]) {
      const uint32_t pe = ent[i - 1];
      L = e - pe;
      const uint64_t r = row_of(rp, n_rows, e), pr = row_of(rp, n_rows, pe);
      atomicMin(rowdep + r, (uint32_t)(r - pr));
    }
    link[e] = L;
  }
}

// shape[0]: bit 0 = every value is exactly 1, bit 1 = every row has exactly z entries (the one-hot two-field
// shape of ratings data); the epoch kernel reads the word and takes its one-hot path when both hold
__global__ void ord_shape_kernel(const float* __restrict__ val, uint64_t nnz, const uint64_t* __restrict__ rp,
                                 uint64_t n_rows, uint32_t z, uint32_t* shape) {
  uint32_t clear = 0;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < nnz; i += (uint64_t)gridDim.x * blockDim.x)
    if (val[i] != 1.0f) clear |= 1u;
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rows;
       r += (uint64_t)gridDim.x * blockDim.x)
    if (rp[r + 1] - rp[r] != z) clear |= 2u;
  if (clear) atomicAnd(shape, ~clear);
}

// One CTA, one group of GL lanes per example of a run: ORD_SMAX * GL compute threads (at most 1 024; small k
// leaves the register file to few threads, k <= 8: 128).  HELPERS (k <= 32 only, where they fit): then
// ORD_PARKED threads that leave after the set-up and ORD_HELPERS helper threads (write-back, fetch); without
// them the compute threads do that work themselves (ordered_epoch).  ONE helper warp: every further helper
// warp slowed the epoch by ~5% although the helpers idle most of the time -- their bursts of shared-memory / LSU
// traffic delay the compute warps' loads (r02 calls M, N, the same build on one box, C2-shaped 200 000 rows:
// 1 / 2 / 3 / 4 helper warps = 6.30 / 6.64-6.74 / 6.92 / 7.33 ms; which schedulers the helpers sit on matters
// little).  The parked threads keep the helper warp's index a multiple of 4 apart from compute warp 3.
constexpr int ORD_PARKED = 96;
constexpr int ORD_HELPERS = 32;
template <int GL, int KF, int TASK, int ZF, bool HELPERS>
__global__ void __launch_bounds__(HELPERS ? ORD_SMAX * GL + ORD_PARKED + ORD_HELPERS
                                          : (ORD_SMAX * GL < 256 ? 256 : (ORD_SMAX * GL < ORD_MAX_THREADS ? ORD_SMAX * GL : ORD_MAX_THREADS)), 1)
    fm_sgd_ordered_kernel(const OrderedArgs a) {
  extern __shared__ __align__(128) unsigned char ord_smem[];
  if constexpr (HELPERS) ordered_epoch_body_ws<GL, KF, TASK, ZF>(a, ord_smem, ORD_SMAX * GL, ORD_PARKED);
  else ordered_epoch_body<GL, KF, TASK, ZF>(a, ord_smem);
}

using OrdFn = void (*)(const OrderedArgs);

// (GL lanes per example, KF consecutive factors per lane): KF <= 8; k <= 8 runs one lane per example
inline void ordered_shape(int k, int* GL, int* KF) {
  if (k <= 8) {
    *GL = 1;
    *KF = k <= 1 ? 1 : (k <= 2 ? 2 : (k <= 4 ? 4 : 8));
    return;
  }
  *KF = 8;
  int g = 2;
  while (g * 8 < k) g <<= 1;
  *GL = g;
}

// the register-resident fast path where `fast` allows it (k in {2,4,8} exactly, rows of at most 2 / 4
// entries), else the general kernel of ordered_shape's (GL, KF); with helpers where H asks for them (k <= 32)
template <int TASK, bool H>
OrdFn pick_kernel(int k, uint32_t max_row_nnz, bool fast) {
  if (fast && max_row_nnz >= 1 && max_row_nnz <= 4) {
    const bool z2 = max_row_nnz <= 2;
    if (k == 2) return z2 ? fm_sgd_ordered_kernel<1, 2, TASK, 2, H> : fm_sgd_ordered_kernel<1, 2, TASK, 4, H>;
    if (k == 4) return z2 ? fm_sgd_ordered_kernel<1, 4, TASK, 2, H> : fm_sgd_ordered_kernel<1, 4, TASK, 4, H>;
    if (k == 8) return z2 ? fm_sgd_ordered_kernel<1, 8, TASK, 2, H> : fm_sgd_ordered_kernel<1, 8, TASK, 4, H>;
  }
  if (k <= 1) return fm_sgd_ordered_kernel<1, 1, TASK, 0, H>;
  if (k <= 2) return fm_sgd_ordered_kernel<1, 2, TASK, 0, H>;
  if (k <= 4) return fm_sgd_ordered_kernel<1, 4, TASK, 0, H>;
  if (k <= 8) return fm_sgd_ordered_kernel<1, 8, TASK, 0, H>;
  if (k <= 16) return fm_sgd_ordered_kernel<2, 8, TASK, 0, H>;
  if (k <= 32) return fm_sgd_ordered_kernel<4, 8, TASK, 0, H>;
  if (k <= 64) return fm_sgd_ordered_kernel<8, 8, TASK, 0, false>;
  if (k <= 128) return fm_sgd_ordered_kernel<16, 8, TASK, 0, false>;
  return fm_sgd_ordered_kernel<32, 8, TASK, 0, false>;
}

// the stable (id, entry) sort in the scratch of the index build, [ids | ent_in | ent | sort temp]
SortedEntries sorted_view(const DataSlot& d) {
  const size_t words = ((size_t)d.nnz + 63) & ~(size_t)63;
  const uint32_t* ids = reinterpret_cast<const uint32_t*>(d.ord_scratch.get());
  return SortedEntries{ids, ids + 2 * words};
}

}  // namespace

cudaError_t build_ordered_links(fmb200_ctx* c, DataSlot& d, SortedEntries* sorted) {
  // (a large data set releases its sort once the index is built: a caller that needs it rebuilds)
  if (d.links_ready && !(sorted && d.nnz > 0 && !d.ord_scratch)) {
    if (sorted) *sorted = sorted_view(d);
    return cudaSuccess;
  }
  if (d.nnz >= 0xffffffffull) return cudaErrorInvalidValue;
  cudaError_t e;
  const uint64_t cap_e = d.cap_nnz + kEntrySlack, cap_r = d.cap_rows + kRowSlack;
  if ((e = grow(d.link, d.link_cap, cap_e)) != cudaSuccess) return e;
  if ((e = grow(d.rowdep, d.rowdep_cap, cap_r + 4)) != cudaSuccess) return e;  // + the shape word
  d.ord_shape = d.rowdep.get() + cap_r;
  {
    if ((e = cudaMemsetAsync(d.ord_shape, 0x03, sizeof(uint32_t), c->stream)) != cudaSuccess) return e;
    ord_shape_kernel<<<grid_for(c, d.nnz + d.n_rows), 256, 0, c->stream>>>(d.val.get(), d.nnz, d.row_ptr.get(),
                                                                           d.n_rows, d.max_row_nnz, d.ord_shape);
    c->launches++;
  }
  if ((e = cudaMemsetAsync(d.link.get(), 0xff, cap_e * sizeof(uint32_t), c->stream)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(d.rowdep.get(), 0xff, cap_r * sizeof(uint32_t), c->stream)) != cudaSuccess) return e;
  if (d.nnz > 0) {
    int bits = 1;
    while (bits < 32 && (1ull << bits) < (uint64_t)c->n) bits++;
    size_t tmp_bytes = 0;
    e = cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, d.col.get(), (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                        (uint32_t*)nullptr, (uint64_t)d.nnz, 0, bits, c->stream);
    if (e != cudaSuccess) return e;
    // scratch of the index build: [ids | ent_in | ent | sort temp].  Kept with the slot for data sets up to
    // 64 M entries (a re-upload then rebuilds its index without a single allocation or host sync -- the
    // end-to-end path uploads a fresh data set every step); larger ones release it right away.
    const size_t words = ((size_t)d.nnz + 63) & ~(size_t)63;
    const size_t need = 3 * words * sizeof(uint32_t) + ((tmp_bytes + 255) & ~(size_t)255) + 256;
    if ((e = grow(d.ord_scratch, d.ord_scratch_bytes, need)) != cudaSuccess) return e;
    uint32_t* ids = reinterpret_cast<uint32_t*>(d.ord_scratch.get());
    uint32_t* ent_in = ids + words;
    uint32_t* ent = ent_in + words;
    void* tmp = ent + words;
    ord_iota_kernel<<<grid_for(c, d.nnz), 256, 0, c->stream>>>(ent_in, d.nnz);
    e = cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, d.col.get(), ids, ent_in, ent, (uint64_t)d.nnz, 0, bits,
                                        c->stream);
    if (e != cudaSuccess) return e;
    ord_link_kernel<<<grid_for(c, d.nnz), 256, 0, c->stream>>>(ids, ent, d.nnz, d.row_ptr.get(), d.n_rows,
                                                                d.link.get(), d.rowdep.get());
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    c->launches += 3;  // iota, link + the library's sort passes counted as one
    if (d.nnz > (64ull << 20) && !sorted) {
      if ((e = cudaStreamSynchronize(c->stream)) != cudaSuccess) return e;
      d.ord_scratch.reset();
      d.ord_scratch_bytes = 0;
    }
  }
  d.links_ready = true;
  if (sorted) *sorted = sorted_view(d);
  return cudaSuccess;
}

// Pick the tile geometry; false if not even one row fits the ring (caller falls back to the
// row-at-a-time kernel, which is also sequentially consistent).
bool ordered_geometry(const fmb200_ctx* c, const DataSlot& d, int* TR_out, uint32_t* TE_out, int* kw_out,
                      int* rs_out, size_t* smem_out) {
  const int k = c->k;
  const int kw = (k & 1) ? k + 1 : k;
  const int rs = kw + 2;
  const size_t limit = (size_t)c->max_smem_optin;
  for (int TR = 256; TR >= 1; TR >>= 1) {
    uint64_t span;
    if (TR >= 32) {
      int idx = 0;
      while ((32 << idx) < TR) idx++;
      span = d.tile_span[idx];
    } else {
      span = (uint64_t)TR * d.max_row_nnz + 6;
      if (span > d.tile_span[0]) span = d.tile_span[0];
    }
    const uint64_t TE64 = ((span + 3) & ~3ull) + 4;
    if (TE64 > (1u << 20)) continue;
    const uint32_t TE = (uint32_t)TE64;
    const size_t need = ord_smem_bytes(TR, TE, rs);
    if (need <= limit) {
      *TR_out = TR;
      *TE_out = TE;
      *kw_out = kw;
      *rs_out = rs;
      *smem_out = need;
      return true;
    }
  }
  return false;
}

cudaError_t launch_sgd_ordered(fmb200_ctx* c, DataSlot& d, bool* handled) {
  *handled = false;
  if (d.n_rows == 0) {
    *handled = true;
    return cudaSuccess;
  }
  if (d.nnz >= 0xffffffffull) return cudaSuccess;  // 32-bit entry distances: not eligible
  int TR = 0, kw = 0, rs = 0;
  uint32_t TE = 0;
  size_t smem = 0;
  if (!ordered_geometry(c, d, &TR, &TE, &kw, &rs, &smem)) return cudaSuccess;
  cudaError_t e = build_ordered_links(c, d);
  if (e != cudaSuccess) return e;

  OrderedArgs a{};
  a.row_ptr = d.row_ptr.get();
  a.col = d.col.get();
  a.val = d.val.get();
  a.target = d.target.get();
  a.link = d.link.get();
  a.rowdep = d.rowdep.get();
  a.shape = d.ord_shape;
  a.n_rows = d.n_rows;
  a.n_tiles = (uint32_t)((d.n_rows + TR - 1) / TR);
  a.tile_rows = TR;
  a.tile_cap = TE;
  a.w0 = c->p64.w0();
  a.w = c->p64.w();
  a.v = c->p64.v();
  a.k = c->k;
  a.kw = kw;
  a.rs = rs;
  a.use_w0 = c->k0;
  a.use_w = c->k1;
  a.lr = c->hp.lr;
  a.reg0 = c->hp.reg0;
  a.regw = c->hp.regw;
  a.regv = c->hp.regv;
  a.min_target = c->hp.min_target;
  a.max_target = c->hp.max_target;
  a.csr_bytes = ord_csr_bytes(TR, TE);
  a.rec_bytes = TE * (uint32_t)rs * 8u;
  a.debug = (c->tune_variant >= 100) ? c->tune_variant - 100 : 0;  // timing experiments (wrong results)
  const bool want_prof = (a.debug & 32) != 0;  // variant 132 (+ skip bits): print the phase timers
  a.debug &= 31;
  PhaseTimers prof;
  if (want_prof && (e = prof.start(16, c->stream)) != cudaSuccess) return e;
  a.prof = prof.slots.get();

  int GL = 1, KF = 1;
  ordered_shape(c->k, &GL, &KF);
  // one group of GL lanes per example of a run: min(ORD_SMAX, 1024 / GL) examples
  int threads = std::min(ORD_SMAX * GL, ORD_MAX_THREADS);
  const int bound = std::max(threads, 256);  // the launch bound without helpers
  if (c->tune_threads)  // fewer threads = shorter runs; more = threads that only share the fetch issue / write-back
    threads = std::min(bound, std::max(32, (c->tune_threads / (32 > GL ? 32 : GL)) * (32 > GL ? 32 : GL)));
  const bool fast = c->tune_variant != 1;  // variant 1 forces the general path
  // the helper warp is the default where it fits (variant 1 / 2 and explicit thread counts keep every thread a
  // compute thread: comparisons, tests)
  const bool helpers = GL <= 4 && c->tune_variant != 1 && c->tune_variant != 2 && !c->tune_threads;
  const bool reg = c->hp.task == FMB200_TASK_REGRESSION;
  OrdFn fn = (helpers ? (reg ? pick_kernel<0, true> : pick_kernel<1, true>)
                      : (reg ? pick_kernel<0, false> : pick_kernel<1, false>))(c->k, d.max_row_nnz, fast);
  const int ncompute = threads;
  if (helpers) threads += ORD_PARKED + ORD_HELPERS;
  e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  fn<<<1, threads, smem, c->stream>>>(a);
  c->launches++;
  c->last_cfg = EpochConfig{GL, std::min(ORD_SMAX, ncompute / GL), TR, 1, threads, (int)smem, 0};
  *handled = true;
  if (want_prof) {
    static const char* name[16] = {"A scores", "A barrier", "chain", "chain barrier", "check+sgd", "closing barrier",
                                   "tile prologue", "wait for helpers", "H write-back", "H csr", "H fetch issue",
                                   "H fetch landing", "H wait for compute", "-", "-", "between"};
    if ((e = prof.print(c->stream, name, a.n_tiles, 0, true, "[ordered phases, cycles per tile (%u tiles)]",
                        a.n_tiles)) != cudaSuccess)
      return e;
  }
  return cudaGetLastError();
}

}  // namespace fmb
