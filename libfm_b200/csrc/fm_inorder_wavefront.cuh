// fm_inorder_wavefront.cuh -- the wavefront schedule of the sequential-equivalent epochs: the
// window pieces both wavefront kernels are built from, and the SGD epoch (the SGDA epoch is in
// fm_sgda_wavefront.cuh).  Included by fm_inorder.cu (compiled with --fmad=false).  Kept in
// headers of their own so that tests/simt/ can compile this exact source for the host and run it
// as 32 threads (one per lane, barriers where the kernel synchronises) against the oracle and
// under ThreadSanitizer.
#pragma once
#include "fm_loss.cuh"
#include "fmb200_internal.h"

namespace fmb {

// ---------------------------------------------------------------------------------------
// Wavefront schedule of the in-order epoch (short rows, small k).
//
// The row-at-a-time kernel above pays three dependent L2 round trips per example.  The
// sequential semantics only force ONE chain through the epoch: the bias.  Every example
// reads w0 as the FIRST addend of its score (fm_model.h:107-109) and writes it back
// (fm_sgd.h:34-37); because floating-point addition is not associative the whole
// left-to-right accumulation  ((w0 + a_1) + a_2 ...) + b_1 ... + b_k  has to run after
// w0 is known, but the addends themselves -- a_i = w[id_i]*x_i and
// b_f = 0.5*(sum_f^2 - sumsq_f) -- depend only on the rows of w and V the example touches.
// Consecutive examples that share no feature can therefore gather and form their addends
// in parallel, run the scalar chain one after the other, and scatter their updates in
// parallel, with every rounding identical to the sequential loop.
//
// One warp, lane = example.  Per window:
//   1. the next 32 examples load their entries (WfRow); a shared-memory hash table (WfHash)
//      finds the longest prefix P in which no example touches a feature of an earlier one
//      (hash collisions only shorten P -- conservative);
//   2. lanes < P gather w / V rows (fp64) and form their addends into shared memory (WfGather);
//   3. all lanes walk the chain t = 0..P-1 redundantly from shared memory (broadcast
//      reads, software-prefetched one example ahead): about nnz + k + 6 dependent fp64
//      operations per example, the only serial part left;
//   4. lanes < P apply fm_SGD to their own rows (WfGather::scatter: cached values; a row that
//      names the same feature twice re-reads memory so the second update sees the first).
// The next window starts at example base + P.
constexpr int WF_Z = 4;        // entries per row
constexpr int WF_K = 8;        // factors
constexpr int WF_HASH = 2048;  // hash slots (power of two)

// the shapes a wavefront kernel takes: k <= WF_K and rows of at most WF_Z entries
inline bool wavefront_fits(int k, uint32_t max_row_nnz) { return k <= WF_K && max_row_nnz <= (uint32_t)WF_Z; }

// what a wavefront epoch reports (fmb200_get_epoch_config): one warp, lane = row
inline EpochConfig wavefront_config(int smem) { return EpochConfig{32, WF_Z, 32, 1, 32, smem, 0}; }

__device__ __forceinline__ uint32_t wf_hash(uint32_t id) {
  return (id * 2654435761u) >> (32 - 11);
}
static_assert(WF_HASH == (1 << 11), "wf_hash produces 11 bits");

// A CSR row of at most WF_Z (id, value) entries in registers; unused slots hold (0, 0).
struct WfRow {
  int size;
  uint32_t id[WF_Z];
  float x[WF_Z];

  // entries [beg, end) of the CSR (beg == end: an empty row)
  __device__ __forceinline__ void load(const uint32_t* __restrict__ col, const float* __restrict__ val,
                                       uint64_t beg, uint64_t end) {
    size = (int)(end - beg);
#pragma unroll
    for (int j = 0; j < WF_Z; j++) {
      id[j] = 0;
      x[j] = 0.f;
      if (j < size) {
        id[j] = col[beg + j];
        x[j] = val[beg + j];
      }
    }
  }

  __device__ __forceinline__ bool names_a_feature_twice() const {
    bool dup = false;
#pragma unroll
    for (int j = 1; j < WF_Z; j++)
#pragma unroll
      for (int j2 = 0; j2 < j; j2++)
        if (j < size && id[j] == id[j2]) dup = true;
    return dup;
  }
};

// The window's conflict table: WF_HASH slots of shared memory.  Slot wf_hash(id) holds
// (seq << 5) | (31 - lane) of the lowest lane of window seq whose marked row has feature id
// (atomicMax: the larger tag is the later window, then the lower lane).
struct WfHash {
  unsigned int* slot;
  unsigned int seq;
  unsigned int tag;  // this lane's tag in the current window

  // clears the table; the caller synchronises the warp before the first window
  __device__ __forceinline__ WfHash(unsigned int* s, int lane) : slot(s), seq(0), tag(0) { clear(lane); }

  __device__ __forceinline__ void clear(int lane) {
    for (int i = lane; i < WF_HASH; i += 32) slot[i] = 0;
  }

  // every lane, once per window
  __device__ __forceinline__ void next_window(int lane) {
    if (++seq == (1u << 27)) {  // window counter about to leave its 27 bits: start over
      clear(lane);
      seq = 1;
      __syncwarp();
    }
    tag = (seq << 5) | (unsigned int)(31 - lane);
  }

  // every lane marks its row's features; returns when all marks are in
  __device__ __forceinline__ void mark(const WfRow& r) {
#pragma unroll
    for (int j = 0; j < WF_Z; j++)
      if (j < r.size) atomicMax(&slot[wf_hash(r.id[j])], tag);
    __syncwarp();
  }

  // an earlier lane's row has one of the features of r, this lane's marked row (whose slots
  // therefore hold tags of this window)
  __device__ __forceinline__ bool earlier_has(const WfRow& r, int lane) const {
    bool hit = false;
#pragma unroll
    for (int j = 0; j < WF_Z; j++)
      if (j < r.size) {
        const unsigned int h = slot[wf_hash(r.id[j])];
        if (31 - (int)(h & 31u) < lane) hit = true;
      }
    return hit;
  }

  // this lane's or an earlier lane's marked row has one of the features of r, an unmarked row
  __device__ __forceinline__ bool this_or_earlier_has(const WfRow& r, int lane) const {
    bool hit = false;
#pragma unroll
    for (int j = 0; j < WF_Z; j++)
      if (j < r.size) {
        const unsigned int h = slot[wf_hash(r.id[j])];
        if ((h >> 5) == seq && 31 - (int)(h & 31u) <= lane) hit = true;
      }
    return hit;
  }
};

// P, the window's conflict-free prefix: the lanes before the first whose stop is set (32 if none)
__device__ __forceinline__ int wf_prefix(bool stop) {
  const unsigned m = __ballot_sync(0xffffffffu, stop);
  return m ? __ffs(m) - 1 : 32;
}

// A row's w and V as the window's start left them, its score's addends, and the scatter of its
// updates.
struct WfGather {
  double wv[WF_Z], vv[WF_Z][WF_K], sum[WF_K];

  __device__ __forceinline__ void gather(const WfRow& r, const double* w, const double* v, int k, bool k1) {
#pragma unroll
    for (int j = 0; j < WF_Z; j++) {
      wv[j] = 0;
      if (j < r.size && k1) wv[j] = w[r.id[j]];
#pragma unroll
      for (int f = 0; f < WF_K; f++) {
        vv[j][f] = 0;
        if (j < r.size && f < k) vv[j][f] = v[(size_t)r.id[j] * k + f];
      }
    }
  }

  // add[WF_Z + WF_K] (fm_model.h:107-121): a_i = w_i x_i, then b_f = 0.5 (sum_f^2 - sumsq_f)
  // with sum_f = ((0 + d_0) + d_1) + ..., kept for the update.  Unused slots hold -0.0, the
  // exact identity of IEEE addition (x + -0.0 == x for every x, signed zeros included), so a
  // chain adds all WF_Z + WF_K of them without a select.
  __device__ __forceinline__ void addends(const WfRow& r, int k, bool k1, double* add) {
#pragma unroll
    for (int j = 0; j < WF_Z; j++) add[j] = (j < r.size && k1) ? wv[j] * (double)r.x[j] : -0.0;
#pragma unroll
    for (int f = 0; f < WF_K; f++) {
      double sf = 0, ss = 0;
#pragma unroll
      for (int j = 0; j < WF_Z; j++)
        if (j < r.size) {
          const double d = vv[j][f] * (double)r.x[j];
          sf += d;
          ss += d * d;
        }
      sum[f] = sf;
      add[WF_Z + f] = (f < k) ? 0.5 * (sf * sf - ss) : -0.0;
    }
  }

  // The row's updates in fm_sgd.h:38-50's order: the w entries, then V factor by factor.  The
  // rule maps the current value c to the new one: upd_w(j, at, c) for w[at], upd_v(j, f, at, c)
  // for v[at], at = id_j * k + f.  c is the gathered value, or, when the row names a feature
  // twice, re-read from memory so that the second update sees the first.
  template <class UpdW, class UpdV>
  __device__ __forceinline__ void scatter(const WfRow& r, bool dup, double* w, double* v, int k, bool k1,
                                          UpdW upd_w, UpdV upd_v) const {
    if (k1)
#pragma unroll
      for (int j = 0; j < WF_Z; j++)
        if (j < r.size) {
          double* c = &w[r.id[j]];
          *c = upd_w(j, r.id[j], dup ? *c : wv[j]);
        }
#pragma unroll
    for (int f = 0; f < WF_K; f++)
      if (f < k)
#pragma unroll
        for (int j = 0; j < WF_Z; j++)
          if (j < r.size) {
            const size_t at = (size_t)r.id[j] * k + f;
            double* c = &v[at];
            *c = upd_v(j, f, at, dup ? *c : vv[j][f]);
          }
  }
};

template <bool K0, int TASK>
__global__ void __launch_bounds__(32, 1)
    fm_sgd_inorder_wavefront_kernel(Params64 p, int n_factor, int use_w0, int use_w, HParams hp,
                                    uint64_t n_rows, const uint64_t* __restrict__ row_ptr,
                                    const uint32_t* __restrict__ col,
                                    const float* __restrict__ val,
                                    const float* __restrict__ target) {
  constexpr int NA = WF_Z + WF_K;  // addends per example
  __shared__ __align__(16) double s_add[32][NA];
  __shared__ float s_y[32];
  __shared__ unsigned int s_hash[WF_HASH];

  const int lane = threadIdx.x;
  const int k = n_factor;
  constexpr bool k0 = K0;
  const bool k1 = use_w != 0;
  double* w = p.w();
  double* v = p.v();
  double w0 = k0 ? *p.w0() : 0.0;
  const double lr = hp.lr, reg0 = hp.reg0, regw = hp.regw, regv = hp.regv;

  WfHash hash(s_hash, lane);
  __syncwarp();

  uint64_t base = 0;
  // Row bounds, targets and entries of the coming window are fetched one window ahead (the
  // loads are in flight while the chain of the current window runs).
  WfRow row;
  float yf = 0.f;
  {
    uint64_t beg = 0, end = 0;
    if (lane < n_rows) {
      beg = row_ptr[lane];
      end = row_ptr[lane + 1];
      yf = target[lane];
    }
    row.load(col, val, beg, end);
  }

  while (base < n_rows) {
    // (1) conflict-free prefix
    const bool valid = base + lane < n_rows;  // an invalid lane's row is empty
    double x[WF_Z];  // converted once per window: the scatter reads each value k + 1 times
#pragma unroll
    for (int j = 0; j < WF_Z; j++) x[j] = (double)row.x[j];
    const bool dup = row.names_a_feature_twice();
    hash.next_window(lane);
    hash.mark(row);
    const int P = wf_prefix(hash.earlier_has(row, lane) || !valid);  // >= 1: lane 0 is valid and never in conflict
    const bool active = lane < P;

    // (2) gather + addends
    WfGather gat;
    if (active) gat.gather(row, w, v, k, k1);
    // bounds of the next window's examples: in flight during the chain
    const uint64_t nr = base + P + lane;
    uint64_t nbeg = 0, nend = 0;
    float nyf = 0.f;
    if (nr < n_rows) {
      nbeg = row_ptr[nr];
      nend = row_ptr[nr + 1];
      nyf = target[nr];
    }
    if (active) {
      gat.addends(row, k, k1, s_add[lane]);
      s_y[lane] = yf;
    }
    __syncwarp();
    // entries of the next window's examples: in flight during the chain
    WfRow next;
    next.load(col, val, nbeg, nend);

    // (3) the bias chain, every lane redundantly
    double my_mult = 0;
    double cur[NA], nxt[NA];
#pragma unroll
    for (int a = 0; a < NA; a++) cur[a] = s_add[0][a];
    for (int t = 0; t < P; t++) {
      const int tn = (t + 1 < P) ? t + 1 : t;
#pragma unroll
      for (int a = 0; a < NA; a++) nxt[a] = s_add[tn][a];
      // No select sits in the dependent chain (unused addends are -0.0).  A model without
      // bias keeps the local w0 at +0.0, so 0.0 + w0 is the reference's `result = 0`.
      double pr = 0.0 + w0;
#pragma unroll
      for (int a = 0; a < NA; a++) pr += cur[a];
      const double mult = sgd_mult_select<TASK>(hp, pr, (double)s_y[t]);  // fm_learn_sgd_element.h:58-65
      if (k0) w0 -= lr * (mult + reg0 * w0);  // fm_sgd.h:34-37
      if (lane == t) my_mult = mult;
#pragma unroll
      for (int a = 0; a < NA; a++) cur[a] = nxt[a];
    }

    // (4) scatter: fm_sgd.h:38-50 for the lane's own example
    if (active)
      gat.scatter(
          row, dup, w, v, k, k1,
          [&](int j, uint32_t, double c) { return c - lr * (my_mult * x[j] + regw * c); },
          [&](int j, int f, size_t, double c) {
            const double grad = gat.sum[f] * x[j] - c * x[j] * x[j];
            return c - lr * (my_mult * grad + regv * c);
          });
    __syncwarp();  // the next window's gathers (other lanes) must see these stores
    base += P;
    row = next;
    yf = nyf;
  }
  if (lane == 0 && k0) *p.w0() = w0;
}

}  // namespace fmb
