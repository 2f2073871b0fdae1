// fm_mcmc.cu -- MCMC and ALS learning (reference libfm/src/fm_learn_mcmc.h and
// fm_learn_mcmc_simultaneous.h, data sets without relations), bit-identical to the reference.
//
// One iteration = draw_all (fm_learn_mcmc.h:430-641) + re-prediction + target step
// (fm_learn_mcmc_simultaneous.h:88-200).  Split:
//  - host: the libc rand() stream, the O(G k) hyperparameter draws, the O(N) serial case sums
//    (alpha, w0) and the train / test evaluation.  The host already holds the e-terms for the
//    evaluation anyway; whether one host core runs the 10 M-long dependent fp64 chains faster
//    than one device thread would is not measured.
//  - device: one cooperative kernel per iteration runs the e shift of draw_w0, the w sweep and,
//    per factor, the q rebuild and the v sweep, with grid barriers between phases.  The sweeps
//    walk the feature ids as maximal runs of consecutive ids no two of which share a training
//    case: within a run every draw reads exactly the cache values the sequential sweep gives
//    it, so a run's features are drawn in parallel (one warp each).  A warp gathers 32 entries
//    of its column at a time and adds their terms in column order, so each column sum is the
//    reference's serial chain.  The e-term re-prediction is fm_eterm64_kernel.
// Out of core (fmb200_mcmc_begin_xt): a data set given as blocks of its .xt file is streamed through two slots
// on every pass (xt_pass).  Column sums lie inside one column, so inside one block, and draw_feature runs as
// it is on the block's columns.  Per-case chains (the q rebuild, the three e-term parts, the begin-time prev
// index) cross blocks: each case accumulates block by block in file order and, inside a block, in column
// order, through the block's entries stably sorted by case (xt_case_kernel).  Runs are cut at every block
// start besides the resident cut.  Passes per iteration: train 1 + k sweeps (the q of factor f + 1 is rebuilt
// on the pass that sweeps f, into the second q) and k + k1 e-term passes; test k + k1 e-term passes.
// Each draw needs one standard normal; the host draws them in the reference's order before the
// launch.  A sampled draw the reference would skip without consuming one (posterior variance
// not finite, or stdev 0) cannot arise from a finite state; the device flags it and the
// iteration fails instead of desynchronising the stream.
// This TU is compiled with --fmad=false: every product and sum rounds as the reference's do.
#include <cooperative_groups.h>
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <climits>
#include <cmath>
#include <vector>

#include "fm_roworder.cuh"
#include "fmb200_internal.h"
#include "ref_random.h"

namespace cg = cooperative_groups;

namespace fmb {

using namespace ref_random;

// hyperpriors, fm_learn_mcmc.h:1107-1114
constexpr double kAlpha0 = 1.0, kGamma0 = 1.0, kBeta0 = 1.0, kMu0 = 0.0, kW0Mean0 = 0.0;

// device flag words
enum { F_NAN_W = 0, F_INF_W, F_NAN_V, F_INF_V, F_SKIP, F_WORDS = 8 };

// The CTA that sweeps narrow runs (mcmc_cta_sweep_kernel): kCtaSweepThreads threads by default, any multiple of 32
// up to kCtaSweepMaxThreads through fmb200_set_tuning's threads; a run is narrow when it has at most as many
// features as that CTA has warps (DESIGN §3.8)
constexpr int kCtaSweepThreads = 256, kCtaSweepMaxThreads = 1024;

// A stretch of consecutive runs [r_lo, r_hi) of one segment, swept by one launch: one CTA when they are all narrow,
// the cooperative grid otherwise
struct Stretch {
  uint32_t r_lo, r_hi;
  bool narrow;
};

// A data set streamed from blocks of its .xt (fmb200_mcmc_begin_xt)
struct XtSet {
  fmb200_xt_blocks src{};
  std::vector<uint32_t> col_lo;  // [n_blocks + 1]
  std::vector<uint64_t> nnz;     // [n_blocks]
  uint64_t n_blocks() const { return nnz.size(); }
};

// One relation block on the device, as the kernels see it
struct RelView {
  uint32_t rows;
  const uint64_t* col_ptr;  // the block's .xt: column j - attr_offset at [col_ptr[j - attr_offset], ...)
  const uint32_t* xt_row;
  const float* xt_val;
  const uint64_t* row_ptr;  // its row-major copy: each row's entries in (model id, position) order
  const uint32_t* col;
  const float* val;
  const uint32_t* join[2];  // train, test case -> row
  const uint64_t* inv_ptr;  // row -> its train cases, ascending: inv_case[inv_ptr[row] .. inv_ptr[row + 1])
  const uint32_t* inv_case;
  // relation_cache (fm_learn_mcmc.h:51-59) field by field; qf[row][k]: the q_f of the last e-term pass
  double *wnum, *we, *weq, *wc, *wc_sqr, *y, *q, *qf;
};

// The columns a sweep draws from: column j's positions are [col_ptr[j - lo], col_ptr[j - lo + 1]) for j < hi, and
// the columns from hi on are empty (a streamed block and the features after the .xt)
struct Cols {
  const uint64_t* col_ptr;
  uint32_t lo, hi;
  const uint32_t* cs_case;
  const float* cs_x;
};

struct RelDev {
  uint32_t rows = 0, nf = 0, off = 0;
  DevPtr<uint64_t> col_ptr, row_ptr, inv_ptr;
  DevPtr<uint32_t> xt_row, col, join[2], inv_case;
  DevPtr<float> xt_val, val;
  DevPtr<double> cache;  // wnum | we | weq | wc | wc_sqr | y | q, [rows] each, then qf [rows][k]
  RelView view() const {
    double* p = cache.get();
    const size_t r = rows;
    return RelView{rows, col_ptr.get(), xt_row.get(), xt_val.get(), row_ptr.get(), col.get(), val.get(),
                   {join[0].get(), join[1].get()}, inv_ptr.get(), inv_case.get(),
                   p, p + r, p + 2 * r, p + 3 * r, p + 4 * r, p + 5 * r, p + 6 * r, p + 7 * r};
  }
  Cols cols() const { return Cols{col_ptr.get(), off, off + nf, xt_row.get(), xt_val.get()}; }
};

// The scratch of sort_by_key: iota = 0, 1, ... (the positions the sort carries) and CUB's temporary storage
struct SortScratch {
  DevPtr<uint32_t> iota;
  DevPtr<unsigned char> tmp;
  size_t tmp_bytes = 0;
};

// The train or the test set
struct McmcSet {
  int slot = 0;
  std::unique_ptr<XtSet> xt;  // null when the set is resident in its slot
  uint64_t n = 0, gen = 0;    // cases; the slot's upload generation (resident)
  std::vector<float> y;
  std::vector<double> e;
  DevPtr<double> e_d;
  const float* y_dev = nullptr;  // train: the targets on the device (the slot's, or y_d when streamed)
  DevPtr<float> y_d;
  // the two per-case chains of the streamed e-term passes; the train set's are the sweep's q (also resident) and
  // the second q
  DevPtr<double> chain[2];
};

struct McmcState {
  McmcSet set[2];  // train, test
  bool sample = true, multilevel = true;
  uint32_t G = 1;
  std::vector<uint32_t> group, per_group;  // attr_group[n], num_attr_per_group[G]
  double alpha = 1.0, reg0 = 0.0;
  std::vector<double> w_mu, w_lambda, v_mu, v_lambda;  // [G], [G][k]
  std::vector<double> pred_this, pred_all, pred_but5;
  std::vector<double> state;  // host image of the fp64 state (Params64 layout)
  std::vector<double> z, hyp;
  std::vector<uint32_t> runs;  // run starts, then n
  // The id space in segments, each swept by its own launches: a streamed training set's blocks, or the main table
  // and then each relation block.  Segment i sweeps the runs [seg_run[i], seg_run[i + 1]).
  std::vector<uint32_t> seg_run;
  // the launch plan: segment i's runs as maximal stretches of narrow and of wide runs, in order (plan_sweeps)
  std::vector<std::vector<Stretch>> plan;
  int cta_threads = kCtaSweepThreads;
  uint32_t iter = 0;
  uint32_t counters[16] = {0};
  // device
  DevPtr<uint64_t> col_ptr;
  DevPtr<uint32_t> cs_case, dup, group_d, runs_d;
  DevPtr<float> cs_x;
  DevPtr<double> z_d, hyp_d;
  DevPtr<unsigned int> flag_d;
  int grid = 0;
  // streamed sets: a block's entries stably sorted by case (the case ids and the entries' positions in the block)
  DevPtr<uint32_t> srt_key, srt_pos;
  SortScratch srt;
  std::vector<RelDev> rel;  // relation blocks (fmb200_mcmc_set_relations)
  DevPtr<RelView> rel_d;
};

void McmcDelete::operator()(McmcState* s) const { delete s; }

namespace {

// ---- device: index build -------------------------------------------------------------------
// prev[j] = 1 + the largest id below j that shares a case with j (0: none); one thread per case
__global__ void mcmc_prev_kernel(const uint64_t* __restrict__ rp, const uint32_t* __restrict__ col, uint64_t n_rows,
                                 unsigned int* prev) {
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rows; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t b = rp[r], e = rp[r + 1];
    for (uint64_t i = b; i < e; i++) {
      const uint32_t j = col[i];
      unsigned int best = 0;
      for (uint64_t t = b; t < e; t++)
        if (col[t] < j) best = max(best, col[t] + 1u);
      if (best) atomicMax(prev + j, best);
    }
  }
}

// the transposed training data from the stable (id, entry) sort: case and value of every
// position; dup[j] = 1 when column j names a case twice (its entries are then adjacent)
__global__ void mcmc_csc_kernel(const uint32_t* __restrict__ ids, const uint32_t* __restrict__ ent, uint64_t nnz,
                                const uint64_t* __restrict__ rp, uint64_t n_rows, const float* __restrict__ val,
                                uint32_t* cs_case, float* cs_x, uint32_t* dup) {
  for (uint64_t p = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; p < nnz; p += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t r = (uint32_t)row_of(rp, n_rows, ent[p]);
    cs_case[p] = r;
    cs_x[p] = val[ent[p]];
    if (p > 0 && ids[p - 1] == ids[p] && (uint32_t)row_of(rp, n_rows, ent[p - 1]) == r) dup[ids[p]] = 1u;
  }
}

__global__ void mcmc_colptr_kernel(const uint32_t* __restrict__ ids, uint64_t nnz, uint32_t n, uint64_t* col_ptr) {
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j <= n; j += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t lo = 0, hi = nnz;  // first position with id >= j
    while (lo < hi) {
      const uint64_t mid = (lo + hi) >> 1;
      if (ids[mid] < j) lo = mid + 1;
      else hi = mid;
    }
    col_ptr[j] = lo;
  }
}

__global__ void mcmc_residual_kernel(double* e, const float* __restrict__ y, uint64_t n) {
  for (uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; c < n; c += (uint64_t)gridDim.x * blockDim.x)
    e[c] = e[c] - y[c];
}

// ---- device: the sweep -----------------------------------------------------------------------
struct SweepArgs {
  Cols cols;
  const uint32_t* dup;
  const uint32_t* group;
  const uint32_t* runs;
  uint32_t n_runs, n, G;
  const uint64_t* row_ptr;
  const uint32_t* col;
  const float* val;
  uint64_t n_rows;
  double* e;
  double* q;
  double* w;
  double* v;
  int k, use_w, sample, shift;
  double alpha, e_shift;
  const double* z;    // [n] for w, then [k][n] for v
  const double* hyp;  // w_mu[G] | w_lambda[G] | v_mu[G][k] | v_lambda[G][k]
  unsigned int* flag;
  RelView rel;  // the sweep of a relation block (REL): its rows play the cases, q is the rows' q
};

// draw_w (fm_learn_mcmc.h:685-732) / draw_v (:792-847) of feature j, one warp; with REL draw_w_rel (:734-790) /
// draw_v_rel (:849-935) of a relation block's feature
template <bool V, bool REL = false>
__device__ void draw_feature(const SweepArgs& a, uint32_t j, int f, int lane) {
  const uint32_t g = a.group[j];
  double mu, lam, zz;
  double* par;
  if (V) {
    mu = a.hyp[2 * a.G + (size_t)g * a.k + f];
    lam = a.hyp[2 * a.G + (size_t)a.G * a.k + (size_t)g * a.k + f];
    par = a.v + (size_t)j * a.k + f;
    zz = a.sample ? a.z[a.n + (size_t)f * a.n + j] : 0.0;
  } else {
    mu = a.hyp[g];
    lam = a.hyp[a.G + g];
    par = a.w + j;
    zz = a.sample ? a.z[j] : 0.0;
  }
  const double old = *par;
  uint32_t beg = 0, end = 0;
  if (j < a.cols.hi) {
    beg = (uint32_t)a.cols.col_ptr[j - a.cols.lo];
    end = (uint32_t)a.cols.col_ptr[j - a.cols.lo + 1];
  }
  double m = 0.0, s = 0.0;
  for (uint32_t b = beg; b < end; b += 32) {
    const uint32_t idx = b + lane;
    double tm = 0.0, ts = 0.0;
    if (idx < end) {
      const uint32_t c = a.cols.cs_case[idx];
      const float x = a.cols.cs_x[idx];
      const double xd = (double)x;
      if (REL) {
        if (V) {
          const double h = xd * (a.q[c] - xd * old);
          tm = h * a.rel.we[c] + xd * a.rel.weq[c];
          ts = h * h * a.rel.wnum[c] + 2 * a.rel.wc[c] * xd * h + (double)(x * x) * a.rel.wc_sqr[c];
        } else {
          tm = xd * a.rel.we[c];
          ts = (double)(x * x) * a.rel.wnum[c];
        }
      } else if (V) {
        const double h = xd * (a.q[c] - xd * old);
        tm = h * a.e[c];
        ts = h * h;
      } else {
        tm = xd * (a.e[c] - old * xd);
        ts = (double)(x * x);  // FM_FLOAT product, widened by the += (fm_learn_mcmc.h:692)
      }
    }
    const uint32_t cnt = min(32u, end - b);
    for (uint32_t i = 0; i < cnt; i++) {  // column order: the reference's serial chain
      m += __shfl_sync(0xffffffffu, tm, i);
      s += __shfl_sync(0xffffffffu, ts, i);
    }
  }
  if (V || REL) m -= old * s;
  const double sig = 1.0 / (lam + a.alpha * s);
  const double mean = -sig * (a.alpha * m - mu * lam);
  double nv;
  bool skipped = false;
  if (isnan(sig) || isinf(sig)) {
    nv = 0.0;
    skipped = a.sample != 0;
  } else if (a.sample) {
    const double sd = sqrt(sig);
    if (sd == 0.0 || isnan(sd)) {
      nv = mean;
      skipped = true;
    } else {
      nv = mean + sd * zz;
    }
  } else {
    nv = mean;
  }
  if (skipped && lane == 0) atomicMin(a.flag + F_SKIP, V ? 1u + (unsigned)f : 0u);
  if (isnan(nv)) {
    if (lane == 0) atomicAdd(a.flag + (V ? F_NAN_V : F_NAN_W), 1u);
    return;
  }
  if (isinf(nv)) {
    if (lane == 0) atomicAdd(a.flag + (V ? F_INF_V : F_INF_W), 1u);
    return;
  }
  if (lane == 0) *par = nv;
  const double d = old - nv;
  // a column that names a case twice updates serially: the second entry reads the q the first left
  const bool serial = a.dup[j] != 0;
  if (serial && lane != 0) return;
  for (uint32_t idx = beg + (serial ? 0 : lane); idx < end; idx += serial ? 1 : 32) {
    const uint32_t c = a.cols.cs_case[idx];
    const double xd = (double)a.cols.cs_x[idx];
    if (REL) {
      if (V) {
        const double h = xd * (a.q[c] - xd * old);
        a.rel.we[c] -= d * (h * a.rel.wnum[c] + xd * a.rel.wc[c]);
        a.q[c] -= d * xd;
        a.rel.weq[c] -= d * (h * a.rel.wc[c] + xd * a.rel.wc_sqr[c]);
        a.rel.y[c] += (nv - old) * h;
      } else {
        a.rel.we[c] -= xd * d * a.rel.wnum[c];
        a.rel.y[c] += (nv - old) * xd;
      }
    } else if (V) {
      const double h = xd * (a.q[c] - xd * old);
      a.q[c] -= xd * d;
      a.e[c] -= h * d;
    } else {
      a.e[c] -= xd * d;
    }
  }
}

// runs [r_lo, r_hi), sync() after each: a grid barrier, or a CTA barrier when one CTA sweeps them
template <bool V, bool REL = false, class Sync>
__device__ void sweep_runs(const SweepArgs& a, Sync sync, int f, uint32_t r_lo, uint32_t r_hi, uint32_t warp,
                           uint32_t nwarp, int lane) {
  for (uint32_t r = r_lo; r < r_hi; r++) {
    const uint32_t j1 = a.runs[r + 1];
    for (uint32_t j = a.runs[r] + warp; j < j1; j += nwarp) draw_feature<V, REL>(a, j, f, lane);
    sync();
  }
}

// q_f of case c from its row (add_main_q, :406-428)
__device__ __forceinline__ double main_q(const SweepArgs& a, uint64_t c, int f) {
  const uint64_t beg = a.row_ptr[c];
  RowOrder o;
  o.init(a.col + beg, (uint32_t)(a.row_ptr[c + 1] - beg));
  return row_q(o, a.v, a.k, f, a.val + beg);
}

__global__ void __launch_bounds__(256) mcmc_sweep_kernel(const SweepArgs a) {
  cg::grid_group grid = cg::this_grid();
  const uint64_t tid = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint64_t nth = (uint64_t)gridDim.x * blockDim.x;
  const uint32_t warp = (uint32_t)(tid >> 5), nwarp = (uint32_t)(nth >> 5);
  const int lane = threadIdx.x & 31;
  if (a.shift) {  // draw_w0's update of e (fm_learn_mcmc.h:680-682)
    for (uint64_t c = tid; c < a.n_rows; c += nth) a.e[c] -= a.e_shift;
    grid.sync();
  }
  auto sync = [&] { grid.sync(); };
  if (a.use_w) sweep_runs<false>(a, sync, 0, 0, a.n_runs, warp, nwarp, lane);
  for (int f = 0; f < a.k; f++) {
    for (uint64_t c = tid; c < a.n_rows; c += nth) a.q[c] = main_q(a, c, f);  // the q rebuild
    grid.sync();
    sweep_runs<true>(a, sync, f, 0, a.n_runs, warp, nwarp, lane);
  }
}

// ---- device: the streamed passes ---------------------------------------------------------------
// the sweep of w (V = false) or of factor f over the runs [r_lo, r_hi) of one block; with REL, of a relation block
template <bool V, bool REL = false>
__global__ void __launch_bounds__(256) mcmc_block_sweep_kernel(const SweepArgs a, uint32_t r_lo, uint32_t r_hi, int f) {
  cg::grid_group grid = cg::this_grid();
  const uint64_t tid = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint64_t nth = (uint64_t)gridDim.x * blockDim.x;
  sweep_runs<V, REL>(a, [&] { grid.sync(); }, f, r_lo, r_hi, (uint32_t)(tid >> 5), (uint32_t)(nth >> 5),
                     threadIdx.x & 31);
}

// The same sweep over narrow runs (no wider than the CTA has warps), by one CTA launched normally: a run's features
// get a warp each, as in the grid, and __syncthreads() between runs stands for the grid barrier.  It orders and
// makes visible every global write of the CTA's threads before the next run's reads, so each draw reads what it
// reads in mcmc_block_sweep_kernel and the results are the same bits.  (One CTA per launch: the bound's 1 lets
// ptxas use up to 64 registers, and it spills none.)
template <bool V, bool REL = false>
__global__ void __launch_bounds__(kCtaSweepMaxThreads, 1) mcmc_cta_sweep_kernel(const SweepArgs a, uint32_t r_lo,
                                                                               uint32_t r_hi, int f) {
  sweep_runs<V, REL>(a, [] { __syncthreads(); }, f, r_lo, r_hi, threadIdx.x >> 5, blockDim.x >> 5, threadIdx.x & 31);
}

// What a case adds from one block, in column order (the block's entries stably sorted by case):
//   CH_Q        q[c] += v[j][f] x                           the q rebuild (add_main_q, fm_learn_mcmc.h:406-428)
//   CH_ETERM_V  q[c] += v[j][f] x;  q2[c] -= 0.5 v^2 x^2    e-term parts (1) and (2) of factor f (:172-306)
//   CH_ETERM_W  q2[c] += w[j] x                             e-term part (3) (:309-346)
//   CH_PREV     prev[j] := max(prev[j], 1 + the largest id below j the case names, in this block or before
//               it: last[c]); dup[j] := 1 when the case is named twice by column j; last[c] := 1 + its last id
// Every sum is the one fm_eterm64_kernel / row_q form for the case, in the same order (--fmad=false).
enum { CH_Q = 0, CH_ETERM_V, CH_ETERM_W, CH_PREV };
struct ChainArgs {
  const uint32_t* key;      // the entries' cases, sorted
  const uint32_t* pos;      // the entries' positions in the block, in that order
  uint64_t nnz;
  const uint64_t* col_ptr;  // the block's column offsets
  uint64_t n_cols;
  uint32_t col_lo;          // the block's first column
  const float* val;
  const double* v;
  const double* w;
  int k, f;
  double* q;
  double* q2;
  uint32_t* last;
  unsigned int* prev;
  uint32_t* dup;
};

template <int OP>
__global__ void xt_case_kernel(const ChainArgs a) {
  for (uint64_t p = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; p < a.nnz; p += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t c = a.key[p];
    if (p > 0 && a.key[p - 1] == c) continue;  // one thread per case: the one at its first entry
    double q = 0.0, q2 = 0.0;
    if (OP == CH_Q || OP == CH_ETERM_V) q = a.q[c];
    if (OP == CH_ETERM_V || OP == CH_ETERM_W) q2 = a.q2[c];
    uint32_t below = 0, cur = 0xffffffffu;
    if (OP == CH_PREV) below = a.last[c];
    for (uint64_t i = p; i < a.nnz && a.key[i] == c; i++) {
      const uint32_t e = a.pos[i];
      const uint32_t j = a.col_lo + (uint32_t)row_of(a.col_ptr, a.n_cols, e);
      if (OP == CH_Q) q += a.v[(size_t)j * a.k + a.f] * (double)a.val[e];
      if (OP == CH_ETERM_V) {
        const double vif = a.v[(size_t)j * a.k + a.f];
        const float xi = a.val[e];
        q += vif * (double)xi;
        q2 -= 0.5 * vif * vif * xi * xi;
      }
      if (OP == CH_ETERM_W) q2 += a.w[j] * (double)a.val[e];
      if (OP == CH_PREV) {
        if (j == cur) {
          a.dup[j] = 1u;
        } else {
          if (cur != 0xffffffffu) below = cur + 1;
          cur = j;
        }
        if (below) atomicMax(a.prev + j, below);
      }
    }
    if (OP == CH_Q || OP == CH_ETERM_V) a.q[c] = q;
    if (OP == CH_ETERM_V || OP == CH_ETERM_W) a.q2[c] = q2;
    if (OP == CH_PREV) a.last[c] = cur + 1;
  }
}

// after the e-term pass of a factor: e += 0.5 q^2 (:250), and q restarts at 0 for the next factor
__global__ void eterm_factor_kernel(double* e, double* q, uint64_t n) {
  for (uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; c < n; c += (uint64_t)gridDim.x * blockDim.x) {
    const double qc = q[c];
    e[c] += 0.5 * qc * qc;
    q[c] = 0.0;
  }
}

// e = (e + q2) + w0 (:350-362)
__global__ void eterm_final_kernel(double* e, const double* q2, uint64_t n, int use_w0, const double* w0) {
  for (uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; c < n; c += (uint64_t)gridDim.x * blockDim.x) {
    double x = e[c];
    x = x + q2[c];
    if (use_w0) x += *w0;
    e[c] = x;
  }
}

// draw_w0's update of e (:680-682)
__global__ void mcmc_shift_kernel(double* e, uint64_t n, double e_shift) {
  for (uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; c < n; c += (uint64_t)gridDim.x * blockDim.x)
    e[c] -= e_shift;
}

__global__ void iota_kernel(uint32_t* x, uint64_t n) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    x[i] = (uint32_t)i;
}

// ---- device: relation blocks (fm_learn_mcmc.h, the relational parts) ------------------------------------------
// The row-major copy of a block from the by-row stable sort of its .xt entries (pos = their positions): every
// row's entries in ascending model id, a repeated id in file order, which is the order in which the reference's
// walks over the .xt reach a row.  dup[j] = 1 when column j names a row twice.
__global__ void rel_rowmajor_kernel(const uint32_t* __restrict__ pos, uint64_t nnz, const uint64_t* __restrict__ col_ptr,
                                    uint32_t nf, uint32_t off, const float* __restrict__ xt_val, uint32_t* col, float* val) {
  for (uint64_t p = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; p < nnz; p += (uint64_t)gridDim.x * blockDim.x) {
    col[p] = off + (uint32_t)row_of(col_ptr, nf, pos[p]);
    val[p] = xt_val[pos[p]];
  }
}

__global__ void rel_dup_kernel(const uint64_t* __restrict__ row_ptr, const uint32_t* __restrict__ col, uint32_t rows,
                               uint32_t* dup) {
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < rows; r += (uint64_t)gridDim.x * blockDim.x)
    for (uint64_t i = row_ptr[r] + 1; i < row_ptr[r + 1]; i++)
      if (col[i] == col[i - 1]) dup[col[i]] = 1u;
}

// #^R: the train cases that join each row (:1183-1188), a count of 1.0 steps
__global__ void rel_wnum_kernel(const RelView r) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < r.rows; i += (uint64_t)gridDim.x * blockDim.x)
    r.wnum[i] = (double)(r.inv_ptr[i + 1] - r.inv_ptr[i]);
}

// Per row, one thread.  REL_Q: q = q_f of the row (:538-562).  REL_ETERM: the block's part of the e-term pass
// (:148-378): qf[row][f] = q_f, q = its parts (2) and (3), y = sum_f 0.5 q_f^2 + q.
enum { REL_Q = 0, REL_ETERM };
template <int OP>
__global__ void rel_row_kernel(const RelView r, const double* __restrict__ v, const double* __restrict__ w, int k, int f,
                               int use_w) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < r.rows; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t beg = r.row_ptr[i];
    RowOrder o;
    o.init(r.col + beg, (uint32_t)(r.row_ptr[i + 1] - beg));
    if (OP == REL_Q) {
      r.q[i] = row_q(o, v, k, f, r.val + beg);
    } else {
      r.y[i] = case_eterm(o, v, w, k, use_w, 0, 0.0, r.val + beg, [&](int g, double& q) { r.qf[i * k + g] = q; },
                          [&](double& q) { r.q[i] = q; });
    }
  }
}

// Per row, one thread, over its train cases in ascending order: the reference's loop over all cases restricted
// to the cases of one row (each case joins one row).  W: :482-487; V: :603-616.
template <bool V>
__global__ void rel_unsync_kernel(const RelView r, double* e, double* q) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < r.rows; i += (uint64_t)gridDim.x * blockDim.x) {
    const double y = r.y[i], rq = V ? r.q[i] : 0.0;
    double we = 0.0, weq = 0.0, wc = 0.0, wc_sqr = 0.0;
    for (uint64_t t = r.inv_ptr[i]; t < r.inv_ptr[i + 1]; t++) {
      const uint32_t c = r.inv_case[t];
      if (V) {
        q[c] -= rq;  // main q out of sync
        we += e[c];
        weq += (e[c] * q[c]);
        wc += q[c];
        wc_sqr += (q[c] * q[c]);
        e[c] -= (y + q[c] * rq);  // main e out of sync
      } else {
        we += e[c];
        e[c] -= y;
      }
    }
    r.we[i] = we;
    if (V) {
      r.weq[i] = weq;
      r.wc[i] = wc;
      r.wc_sqr[i] = wc_sqr;
    }
  }
}

// Per case: the resync after a block's sweep.  W: :505-507; V: :634-637.
template <bool V>
__global__ void rel_resync_kernel(const RelView r, double* e, double* q, uint64_t n) {
  for (uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; c < n; c += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = r.join[0][c];
    if (V) {
      e[c] += (r.y[i] + q[c] * r.q[i]);
      q[c] += r.q[i];
    } else {
      e[c] += r.y[i];
    }
  }
}

// Per case: q_f = its own row's q_f (add_main_q) + the blocks' q_f of its rows in relation order (:565-570)
__global__ void rel_case_q_kernel(const SweepArgs a, int f, const RelView* __restrict__ rel, uint32_t n_rel) {
  for (uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; c < a.n_rows; c += (uint64_t)gridDim.x * blockDim.x) {
    double q = main_q(a, c, f);
    for (uint32_t r = 0; r < n_rel; r++) q += rel[r].q[rel[r].join[0][c]];
    a.q[c] = q;
  }
}

// The e-term pass (fm_learn_mcmc.h:148-378): the learner re-predicts every case once per iteration through the
// TRANSPOSED copy of the data, so each case accumulates its terms in ascending feature id (ties in row order) and in
// a different association than fm_model::predict:
//   e = sum_f 0.5 q_f^2 ;  q = sum_f sum_i -0.5 v_if^2 x_i^2  (+ sum_i w_i x_i) ;  e = (e + q) + w0
// One thread per case, every operation in that order (this TU is compiled with --fmad=false): bit-identical
// e-terms.  RowOrder (fm_roworder.cuh) gives that order for unsorted rows.  REL: the relation blocks' q_f and q of
// the case's rows (join `side`) are added in relation order (:227-240, :352-368).
template <bool REL>
__global__ void __launch_bounds__(128)
    fm_eterm64_kernel(Params64 p, int k, int use_w0, int use_w, uint64_t n_rows, const uint64_t* __restrict__ row_ptr,
                      const uint32_t* __restrict__ col, const float* __restrict__ val, double* __restrict__ e_out,
                      const RelView* __restrict__ rel, uint32_t n_rel, int side) {
  const double* w = p.w();
  const double* v = p.v();
  const double w0 = *p.w0();
  for (uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; c < n_rows; c += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t beg = row_ptr[c];
    RowOrder o;
    o.init(col + beg, (uint32_t)(row_ptr[c + 1] - beg));
    e_out[c] = case_eterm(
        o, v, w, k, use_w, use_w0, w0, val + beg,
        [&](int f, double& q) {
          if (REL)
            for (uint32_t r = 0; r < n_rel; r++) q += rel[r].qf[(size_t)rel[r].join[side][c] * k + f];
        },
        [&](double& q) {
          if (REL)
            for (uint32_t r = 0; r < n_rel; r++) q += rel[r].q[rel[r].join[side][c]];
        });
  }
}

}  // namespace

cudaError_t launch_mcmc_eterms(fmb200_ctx* c, const DataSlot& d, double* e_out, const RelView* rel, uint32_t n_rel,
                               int side) {
  if (d.n_rows == 0) return cudaSuccess;
  // one thread per case, blocks of 128, at most 16 blocks per SM
  const int grid = (int)std::min<uint64_t>((d.n_rows + 127) / 128, (uint64_t)c->sm_count * 16);
  auto kernel = rel ? fm_eterm64_kernel<true> : fm_eterm64_kernel<false>;
  kernel<<<grid, 128, 0, c->stream>>>(c->p64, c->k, c->k0, c->k1, d.n_rows, d.row_ptr.get(), d.col.get(), d.val.get(),
                                      e_out, rel, n_rel, side);
  c->launches++;
  return cudaGetLastError();
}

// ---- host: the learner -------------------------------------------------------------------------
#define MK(expr)                                            \
  do {                                                      \
    cudaError_t e__ = (expr);                               \
    if (e__ != cudaSuccess) return std::string(#expr " failed: ") + cudaGetErrorString(e__); \
  } while (0)

namespace {

// ---- streamed sets -----------------------------------------------------------------------------
// One pass over a streamed set in file order: use(slot, b) once per block, in order.  Block b is fetched and
// goes to slot src.slot[b % 2] on the copy stream, so the copy of block b + 1 runs while the work use()
// enqueued on block b does; before block b + 1 overwrites block b - 1's slot, the work on b - 1 has run.
template <class F>
std::string xt_pass(fmb200_ctx* c, XtSet& x, F use) {
  const uint64_t nb = x.n_blocks();
  auto slot = [&](uint64_t b) { return x.src.slot[b % 2]; };
  auto upload = [&](uint64_t b) -> std::string {
    const void* words = nullptr;
    const uint32_t* sizes = nullptr;
    if (x.src.fetch(x.src.user, b, &words, &sizes) != 0) return "fetching block " + std::to_string(b) + " of the .xt failed";
    if (upload_xt_enqueue(c, slot(b), x.col_lo[b + 1] - x.col_lo[b], x.nnz[b], words, sizes, c->copy_stream))
      return fmb200_last_error();
    return "";
  };
  MK(cudaStreamSynchronize(c->stream));  // the slots may hold blocks the previous pass still works on
  std::string err = upload(0);
  for (uint64_t b = 0; err.empty() && b < nb; b++) {
    if (b + 1 < nb) {
      if (b > 0) MK(cudaStreamSynchronize(c->stream));
      err = upload(b + 1);
      if (!err.empty()) break;
    }
    if (upload_xt_finish(c, slot(b), x.col_lo[b], x.src.n_cases)) {
      err = fmb200_last_error();
      break;
    }
    x.src.release(x.src.user, b);  // its copy has finished
    err = use(slot(b), b);
  }
  if (!err.empty()) cudaStreamSynchronize(c->copy_stream);  // no copy may still read a fetched block
  return err;
}

// d := a device copy of h[n], on c->stream
template <class T>
cudaError_t to_device(fmb200_ctx* c, DevPtr<T>& d, const T* h, uint64_t n) {
  const cudaError_t e = alloc(d, n);
  return e != cudaSuccess ? e : cudaMemcpyAsync(d.get(), h, n * sizeof(T), cudaMemcpyHostToDevice, c->stream);
}

int key_bits(uint64_t n_keys) {
  int bits = 1;
  while (bits < 32 && ((n_keys - 1) >> bits) != 0) bits++;
  return bits;
}

// The scratch of sort_by_key for n keys below n_keys
std::string sort_scratch(fmb200_ctx* c, uint64_t n, uint64_t n_keys, SortScratch& sc) {
  MK(alloc(sc.iota, n));
  if (n > 0) MK(launch_for(c, n, iota_kernel, sc.iota.get(), n));
  MK(cub::DeviceRadixSort::SortPairs(nullptr, sc.tmp_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                     (const uint32_t*)nullptr, (uint32_t*)nullptr, n, 0, key_bits(n_keys), c->stream));
  MK(alloc(sc.tmp, sc.tmp_bytes));
  return "";
}

// keys[n] (all below n_keys) stably sorted into key_out, and the positions they came from into pos_out; sc is a
// sort_scratch for at least n keys below at least n_keys
cudaError_t sort_by_key(fmb200_ctx* c, const SortScratch& sc, const uint32_t* keys, uint64_t n, uint64_t n_keys,
                        uint32_t* key_out, uint32_t* pos_out) {
  size_t tmp = sc.tmp_bytes;
  c->launches++;
  return cub::DeviceRadixSort::SortPairs(sc.tmp.get(), tmp, keys, key_out, sc.iota.get(), pos_out, n, 0,
                                         key_bits(n_keys), c->stream);
}

// sort_by_key with outputs and scratch of its own (the begin-time sorts); the scratch is freed on return
std::string sort_once(fmb200_ctx* c, const uint32_t* keys, uint64_t n, uint64_t n_keys, DevPtr<uint32_t>& key_out,
                      DevPtr<uint32_t>& pos_out) {
  MK(alloc(key_out, n));
  MK(alloc(pos_out, n));
  SortScratch sc;
  const std::string err = sort_scratch(c, n, n_keys, sc);
  if (!err.empty()) return err;
  if (n > 0) MK(sort_by_key(c, sc, keys, n, n_keys, key_out.get(), pos_out.get()));
  MK(cudaStreamSynchronize(c->stream));
  return "";
}

// Chain OP (xt_case_kernel) over the block in d, whose entries are first sorted by case, stably (s.srt_key: their
// cases, s.srt_pos: their positions).  a holds the chain's own arguments: f, q and q2, or last, prev and dup.
template <int OP>
std::string case_chain(fmb200_ctx* c, McmcState& s, const DataSlot& d, uint64_t n_cases, uint32_t col_lo, ChainArgs a) {
  MK(sort_by_key(c, s.srt, d.col.get(), d.nnz, n_cases, s.srt_key.get(), s.srt_pos.get()));
  a.key = s.srt_key.get();
  a.pos = s.srt_pos.get();
  a.nnz = d.nnz;
  a.col_ptr = d.row_ptr.get();
  a.n_cols = d.n_rows;
  a.col_lo = col_lo;
  a.val = d.val.get();
  a.v = c->p64.v();
  a.w = c->p64.w();
  a.k = c->k;
  MK(launch_for(c, a.nnz, xt_case_kernel<OP>, a));
  return "";
}

// The e-terms of a streamed set into its e_d (fm_eterm64_kernel's sums, case by case in the same order): one pass
// per factor for parts (1) and (2), one for part (3), through the set's two per-case chains
std::string xt_eterms(fmb200_ctx* c, McmcState& s, McmcSet& t) {
  XtSet& x = *t.xt;
  const uint64_t n = t.n;
  double *e = t.e_d.get(), *acc = t.chain[0].get(), *acc2 = t.chain[1].get();
  if (n == 0) return "";
  MK(cudaMemsetAsync(e, 0, n * sizeof(double), c->stream));
  MK(cudaMemsetAsync(acc, 0, n * sizeof(double), c->stream));
  MK(cudaMemsetAsync(acc2, 0, n * sizeof(double), c->stream));
  for (int f = 0; f <= c->k; f++) {
    if (f == c->k && !c->k1) break;
    const std::string err = xt_pass(c, x, [&](int slot, uint64_t b) -> std::string {
      const DataSlot& d = c->slots[slot];
      if (d.nnz == 0) return "";
      ChainArgs a{};
      a.f = f;
      a.q = acc;
      a.q2 = acc2;
      return f < c->k ? case_chain<CH_ETERM_V>(c, s, d, n, x.col_lo[b], a)
                      : case_chain<CH_ETERM_W>(c, s, d, n, x.col_lo[b], a);
    });
    if (!err.empty()) return err;
    if (f < c->k) MK(launch_for(c, n, eterm_factor_kernel, e, acc, n));
  }
  MK(launch_for(c, n, eterm_final_kernel, e, acc2, n, (int)c->k0, c->p64.w0()));
  return "";
}

// mcmc_block_sweep_kernel<V, REL> by [V][REL]
const void* const kBlockSweep[2][2] = {
    {(const void*)mcmc_block_sweep_kernel<false, false>, (const void*)mcmc_block_sweep_kernel<false, true>},
    {(const void*)mcmc_block_sweep_kernel<true, false>, (const void*)mcmc_block_sweep_kernel<true, true>}};

// mcmc_cta_sweep_kernel<V, REL> by [V][REL]
const void* const kCtaSweep[2][2] = {
    {(const void*)mcmc_cta_sweep_kernel<false, false>, (const void*)mcmc_cta_sweep_kernel<false, true>},
    {(const void*)mcmc_cta_sweep_kernel<true, false>, (const void*)mcmc_cta_sweep_kernel<true, true>}};

// The sweep of w (v = false) or of factor f over the runs of segment seg (rel: of a relation block), stretch by
// stretch of the plan: a stretch of narrow runs is one launch of one CTA, a stretch of wide runs one cooperative
// launch; nothing when the segment has no runs
std::string launch_block_sweep(fmb200_ctx* c, const McmcState& s, const SweepArgs& a, bool v, bool rel, size_t seg,
                               int f) {
  for (const Stretch& st : s.plan[seg]) {
    uint32_t r_lo = st.r_lo, r_hi = st.r_hi;
    void* args[] = {(void*)&a, (void*)&r_lo, (void*)&r_hi, (void*)&f};
    if (st.narrow) MK(cudaLaunchKernel(kCtaSweep[v][rel], dim3(1), dim3(s.cta_threads), args, 0, c->stream));
    else MK(cudaLaunchCooperativeKernel(kBlockSweep[v][rel], dim3(s.grid), dim3(256), args, 0, c->stream));
    c->launches++;
  }
  return "";
}

// The sweep over a streamed training set: pass -1 draws w, pass f draws factor f, block by block over the
// block's runs.  The q of factor f + 1 (which reads only v(f + 1, .), untouched by the sweep of f) is rebuilt on
// pass f into the other q array.
std::string xt_sweep(fmb200_ctx* c, McmcState& s, SweepArgs a) {
  McmcSet& t = s.set[0];
  XtSet& x = *t.xt;
  double* q[2] = {t.chain[0].get(), t.chain[1].get()};
  for (int p = -1; p < a.k; p++) {
    const bool sweep = p >= 0 || a.use_w, rebuild = p + 1 < a.k;
    if (!sweep && !rebuild) continue;
    double* qn = rebuild ? q[(p + 1) % 2] : nullptr;
    if (rebuild) MK(cudaMemsetAsync(qn, 0, t.n * sizeof(double), c->stream));
    if (p >= 0) a.q = q[p % 2];
    const std::string err = xt_pass(c, x, [&](int slot, uint64_t b) -> std::string {
      const DataSlot& d = c->slots[slot];
      if (rebuild && d.nnz > 0) {
        ChainArgs ca{};
        ca.f = p + 1;
        ca.q = qn;
        const std::string r = case_chain<CH_Q>(c, s, d, t.n, x.col_lo[b], ca);
        if (!r.empty()) return r;
      }
      if (!sweep) return "";
      a.cols = Cols{d.row_ptr.get(), x.col_lo[b], x.col_lo[b + 1], d.col.get(), d.val.get()};
      return launch_block_sweep(c, s, a, p >= 0, false, b, p < 0 ? 0 : p);
    });
    if (!err.empty()) return err;
  }
  return "";
}

// The e-terms of set `side` into its e_d.  With relations (fm_learn_mcmc.h:148-378) the train side first computes
// every block row's y, q and q_f, which the test side reads as well.
std::string eterms(fmb200_ctx* c, McmcState& s, int side) {
  McmcSet& t = s.set[side];
  if (t.xt) return xt_eterms(c, s, t);
  if (side == 0)
    for (const RelDev& r : s.rel)
      MK(launch_for(c, r.rows, rel_row_kernel<REL_ETERM>, r.view(), c->p64.v(), c->p64.w(), c->k, 0, (int)c->k1));
  MK(launch_mcmc_eterms(c, c->slots[t.slot], t.e_d.get(), s.rel_d.get(), (uint32_t)s.rel.size(), side));
  return "";
}

std::string repredict(fmb200_ctx* c, McmcState& s) {
  for (int side = 0; side < 2; side++) {
    const std::string err = eterms(c, s, side);
    if (!err.empty()) return err;
  }
  for (McmcSet& t : s.set)
    if (t.n) MK(cudaMemcpyAsync(t.e.data(), t.e_d.get(), t.n * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  MK(cudaStreamSynchronize(c->stream));
  return "";
}

// The checks of a fmb200_xt_blocks and the set it describes; "" when it may be streamed.
std::string xt_open(const fmb200_ctx* c, const fmb200_xt_blocks& src, const char* which, std::unique_ptr<XtSet>* out) {
  const std::string w = std::string("the ") + which + " .xt blocks: ";
  if (src.n_blocks == 0 || !src.col_lo || !src.nnz || !src.fetch || !src.release) return w + "no blocks or a null pointer";
  if (src.n_cases && !src.target) return w + "null target";
  if (src.n_cases >= 0xffffffffull) return w + "2^32 cases and more are not supported";
  for (int i = 0; i < 2; i++)
    if (src.slot[i] < 0 || src.slot[i] >= FMB200_MAX_SLOTS) return w + "slot out of range";
  if (src.slot[0] == src.slot[1]) return w + "the two slots must differ";
  if (src.col_lo[0] != 0 || src.col_lo[src.n_blocks] > c->n)
    return w + "the columns must start at 0 and end at or below num_attribute";
  std::unique_ptr<XtSet> x(new XtSet());
  x->src = src;
  x->col_lo.assign(src.col_lo, src.col_lo + src.n_blocks + 1);
  x->nnz.assign(src.nnz, src.nnz + src.n_blocks);
  for (uint64_t b = 0; b < src.n_blocks; b++) {
    if (x->col_lo[b + 1] < x->col_lo[b]) return w + "column ranges out of order";
    if (x->nnz[b] >= 0xffffffffull) return w + "a block of 2^32 entries and more is not supported";
  }
  *out = std::move(x);
  return "";
}

// x := draw when it is finite.  Otherwise x keeps its value, counter a (NaN) or a + 1 (Inf) grows and the
// result is true: the reference restores the old value and, in its per-group loops, stops drawing.
bool reject_nonfinite(double& x, double draw, uint32_t* cnt, int a) {
  if (std::isnan(draw)) { cnt[a]++; return true; }
  if (std::isinf(draw)) { cnt[a + 1]++; return true; }
  x = draw;
  return false;
}

// draw_w_lambda (fm_learn_mcmc.h:980-1017) / one factor of draw_v_lambda (:1059-1097) over one column:
// feature i's parameter is par[i * stride], group g's mean and precision mu[g * stride] and lambda[g * stride].
// True when a draw was not finite (the reference stops there).
bool draw_lambda(const McmcState& s, const double* par, const double* mu, double* lambda, size_t stride,
                 uint32_t* cnt, int a) {
  std::vector<double> gam(s.G);
  for (uint32_t g = 0; g < s.G; g++) {
    const double m = mu[g * stride];
    gam[g] = kBeta0 * (m - kMu0) * (m - kMu0) + kGamma0;
  }
  for (size_t i = 0; i < s.group.size(); i++) {
    const uint32_t g = s.group[i];
    const double m = mu[g * stride];
    gam[g] += (par[i * stride] - m) * (par[i * stride] - m);
  }
  for (uint32_t g = 0; g < s.G; g++) {
    const double al = kAlpha0 + s.per_group[g] + 1;
    if (reject_nonfinite(lambda[g * stride], s.sample ? ran_gamma(al / 2.0, gam[g] / 2.0) : al / gam[g], cnt, a))
      return true;
  }
  return false;
}

// draw_w_mu (:941-978) / one factor of draw_v_mu (:1019-1057), same column layout as draw_lambda
bool draw_mu(const McmcState& s, const double* par, double* mu, const double* lambda, size_t stride, uint32_t* cnt,
             int a) {
  std::vector<double> mean(s.G, 0.0);
  for (size_t i = 0; i < s.group.size(); i++) mean[s.group[i]] += par[i * stride];
  for (uint32_t g = 0; g < s.G; g++) {
    mean[g] = (mean[g] + kBeta0 * kMu0) / (s.per_group[g] + kBeta0);
    const double sig = (double)1.0 / ((s.per_group[g] + kBeta0) * lambda[g * stride]);
    if (reject_nonfinite(mu[g * stride], s.sample ? ran_gaussian(mean[g], std::sqrt(sig)) : mean[g], cnt, a))
      return true;
  }
  return false;
}

// A relation block on the device: its .xt, the row-major copy, the joins and the join inverse, #^R, and the
// block's part of the begin-time index (prev of its ids, dup of its columns)
std::string rel_upload(fmb200_ctx* c, McmcState& s, const RelationHost& h, RelDev& r, unsigned int* prev_d) {
  r.rows = h.num_cases;
  r.nf = h.num_feature;
  r.off = h.attr_offset;
  const uint64_t nnz = h.row.size(), n_join = h.join[0].size(), k = (uint64_t)c->k;
  MK(to_device(c, r.col_ptr, h.col_ptr.data(), r.nf + 1));
  MK(to_device(c, r.xt_row, h.row.data(), nnz));
  MK(to_device(c, r.xt_val, h.val.data(), nnz));
  MK(alloc(r.row_ptr, (uint64_t)r.rows + 1));
  MK(alloc(r.col, nnz));
  MK(alloc(r.val, nnz));
  MK(alloc(r.inv_ptr, (uint64_t)r.rows + 1));
  MK(alloc(r.cache, (7 + k) * r.rows));
  MK(cudaMemsetAsync(r.cache.get(), 0, (7 + k) * r.rows * sizeof(double), c->stream));
  for (int side = 0; side < 2; side++) MK(to_device(c, r.join[side], h.join[side].data(), h.join[side].size()));
  // the row-major copy: the entries stably sorted by row
  DevPtr<uint32_t> key, pos;
  std::string err = sort_once(c, r.xt_row.get(), nnz, r.rows, key, pos);
  if (!err.empty()) return err;
  if (nnz > 0)
    MK(launch_for(c, nnz, rel_rowmajor_kernel, pos.get(), nnz, r.col_ptr.get(), r.nf, r.off, r.xt_val.get(),
                  r.col.get(), r.val.get()));
  MK(launch_for(c, (uint64_t)r.rows + 1, mcmc_colptr_kernel, key.get(), nnz, r.rows, r.row_ptr.get()));
  if (r.rows > 0) {
    MK(launch_for(c, r.rows, rel_dup_kernel, r.row_ptr.get(), r.col.get(), r.rows, s.dup.get()));
    MK(launch_for(c, r.rows, mcmc_prev_kernel, r.row_ptr.get(), r.col.get(), (uint64_t)r.rows, prev_d));
  }
  // the join inverse: the train cases stably sorted by row
  err = sort_once(c, r.join[0].get(), n_join, r.rows, key, r.inv_case);
  if (!err.empty()) return err;
  MK(launch_for(c, (uint64_t)r.rows + 1, mcmc_colptr_kernel, key.get(), n_join, r.rows, r.inv_ptr.get()));
  MK(launch_for(c, r.rows, rel_wnum_kernel, r.view()));
  MK(cudaStreamSynchronize(c->stream));
  return "";
}

// One iteration's sweep with relations (draw_all, fm_learn_mcmc.h:438-640 after draw_w0): the main table's runs,
// then per block the unsync, its runs over its rows and the resync; per factor first the q rebuild of the blocks'
// rows and of the cases
std::string rel_sweep(fmb200_ctx* c, McmcState& s, const SweepArgs& a) {
  const uint64_t N = s.set[0].n;
  auto sweep = [&](bool v, int f) -> std::string {
    std::string err = launch_block_sweep(c, s, a, v, false, 0, f);
    for (uint32_t r = 0; err.empty() && r < s.rel.size(); r++) {
      SweepArgs b = a;
      b.rel = s.rel[r].view();
      b.cols = s.rel[r].cols();
      b.q = b.rel.q;
      MK(launch_for(c, b.rel.rows, v ? rel_unsync_kernel<true> : rel_unsync_kernel<false>, b.rel, a.e, a.q));
      err = launch_block_sweep(c, s, b, v, true, r + 1, f);
      if (err.empty()) MK(launch_for(c, N, v ? rel_resync_kernel<true> : rel_resync_kernel<false>, b.rel, a.e, a.q, N));
    }
    return err;
  };
  if (a.use_w) {
    const std::string err = sweep(false, 0);
    if (!err.empty()) return err;
  }
  for (int f = 0; f < a.k; f++) {
    for (const RelDev& r : s.rel) MK(launch_for(c, r.rows, rel_row_kernel<REL_Q>, r.view(), a.v, a.w, a.k, f, 0));
    MK(launch_for(c, N, rel_case_q_kernel, a, f, s.rel_d.get(), (uint32_t)s.rel.size()));
    const std::string err = sweep(true, f);
    if (!err.empty()) return err;
  }
  return "";
}

// ---- begin, step by step ----------------------------------------------------------------------------------------
// The checks of the train and test sets and of the relations; the streamed sets opened into xt
std::string check_sets(fmb200_ctx* c, int train, int test, const std::vector<RelationHost>& rel,
                       const fmb200_xt_blocks* const src[2], std::unique_ptr<XtSet> xt[2]) {
  if (!rel.empty()) {
    if (train != c->mcmc_rel_slot[0] || test != c->mcmc_rel_slot[1])
      return "the relations were set for train slot " + std::to_string(c->mcmc_rel_slot[0]) + " and test slot " +
             std::to_string(c->mcmc_rel_slot[1]);
    if (c->slots[train].upload_gen != c->mcmc_rel_gen[0] || c->slots[test].upload_gen != c->mcmc_rel_gen[1])
      return "the train or test slot was re-uploaded after fmb200_mcmc_set_relations: set the relations again";
    const uint32_t off0 = rel[0].attr_offset;
    std::vector<float> cnt(c->n - off0);
    for (int slot : {train, test}) {  // the main tables' ids lie below the first block's
      if (cnt.empty() || c->slots[slot].nnz == 0) continue;
      MK(cudaMemcpyAsync(cnt.data(), c->slots[slot].feat_cnt.get() + off0, cnt.size() * sizeof(float),
                         cudaMemcpyDeviceToHost, c->stream));
      MK(cudaStreamSynchronize(c->stream));
      for (size_t j = 0; j < cnt.size(); j++)
        if (cnt[j] != 0.0f)
          return "the data in slot " + std::to_string(slot) + " names attribute " + std::to_string(off0 + j) +
                 ", which belongs to relation block attributes (from " + std::to_string(off0) + " on)";
    }
  }
  const char* name[2] = {"train", "test"};
  for (int side = 0; side < 2; side++)
    if (src[side]) {
      const std::string e = xt_open(c, *src[side], name[side], &xt[side]);
      if (!e.empty()) return e;
    }
  {  // no slot may serve two purposes
    std::vector<int> used;
    for (int side = 0; side < 2; side++)
      if (src[side]) used.insert(used.end(), {src[side]->slot[0], src[side]->slot[1]});
      else if (side == 0 || test != train) used.push_back(side == 0 ? train : test);
    for (size_t i = 0; i < used.size(); i++)
      for (size_t j = 0; j < i; j++)
        if (used[i] == used[j]) return "a streamed set's slots must differ from every other slot in use";
  }
  const DataSlot* d = src[0] ? nullptr : &c->slots[train];
  if ((d ? d->n_rows : src[0]->n_cases) == 0) return "the training set is empty";
  if (d && (d->n_rows >= 0xffffffffull || d->nnz >= 0xffffffffull))
    return "training sets of 2^32 cases or entries and more are not supported";
  return "";
}

// Set `side` (0 train, 1 test): its slot or its streamed .xt, the targets, the e-terms and the per-case chains
std::string open_set(fmb200_ctx* c, McmcState& s, int side, int slot, std::unique_ptr<XtSet> xt) {
  McmcSet& t = s.set[side];
  t.slot = slot;
  t.xt = std::move(xt);
  t.n = t.xt ? t.xt->src.n_cases : c->slots[slot].n_rows;
  t.y.resize(t.n);
  t.e.resize(t.n);
  MK(alloc(t.e_d, t.n));
  if (side == 0 || t.xt) MK(alloc(t.chain[0], t.n));
  if (t.xt) MK(alloc(t.chain[1], t.n));
  if (!t.xt) {
    const DataSlot& d = c->slots[slot];
    t.gen = d.upload_gen;
    t.y_dev = d.target.get();
    if (t.n) MK(cudaMemcpyAsync(t.y.data(), d.target.get(), t.n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  } else {
    std::copy(t.xt->src.target, t.xt->src.target + t.n, t.y.begin());
    if (side == 0) {
      MK(to_device(c, t.y_d, t.y.data(), t.n));
      t.y_dev = t.y_d.get();
    }
  }
  return "";
}

// The index of the training data: the transposed data (resident: from the (id, entry) sort of the ORDERED index;
// streamed: none, the blocks are), dup, and the relation blocks on the device.  prev[j] = 1 + the largest id below
// j that shares a case, or a relation block's row, with j (0: none), from one device array into which every route
// writes: the main tables name no block id (check_sets), so the routes write disjoint ids.
std::string build_index(fmb200_ctx* c, McmcState& s, const std::vector<RelationHost>& rel, std::vector<uint32_t>* prev) {
  const uint32_t n = c->n;
  McmcSet& t = s.set[0];
  MK(alloc(s.dup, n));
  MK(cudaMemsetAsync(s.dup.get(), 0, n * sizeof(uint32_t), c->stream));
  if (t.xt || s.set[1].xt) {  // the by-case sort of the largest block
    uint64_t max_nnz = 1;
    for (const McmcSet& x : s.set)
      if (x.xt) max_nnz = std::max(max_nnz, *std::max_element(x.xt->nnz.begin(), x.xt->nnz.end()));
    MK(alloc(s.srt_key, max_nnz));
    MK(alloc(s.srt_pos, max_nnz));
    const std::string err = sort_scratch(c, max_nnz, 1ull << 32, s.srt);
    if (!err.empty()) return err;
  }
  DataSlot* d = t.xt ? nullptr : &c->slots[t.slot];
  SortedEntries se;
  if (d) {
    MK(alloc(s.col_ptr, n + 1));
    MK(alloc(s.cs_case, d->nnz));
    MK(alloc(s.cs_x, d->nnz));
    if (d->nnz > 0) MK(build_ordered_links(c, *d, &se));
    else MK(cudaMemsetAsync(s.col_ptr.get(), 0, (n + 1) * sizeof(uint64_t), c->stream));
  }
  DevPtr<unsigned int> prev_d;  // allocated after the index build's scratch
  MK(alloc(prev_d, n));
  MK(cudaMemsetAsync(prev_d.get(), 0, n * sizeof(unsigned int), c->stream));
  if (t.xt) {  // one pass over the streamed .xt
    DevPtr<uint32_t> last;
    MK(alloc(last, t.n));
    MK(cudaMemsetAsync(last.get(), 0, t.n * sizeof(uint32_t), c->stream));
    const std::string err = xt_pass(c, *t.xt, [&](int slot, uint64_t b) -> std::string {
      const DataSlot& blk = c->slots[slot];
      if (blk.nnz == 0) return "";
      ChainArgs a{};
      a.last = last.get();
      a.prev = prev_d.get();
      a.dup = s.dup.get();
      return case_chain<CH_PREV>(c, s, blk, t.n, t.xt->col_lo[b], a);
    });
    if (!err.empty()) return err;
  } else if (d->nnz > 0) {
    MK(launch_for(c, d->nnz, mcmc_csc_kernel, se.ids, se.ent, d->nnz, d->row_ptr.get(), d->n_rows, d->val.get(),
                  s.cs_case.get(), s.cs_x.get(), s.dup.get()));
    MK(launch_for(c, (uint64_t)n + 1, mcmc_colptr_kernel, se.ids, d->nnz, n, s.col_ptr.get()));
    MK(launch_for(c, d->n_rows, mcmc_prev_kernel, d->row_ptr.get(), d->col.get(), d->n_rows, prev_d.get()));
  }
  if (!rel.empty()) {
    s.rel.resize(rel.size());
    std::vector<RelView> views;
    for (size_t r = 0; r < rel.size(); r++) {
      const std::string err = rel_upload(c, s, rel[r], s.rel[r], prev_d.get());
      if (!err.empty()) return err;
      views.push_back(s.rel[r].view());
    }
    MK(to_device(c, s.rel_d, views.data(), views.size()));
  }
  prev->assign(n, 0u);
  MK(cudaMemcpyAsync(prev->data(), prev_d.get(), n * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
  MK(cudaStreamSynchronize(c->stream));
  return "";
}

// Cut the ids greedily into runs: j opens a new run when it shares a case with a feature of the current run, and
// at every segment's first id (seg, ascending from 0), so that no run spans two segments
std::string cut_runs(fmb200_ctx* c, McmcState& s, const std::vector<uint32_t>& prev, const std::vector<uint32_t>& seg) {
  const uint32_t n = c->n;
  std::vector<bool> cut(n, false);
  for (uint32_t j : seg)
    if (j < n) cut[j] = true;
  s.runs.clear();
  if (n > 0) s.runs.push_back(0);
  for (uint32_t j = 1; j < n; j++)
    if ((prev[j] != 0 && prev[j] - 1 >= s.runs.back()) || cut[j]) s.runs.push_back(j);
  s.runs.push_back(n);
  // a segment sweeps the runs that start in it; the last one also the features after it
  for (uint32_t j : seg)
    s.seg_run.push_back((uint32_t)(std::lower_bound(s.runs.begin(), s.runs.end() - 1, j) - s.runs.begin()));
  s.seg_run.push_back((uint32_t)s.runs.size() - 1);
  MK(to_device(c, s.runs_d, s.runs.data(), s.runs.size()));
  return "";
}

// The launch plan of the segmented sweeps: each segment's runs in maximal stretches of narrow runs (at most as many
// features as the sweeping CTA has warps) and of wide runs.  fmb200_set_tuning's threads sets the CTA's width, and
// its variant 1 makes every run wide (the cooperative kernel alone, for comparison).
void plan_sweeps(const fmb200_ctx* c, McmcState& s) {
  s.cta_threads = c->tune_threads ? c->tune_threads : kCtaSweepThreads;
  const uint32_t warps = (uint32_t)s.cta_threads / 32;
  s.plan.assign(s.seg_run.size() - 1, {});
  for (size_t i = 0; i + 1 < s.seg_run.size(); i++)
    for (uint32_t r = s.seg_run[i]; r < s.seg_run[i + 1]; r++) {
      const bool narrow = c->tune_variant != 1 && s.runs[r + 1] - s.runs[r] <= warps;
      std::vector<Stretch>& p = s.plan[i];
      if (!p.empty() && p.back().narrow == narrow) p.back().r_hi = r + 1;
      else p.push_back(Stretch{r, r + 1, narrow});
    }
}

// The cooperative grid: as many blocks per SM as every sweep kernel the iteration launches fits
std::string size_grid(fmb200_ctx* c, McmcState& s) {
  std::vector<const void*> fns = {(const void*)mcmc_sweep_kernel};
  if (s.set[0].xt || !s.rel.empty()) fns = {kBlockSweep[0][0], kBlockSweep[1][0]};
  if (!s.rel.empty()) fns.insert(fns.end(), {kBlockSweep[0][1], kBlockSweep[1][1]});
  int occ = INT_MAX;
  for (const void* fn : fns) {
    int o = 0;
    MK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, fn, 256, 0));
    occ = std::min(occ, o);
  }
  if (occ < 1) return "the sweep kernel does not fit an SM";
  s.grid = occ * c->sm_count;
  return "";
}

// ---- an iteration, step by step ---------------------------------------------------------------------------------
// The host draws before the sweep: alpha, w0, w_lambda, w_mu, one normal per w, v_lambda, v_mu, one normal per v.
// True when w0 moved: e then shifts by *e_shift (draw_w0's update of e).
bool draw_hyper(fmb200_ctx* c, McmcState& s, double* e_shift) {
  const uint32_t n = c->n;
  const int k = c->k;
  const uint64_t N = s.set[0].n;
  const std::vector<double>& e = s.set[0].e;
  const bool sample = s.sample, ml = s.multilevel;
  uint32_t* cnt = s.counters;  // nan, inf of: alpha, w0, w, v, w_mu, w_lambda, v_mu, v_lambda
  double& w0 = s.state[0];
  const double* w = s.state.data() + Params64::off_w;
  const double* v = s.state.data() + c->p64.off_v;  // [n][k]

  // draw_alpha, fm_learn_mcmc.h:911-939
  if (!ml) {
    s.alpha = kAlpha0;
  } else {
    const double alpha_n = kAlpha0 + N;
    double gamma_n = kGamma0;
    for (uint64_t i = 0; i < N; i++) gamma_n += e[i] * e[i];
    reject_nonfinite(s.alpha, ran_gamma(alpha_n / 2.0, gamma_n / 2.0), cnt, 0);
  }
  const double alpha = s.alpha;
  // draw_w0, :643-683
  bool shift = false;
  if (c->k0) {
    double mean = 0;
    for (uint64_t i = 0; i < N; i++) mean += e[i] - w0;
    const double sig = (double)1.0 / (s.reg0 + alpha * N);
    mean = -sig * (alpha * mean - kW0Mean0 * s.reg0);
    const double old = w0;
    if (!reject_nonfinite(w0, sample ? ran_gaussian(mean, std::sqrt(sig)) : mean, cnt, 2)) {
      shift = true;
      *e_shift = old - w0;
    }
  }
  if (c->k1) {
    if (ml) {
      draw_lambda(s, w, s.w_mu.data(), s.w_lambda.data(), 1, cnt, 10);
      draw_mu(s, w, s.w_mu.data(), s.w_lambda.data(), 1, cnt, 8);
    } else {
      std::fill(s.w_mu.begin(), s.w_mu.end(), kMu0);
    }
    if (sample)
      for (uint32_t j = 0; j < n; j++) s.z[j] = ran_gaussian();
  }
  if (k > 0) {
    if (ml) {  // a non-finite draw stops the factors that follow too
      for (int f = 0; f < k; f++)
        if (draw_lambda(s, v + f, s.v_mu.data() + f, s.v_lambda.data() + f, k, cnt, 14)) break;
      for (int f = 0; f < k; f++)
        if (draw_mu(s, v + f, s.v_mu.data() + f, s.v_lambda.data() + f, k, cnt, 12)) break;
    } else {
      std::fill(s.v_mu.begin(), s.v_mu.end(), kMu0);
    }
    if (sample)
      for (size_t i = n; i < (size_t)(k + 1) * n; i++) s.z[i] = ran_gaussian();
  }
  return shift;
}

// The sweep on the device: w0, the hyperparameters and the normals go up; then draw_w0's shift of e and the draws of
// w and v, feature run by feature run
std::string sweep(fmb200_ctx* c, McmcState& s, bool shift, double e_shift) {
  const uint32_t n = c->n, G = s.G;
  const int k = c->k;
  McmcSet& t = s.set[0];
  std::copy(s.w_mu.begin(), s.w_mu.end(), s.hyp.begin());
  std::copy(s.w_lambda.begin(), s.w_lambda.end(), s.hyp.begin() + G);
  std::copy(s.v_mu.begin(), s.v_mu.end(), s.hyp.begin() + 2 * G);
  std::copy(s.v_lambda.begin(), s.v_lambda.end(), s.hyp.begin() + 2 * G + (size_t)G * k);
  MK(cudaMemcpyAsync(c->p64.w0(), &s.state[0], sizeof(double), cudaMemcpyHostToDevice, c->stream));
  MK(cudaMemcpyAsync(s.hyp_d.get(), s.hyp.data(), s.hyp.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  if (s.sample) MK(cudaMemcpyAsync(s.z_d.get(), s.z.data(), s.z.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SweepArgs a{};
  if (!t.xt) {
    const DataSlot& d = c->slots[t.slot];
    a.cols = Cols{s.col_ptr.get(), 0, n, s.cs_case.get(), s.cs_x.get()};
    a.row_ptr = d.row_ptr.get();
    a.col = d.col.get();
    a.val = d.val.get();
  }
  a.dup = s.dup.get();
  a.group = s.group_d.get();
  a.runs = s.runs_d.get();
  a.n_runs = (uint32_t)s.runs.size() - 1;
  a.n = n;
  a.G = G;
  a.n_rows = t.n;
  a.e = t.e_d.get();
  a.q = t.chain[0].get();
  a.w = c->p64.w();
  a.v = c->p64.v();
  a.k = k;
  a.use_w = c->k1;
  a.sample = s.sample;
  a.shift = shift;
  a.alpha = s.alpha;
  a.e_shift = e_shift;
  a.z = s.z_d.get();
  a.hyp = s.hyp_d.get();
  a.flag = s.flag_d.get();
  if (!t.xt && s.rel.empty()) {  // resident: one cooperative launch, the shift included
    if (a.shift || a.use_w || k > 0) {
      void* args[] = {(void*)&a};
      MK(cudaLaunchCooperativeKernel((const void*)mcmc_sweep_kernel, dim3(s.grid), dim3(256), args, 0, c->stream));
      c->launches++;
    }
  } else {
    if (shift) MK(launch_for(c, t.n, mcmc_shift_kernel, a.e, t.n, e_shift));
    const std::string err = t.xt ? xt_sweep(c, s, a) : rel_sweep(c, s, a);
    if (!err.empty()) return err;
  }
  unsigned int flag[F_WORDS];
  MK(cudaMemcpyAsync(flag, s.flag_d.get(), sizeof(flag), cudaMemcpyDeviceToHost, c->stream));
  MK(cudaStreamSynchronize(c->stream));
  s.counters[4] = flag[F_NAN_W];
  s.counters[5] = flag[F_INF_W];
  s.counters[6] = flag[F_NAN_V];
  s.counters[7] = flag[F_INF_V];
  if (flag[F_SKIP] != 0xffffffffu) {
    char buf[160];
    if (flag[F_SKIP] == 0) snprintf(buf, sizeof(buf), "iteration %u: a draw of w has a non-finite or zero posterior variance", s.iter);
    else snprintf(buf, sizeof(buf), "iteration %u: a draw of v[f=%u] has a non-finite or zero posterior variance", s.iter, flag[F_SKIP] - 1);
    return std::string(buf) + " (the model state diverged; sampling stops instead of desynchronising the random stream)";
  }
  return "";
}

// Re-prediction and the target step, fm_learn_mcmc_simultaneous.h:122-200
std::string target_step(fmb200_ctx* c, McmcState& s, double* train_metric) {
  std::string err = repredict(c, s);
  if (!err.empty()) return err;
  const uint64_t N = s.set[0].n, NT = s.set[1].n;
  std::vector<double>& e = s.set[0].e;
  const std::vector<double>& e_test = s.set[1].e;
  const std::vector<float>& y = s.set[0].y;
  const uint32_t i = s.iter;
  const double lo = c->hp.min_target, hi = c->hp.max_target;
  const bool reg = c->hp.task == FMB200_TASK_REGRESSION;
  for (uint64_t t = 0; t < NT; t++) {  // a regression prediction is summed clipped to the target range
    const double p = reg ? e_test[t] : cdf_gaussian(e_test[t]), ps = reg ? std::max(lo, std::min(hi, p)) : p;
    s.pred_this[t] = p;
    s.pred_all[t] += ps;
    if (i >= 5) s.pred_but5[t] += ps;
  }
  if (reg) {
    double rmse = 0.0;
    for (uint64_t t = 0; t < N; t++) {
      double p = e[t];
      p = std::min(hi, p);
      p = std::max(lo, p);
      const double er = p - y[t];
      rmse += er * er;
    }
    *train_metric = std::sqrt(rmse / N);
    MK(launch_for(c, N, mcmc_residual_kernel, s.set[0].e_d.get(), s.set[0].y_dev, N));
    for (uint64_t t = 0; t < N; t++) e[t] = e[t] - y[t];
  } else {
    uint64_t acc = 0;
    for (uint64_t t = 0; t < N; t++) {
      const double p = cdf_gaussian(e[t]);
      if (((p >= 0.5) && (y[t] > 0.0)) || ((p < 0.5) && (y[t] < 0.0))) acc++;
      const double mu = e[t];
      double st;
      if (s.sample) {
        st = y[t] >= 0.0 ? ran_left_tgaussian(0.0, mu, 1.0) : ran_right_tgaussian(0.0, mu, 1.0);
      } else {
        const double phi = std::exp(-mu * mu / 2.0) / std::sqrt(3.141 * 2);
        st = y[t] >= 0.0 ? mu + phi / (1 - cdf_gaussian(-mu)) : mu - phi / cdf_gaussian(-mu);
      }
      e[t] = e[t] - st;
    }
    *train_metric = (double)acc / N;
    MK(cudaMemcpyAsync(s.set[0].e_d.get(), e.data(), N * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  }
  MK(cudaStreamSynchronize(c->stream));
  return "";
}

}  // namespace

std::string mcmc_check_relations(const fmb200_ctx* c, int train, int test, uint32_t n_rel, const fmb200_relation* rel,
                                 std::vector<RelationHost>* out) {
  if (!rel) return "null relation list";
  const uint64_t n_cases[2] = {c->slots[train].n_rows, c->slots[test].n_rows};
  const char* side_name[2] = {"train", "test"};
  std::vector<RelationHost> v(n_rel);
  uint64_t next = rel[0].attr_offset;
  for (uint32_t b = 0; b < n_rel; b++) {
    const fmb200_relation& x = rel[b];
    RelationHost& h = v[b];
    const std::string w = "relation " + std::to_string(b) + ": ";
    if (x.attr_offset != next)
      return w + "attr_offset " + std::to_string(x.attr_offset) + " does not follow the previous block's attributes, which end at " +
             std::to_string(next) + " (the blocks' ids must be contiguous)";
    next = (uint64_t)x.attr_offset + x.num_feature;
    if (next > c->n) return w + "its attributes end at " + std::to_string(next) + ", beyond num_attribute " + std::to_string(c->n);
    if (!x.col_ptr) return w + "null col_ptr";
    if (x.col_ptr[0] != 0) return w + "col_ptr[0] must be 0";
    for (uint32_t j = 0; j < x.num_feature; j++)
      if (x.col_ptr[j + 1] < x.col_ptr[j]) return w + "col_ptr is not ascending at column " + std::to_string(j);
    const uint64_t nnz = x.col_ptr[x.num_feature];
    if (nnz >= 0xffffffffull) return w + "blocks of 2^32 entries and more are not supported";
    if (nnz && (!x.row || !x.val)) return w + "null row / val";
    for (uint64_t p = 0; p < nnz; p++)
      if (x.row[p] >= x.num_cases)
        return w + "entry " + std::to_string(p) + " names row " + std::to_string(x.row[p]) + ", not below num_cases " +
               std::to_string(x.num_cases);
    const uint64_t len[2] = {x.n_train, x.n_test};
    const uint32_t* join[2] = {x.train_join, x.test_join};
    for (int side = 0; side < 2; side++) {
      const std::string j = w + "the " + side_name[side] + " join ";
      if (len[side] != n_cases[side])
        return j + "has " + std::to_string(len[side]) + " entries, the " + side_name[side] + " set " +
               std::to_string(n_cases[side]) + " cases";
      if (len[side] && !join[side]) return j + "is null";
      for (uint64_t i = 0; i < len[side]; i++)
        if (join[side][i] >= x.num_cases)
          return j + "maps case " + std::to_string(i) + " to row " + std::to_string(join[side][i]) +
                 ", not below num_cases " + std::to_string(x.num_cases);
      h.join[side].assign(join[side], join[side] + len[side]);
    }
    h.num_cases = x.num_cases;
    h.num_feature = x.num_feature;
    h.attr_offset = x.attr_offset;
    h.col_ptr.assign(x.col_ptr, x.col_ptr + x.num_feature + 1);
    h.row.assign(x.row, x.row + nnz);
    h.val.assign(x.val, x.val + nnz);
  }
  if (next != c->n)
    return "the last block's attributes end at " + std::to_string(next) + ", not at num_attribute " + std::to_string(c->n);
  *out = std::move(v);
  return "";
}

std::string mcmc_begin(fmb200_ctx* c, int train, int test, int do_sample, int do_multilevel, uint32_t G,
                       const uint32_t* attr_group, const uint32_t* attr_per_group, double reg0,
                       const double* w_lambda0, const double* v_lambda0, const fmb200_xt_blocks* train_xt,
                       const fmb200_xt_blocks* test_xt) {
  std::vector<RelationHost> rel = std::move(c->mcmc_rel);  // relations apply to this _begin only
  c->mcmc_rel.clear();
  const fmb200_xt_blocks* src[2] = {train_xt, test_xt};
  std::unique_ptr<XtSet> xt[2];
  std::string err = check_sets(c, train, test, rel, src, xt);
  if (!err.empty()) return err;
  if (G == 0) return "n_groups must be >= 1";
  c->mcmc.reset(new McmcState());
  McmcState& s = *c->mcmc;
  const uint32_t n = c->n;
  const int k = c->k;
  const int slot[2] = {train, test};
  for (int side = 0; side < 2; side++) {
    err = open_set(c, s, side, slot[side], std::move(xt[side]));
    if (!err.empty()) return err;
  }
  s.sample = do_sample != 0;
  s.multilevel = do_multilevel != 0;
  s.G = G;
  s.group.assign(n, 0u);
  s.per_group.assign(G, 0u);
  if (attr_group) {
    for (uint32_t i = 0; i < n; i++) {
      if (attr_group[i] >= G) return "attr_group names a group >= n_groups";
      s.group[i] = attr_group[i];
    }
  }
  if (attr_per_group) std::copy(attr_per_group, attr_per_group + G, s.per_group.begin());
  else for (uint32_t i = 0; i < n; i++) s.per_group[s.group[i]]++;
  s.reg0 = reg0;
  s.alpha = 1.0;  // fm_learn_mcmc.h:1112
  s.w_mu.assign(G, 0.0);
  s.v_mu.assign((size_t)G * k, 0.0);
  s.w_lambda.assign(w_lambda0, w_lambda0 + G);
  s.v_lambda.assign(v_lambda0, v_lambda0 + (size_t)G * k);
  s.pred_this.assign(s.set[1].n, 0.0);
  s.pred_all.assign(s.set[1].n, 0.0);
  s.pred_but5.assign(s.set[1].n, 0.0);
  s.state.resize(c->p64.n_doubles);
  s.z.resize((size_t)(k + 1) * n);
  s.hyp.resize(2 * G + 2 * (size_t)G * k);
  MK(alloc(s.z_d, s.z.size()));
  MK(alloc(s.hyp_d, s.hyp.size()));
  MK(alloc(s.flag_d, F_WORDS));
  MK(to_device(c, s.group_d, s.group.data(), n));

  std::vector<uint32_t> prev;
  err = build_index(c, s, rel, &prev);
  if (!err.empty()) return err;
  // the segments' first ids: a streamed training set's blocks, or the main table and then the relation blocks
  std::vector<uint32_t> seg{0};
  if (s.set[0].xt) seg.assign(s.set[0].xt->col_lo.begin(), s.set[0].xt->col_lo.end() - 1);
  for (const RelationHost& h : rel) seg.push_back(h.attr_offset);
  err = cut_runs(c, s, prev, seg);
  if (err.empty()) err = size_grid(c, s);
  if (!err.empty()) return err;
  plan_sweeps(c, s);

  // fm_learn_mcmc_simultaneous.h:69-86: predict, then e := prediction - target (both tasks)
  err = repredict(c, s);
  if (!err.empty()) return err;
  McmcSet& t = s.set[0];
  for (uint64_t i = 0; i < t.n; i++) t.e[i] = t.e[i] - t.y[i];
  MK(cudaMemcpyAsync(t.e_d.get(), t.e.data(), t.n * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  MK(cudaStreamSynchronize(c->stream));
  return "";
}

std::string mcmc_iteration(fmb200_ctx* c, double* train_metric, uint32_t* counters) {
  McmcState& s = *c->mcmc;
  for (const McmcSet& t : s.set)
    if (!t.xt && c->slots[t.slot].upload_gen != t.gen) return "the train or test slot was re-uploaded: call fmb200_mcmc_begin again";
  std::fill(s.counters, s.counters + 16, 0u);
  MK(cudaMemcpyAsync(s.state.data(), c->p64.base, s.state.size() * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  MK(cudaMemsetAsync(s.flag_d.get(), 0, F_SKIP * sizeof(unsigned int), c->stream));
  MK(cudaMemsetAsync(s.flag_d.get() + F_SKIP, 0xff, sizeof(unsigned int), c->stream));
  MK(cudaStreamSynchronize(c->stream));
  double e_shift = 0.0;
  const bool shift = draw_hyper(c, s, &e_shift);
  std::string err = sweep(c, s, shift, e_shift);
  if (err.empty()) err = target_step(c, s, train_metric);
  if (!err.empty()) return err;
  s.iter++;
  if (counters) std::copy(s.counters, s.counters + 16, counters);
  return "";
}

#undef MK

bool mcmc_get(const fmb200_ctx* c, double* alpha, double* w_mu, double* w_lambda, double* v_mu, double* v_lambda,
              double* pred_this, double* pred_sum_all, double* pred_sum_all_but5, uint32_t* n_runs) {
  const McmcState* s = c->mcmc.get();
  if (!s) return false;
  if (alpha) *alpha = s->alpha;
  if (w_mu) std::copy(s->w_mu.begin(), s->w_mu.end(), w_mu);
  if (w_lambda) std::copy(s->w_lambda.begin(), s->w_lambda.end(), w_lambda);
  if (v_mu) std::copy(s->v_mu.begin(), s->v_mu.end(), v_mu);
  if (v_lambda) std::copy(s->v_lambda.begin(), s->v_lambda.end(), v_lambda);
  if (pred_this) std::copy(s->pred_this.begin(), s->pred_this.end(), pred_this);
  if (pred_sum_all) std::copy(s->pred_all.begin(), s->pred_all.end(), pred_sum_all);
  if (pred_sum_all_but5) std::copy(s->pred_but5.begin(), s->pred_but5.end(), pred_sum_all_but5);
  if (n_runs) *n_runs = (uint32_t)s->runs.size() - 1;
  return true;
}

}  // namespace fmb
