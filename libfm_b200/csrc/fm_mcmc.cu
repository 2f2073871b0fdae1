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
//    reference's serial chain.  The e-term re-prediction is fm_eterm64_kernel (fm_inorder.cu).
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

// A data set streamed from blocks of its .xt (fmb200_mcmc_begin_xt)
struct XtSet {
  fmb200_xt_blocks src{};
  std::vector<uint32_t> col_lo;  // [n_blocks + 1]
  std::vector<uint64_t> nnz;     // [n_blocks]
  std::vector<uint32_t> run_lo;  // train: block b sweeps the runs [run_lo[b], run_lo[b + 1])
  DevPtr<double> acc[2];         // test: the two per-case chains of the e-term passes (train uses q and q2)
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
};

struct McmcState {
  int train = 0, test = 1;
  std::unique_ptr<XtSet> xt[2];  // train, test: null when the set is resident in its slot
  uint64_t train_gen = 0, test_gen = 0;
  bool sample = true, multilevel = true;
  uint32_t G = 1;
  std::vector<uint32_t> group, per_group;  // attr_group[n], num_attr_per_group[G]
  double alpha = 1.0, reg0 = 0.0;
  std::vector<double> w_mu, w_lambda, v_mu, v_lambda;  // [G], [G][k]
  std::vector<float> y, y_test;
  std::vector<double> e, e_test, pred_this, pred_all, pred_but5;
  std::vector<double> state;  // host image of the fp64 state (Params64 layout)
  std::vector<double> z, hyp;
  std::vector<uint32_t> runs;  // run starts, then n
  uint32_t iter = 0;
  uint32_t counters[16] = {0};
  uint64_t n_train = 0, n_test = 0;
  // device
  DevPtr<uint64_t> col_ptr;
  DevPtr<uint32_t> cs_case, dup, group_d, runs_d;
  DevPtr<float> cs_x;
  DevPtr<double> e_d, q_d, e_test_d, z_d, hyp_d;
  DevPtr<unsigned int> flag_d;
  int grid = 0;
  // streamed sets: the train targets, the second q, and a block's entries stably sorted by case (the case
  // ids and the entries' positions in the block; iota = 0, 1, ... is the sort's input)
  DevPtr<float> y_d;
  DevPtr<double> q2_d;
  DevPtr<uint32_t> srt_key, srt_pos, iota;
  DevPtr<unsigned char> srt_tmp;
  size_t srt_tmp_bytes = 0;
  const float* y_dev = nullptr;  // the train targets on the device
  // relation blocks (fmb200_mcmc_set_relations); block r sweeps the runs [rel_run[r], rel_run[r + 1]), the main
  // table the runs before rel_run[0]
  std::vector<RelDev> rel;
  DevPtr<RelView> rel_d;
  std::vector<uint32_t> rel_run;
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
  const uint64_t* col_ptr;  // column j's positions: [col_ptr[j - col_lo], col_ptr[j - col_lo + 1]) for j < col_hi;
  uint32_t col_lo, col_hi;  // columns from col_hi on are empty (a streamed block and the features after the .xt)
  const uint32_t* cs_case;
  const float* cs_x;
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
  // the sweep of a relation block (REL): its rows play the cases, q is the rows' q, and the rows' caches
  const double* wnum;
  double *we, *weq, *wc, *wc_sqr, *y;
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
  if (j < a.col_hi) {
    beg = (uint32_t)a.col_ptr[j - a.col_lo];
    end = (uint32_t)a.col_ptr[j - a.col_lo + 1];
  }
  double m = 0.0, s = 0.0;
  for (uint32_t b = beg; b < end; b += 32) {
    const uint32_t idx = b + lane;
    double tm = 0.0, ts = 0.0;
    if (idx < end) {
      const uint32_t c = a.cs_case[idx];
      const float x = a.cs_x[idx];
      const double xd = (double)x;
      if (REL) {
        if (V) {
          const double h = xd * (a.q[c] - xd * old);
          tm = h * a.we[c] + xd * a.weq[c];
          ts = h * h * a.wnum[c] + 2 * a.wc[c] * xd * h + (double)(x * x) * a.wc_sqr[c];
        } else {
          tm = xd * a.we[c];
          ts = (double)(x * x) * a.wnum[c];
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
    const uint32_t c = a.cs_case[idx];
    const double xd = (double)a.cs_x[idx];
    if (REL) {
      if (V) {
        const double h = xd * (a.q[c] - xd * old);
        a.we[c] -= d * (h * a.wnum[c] + xd * a.wc[c]);
        a.q[c] -= d * xd;
        a.weq[c] -= d * (h * a.wc[c] + xd * a.wc_sqr[c]);
        a.y[c] += (nv - old) * h;
      } else {
        a.we[c] -= xd * d * a.wnum[c];
        a.y[c] += (nv - old) * xd;
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

// runs [r_lo, r_hi)
template <bool V, bool REL = false>
__device__ void sweep_runs(const SweepArgs& a, cg::grid_group& grid, int f, uint32_t r_lo, uint32_t r_hi, uint32_t warp,
                           uint32_t nwarp, int lane) {
  for (uint32_t r = r_lo; r < r_hi; r++) {
    const uint32_t j1 = a.runs[r + 1];
    for (uint32_t j = a.runs[r] + warp; j < j1; j += nwarp) draw_feature<V, REL>(a, j, f, lane);
    grid.sync();
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
  if (a.use_w) sweep_runs<false>(a, grid, 0, 0, a.n_runs, warp, nwarp, lane);
  for (int f = 0; f < a.k; f++) {
    for (uint64_t c = tid; c < a.n_rows; c += nth) a.q[c] = main_q(a, c, f);  // the q rebuild
    grid.sync();
    sweep_runs<true>(a, grid, f, 0, a.n_runs, warp, nwarp, lane);
  }
}

// ---- device: the streamed passes ---------------------------------------------------------------
// the sweep of w (V = false) or of factor f over the runs [r_lo, r_hi) of one block; with REL, of a relation block
template <bool V, bool REL = false>
__global__ void __launch_bounds__(256) mcmc_block_sweep_kernel(const SweepArgs a, uint32_t r_lo, uint32_t r_hi, int f) {
  cg::grid_group grid = cg::this_grid();
  const uint64_t tid = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint64_t nth = (uint64_t)gridDim.x * blockDim.x;
  sweep_runs<V, REL>(a, grid, f, r_lo, r_hi, (uint32_t)(tid >> 5), (uint32_t)(nth >> 5), threadIdx.x & 31);
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

// Per case: the e-term with the blocks' q_f and q of its rows added in relation order (:227-240, :352-368)
__global__ void __launch_bounds__(128)
    rel_eterm_kernel(Params64 p, int k, int use_w0, int use_w, uint64_t n_rows, const uint64_t* __restrict__ row_ptr,
                     const uint32_t* __restrict__ col, const float* __restrict__ val, const RelView* __restrict__ rel,
                     uint32_t n_rel, int side, double* __restrict__ e_out) {
  const double w0 = *p.w0();
  for (uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; c < n_rows; c += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t beg = row_ptr[c];
    RowOrder o;
    o.init(col + beg, (uint32_t)(row_ptr[c + 1] - beg));
    e_out[c] = case_eterm(
        o, p.v(), p.w(), k, use_w, use_w0, w0, val + beg,
        [&](int f, double& q) {
          for (uint32_t r = 0; r < n_rel; r++) q += rel[r].qf[(size_t)rel[r].join[side][c] * k + f];
        },
        [&](double& q) {
          for (uint32_t r = 0; r < n_rel; r++) q += rel[r].q[rel[r].join[side][c]];
        });
  }
}

}  // namespace

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

// The block in `slot` by case, stably: s.srt_key = the entries' cases, s.srt_pos = their positions.  The chain
// arguments for it.
std::string sort_block(fmb200_ctx* c, McmcState& s, const DataSlot& d, uint64_t n_cases, uint32_t col_lo, ChainArgs* a) {
  int bits = 1;
  while (bits < 32 && ((n_cases - 1) >> bits) != 0) bits++;
  size_t tmp = s.srt_tmp_bytes;
  MK(cub::DeviceRadixSort::SortPairs(s.srt_tmp.get(), tmp, d.col.get(), s.srt_key.get(), s.iota.get(), s.srt_pos.get(),
                                     d.nnz, 0, bits, c->stream));
  c->launches++;
  *a = ChainArgs{};
  a->key = s.srt_key.get();
  a->pos = s.srt_pos.get();
  a->nnz = d.nnz;
  a->col_ptr = d.row_ptr.get();
  a->n_cols = d.n_rows;
  a->col_lo = col_lo;
  a->val = d.val.get();
  a->v = c->p64.v();
  a->w = c->p64.w();
  a->k = c->k;
  return "";
}

template <int OP>
std::string chain(fmb200_ctx* c, const ChainArgs& a) {
  xt_case_kernel<OP><<<grid_for(c, a.nnz), 256, 0, c->stream>>>(a);
  c->launches++;
  MK(cudaGetLastError());
  return "";
}

// The e-terms of a streamed set into e[n] (fm_eterm64_kernel's sums, case by case in the same order):
// one pass per factor for parts (1) and (2), one for part (3); acc, acc2: two per-case chains.
std::string xt_eterms(fmb200_ctx* c, McmcState& s, XtSet& x, double* e, double* acc, double* acc2) {
  const uint64_t n = x.src.n_cases;
  if (n == 0) return "";
  MK(cudaMemsetAsync(e, 0, n * sizeof(double), c->stream));
  MK(cudaMemsetAsync(acc, 0, n * sizeof(double), c->stream));
  MK(cudaMemsetAsync(acc2, 0, n * sizeof(double), c->stream));
  for (int f = 0; f <= c->k; f++) {
    if (f == c->k && !c->k1) break;
    const std::string err = xt_pass(c, x, [&](int slot, uint64_t b) -> std::string {
      const DataSlot& d = c->slots[slot];
      if (d.nnz == 0) return "";
      ChainArgs a;
      std::string r = sort_block(c, s, d, n, x.col_lo[b], &a);
      if (!r.empty()) return r;
      a.f = f;
      a.q = acc;
      a.q2 = acc2;
      return f < c->k ? chain<CH_ETERM_V>(c, a) : chain<CH_ETERM_W>(c, a);
    });
    if (!err.empty()) return err;
    if (f < c->k) {
      eterm_factor_kernel<<<grid_for(c, n), 256, 0, c->stream>>>(e, acc, n);
      c->launches++;
    }
  }
  eterm_final_kernel<<<grid_for(c, n), 256, 0, c->stream>>>(e, acc2, n, c->k0, c->p64.w0());
  c->launches++;
  MK(cudaGetLastError());
  return "";
}

// The sweep over a streamed training set: pass -1 draws w, pass f draws factor f, block by block over the
// block's runs.  The q of factor f + 1 (which reads only v(f + 1, .), untouched by the sweep of f) is rebuilt on
// pass f into the other q array.
std::string xt_sweep(fmb200_ctx* c, McmcState& s, SweepArgs a) {
  XtSet& x = *s.xt[0];
  const uint64_t N = s.n_train;
  double* q[2] = {s.q_d.get(), s.q2_d.get()};
  for (int p = -1; p < a.k; p++) {
    const bool sweep = p >= 0 || a.use_w, rebuild = p + 1 < a.k;
    if (!sweep && !rebuild) continue;
    double* qn = rebuild ? q[(p + 1) % 2] : nullptr;
    if (rebuild) MK(cudaMemsetAsync(qn, 0, N * sizeof(double), c->stream));
    if (p >= 0) a.q = q[p % 2];
    const std::string err = xt_pass(c, x, [&](int slot, uint64_t b) -> std::string {
      const DataSlot& d = c->slots[slot];
      if (rebuild && d.nnz > 0) {
        ChainArgs ca;
        std::string r = sort_block(c, s, d, N, x.col_lo[b], &ca);
        if (r.empty()) {
          ca.f = p + 1;
          ca.q = qn;
          r = chain<CH_Q>(c, ca);
        }
        if (!r.empty()) return r;
      }
      uint32_t r_lo = x.run_lo[b], r_hi = x.run_lo[b + 1];
      if (sweep && r_lo < r_hi) {
        a.col_ptr = d.row_ptr.get();
        a.cs_case = d.col.get();
        a.cs_x = d.val.get();
        a.col_lo = x.col_lo[b];
        a.col_hi = x.col_lo[b + 1];
        int f = p < 0 ? 0 : p;
        void* args[] = {(void*)&a, (void*)&r_lo, (void*)&r_hi, (void*)&f};
        const void* fn = p < 0 ? (const void*)mcmc_block_sweep_kernel<false> : (const void*)mcmc_block_sweep_kernel<true>;
        MK(cudaLaunchCooperativeKernel(fn, dim3(s.grid), dim3(256), args, 0, c->stream));
        c->launches++;
      }
      return "";
    });
    if (!err.empty()) return err;
  }
  return "";
}

// The e-term pass with relations (fm_learn_mcmc.h:148-378) into e: side 0 (train) first computes every block
// row's y, q and q_f, which side 1 (test) reads as well
std::string rel_eterms(fmb200_ctx* c, McmcState& s, int side, double* e) {
  if (side == 0)
    for (const RelDev& r : s.rel) {
      rel_row_kernel<REL_ETERM><<<grid_for(c, r.rows), 256, 0, c->stream>>>(r.view(), c->p64.v(), c->p64.w(), c->k, 0,
                                                                            c->k1);
      c->launches++;
    }
  const DataSlot& d = c->slots[side == 0 ? s.train : s.test];
  if (d.n_rows > 0) {
    const int grid = (int)std::min<uint64_t>((d.n_rows + 127) / 128, (uint64_t)c->sm_count * 16);
    rel_eterm_kernel<<<grid, 128, 0, c->stream>>>(c->p64, c->k, c->k0, c->k1, d.n_rows, d.row_ptr.get(), d.col.get(),
                                                  d.val.get(), s.rel_d.get(), (uint32_t)s.rel.size(), side, e);
    c->launches++;
  }
  MK(cudaGetLastError());
  return "";
}

std::string repredict(fmb200_ctx* c, McmcState& s) {
  if (!s.rel.empty()) {
    const std::string err = rel_eterms(c, s, 0, s.e_d.get());
    if (!err.empty()) return err;
  } else if (s.xt[0]) {
    const std::string err = xt_eterms(c, s, *s.xt[0], s.e_d.get(), s.q_d.get(), s.q2_d.get());
    if (!err.empty()) return err;
  } else {
    MK(launch_mcmc_eterms(c, c->slots[s.train], s.e_d.get()));
  }
  if (!s.rel.empty()) {
    const std::string err = rel_eterms(c, s, 1, s.e_test_d.get());
    if (!err.empty()) return err;
  } else if (s.xt[1]) {
    const std::string err = xt_eterms(c, s, *s.xt[1], s.e_test_d.get(), s.xt[1]->acc[0].get(), s.xt[1]->acc[1].get());
    if (!err.empty()) return err;
  } else {
    MK(launch_mcmc_eterms(c, c->slots[s.test], s.e_test_d.get()));
  }
  MK(cudaMemcpyAsync(s.e.data(), s.e_d.get(), s.n_train * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  if (s.n_test) MK(cudaMemcpyAsync(s.e_test.data(), s.e_test_d.get(), s.n_test * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
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

// keys[n] (all below n_keys) stably sorted: keys_out, and the positions they came from in pos_out
std::string sort_by_key(fmb200_ctx* c, const uint32_t* keys, uint64_t n, uint64_t n_keys, DevPtr<uint32_t>& keys_out,
                        DevPtr<uint32_t>& pos_out) {
  DevPtr<uint32_t> iota;
  MK(alloc(keys_out, n));
  MK(alloc(pos_out, n));
  MK(alloc(iota, n));
  if (n == 0) return "";
  iota_kernel<<<grid_for(c, n), 256, 0, c->stream>>>(iota.get(), n);
  c->launches++;
  int bits = 1;
  while (bits < 32 && ((n_keys - 1) >> bits) != 0) bits++;
  size_t tmp_bytes = 0;
  MK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys, keys_out.get(), iota.get(), pos_out.get(), n, 0, bits,
                                     c->stream));
  DevPtr<unsigned char> tmp;
  MK(alloc(tmp, tmp_bytes));
  MK(cub::DeviceRadixSort::SortPairs(tmp.get(), tmp_bytes, keys, keys_out.get(), iota.get(), pos_out.get(), n, 0, bits,
                                     c->stream));
  c->launches++;
  MK(cudaStreamSynchronize(c->stream));  // iota and tmp are freed on return
  return "";
}

// A relation block on the device: its .xt, the row-major copy, the joins and the join inverse, #^R, and the
// block's part of the begin-time index (prev of its ids, dup of its columns)
std::string rel_upload(fmb200_ctx* c, McmcState& s, const RelationHost& h, RelDev& r, unsigned int* prev_d) {
  r.rows = h.num_cases;
  r.nf = h.num_feature;
  r.off = h.attr_offset;
  const uint64_t nnz = h.row.size(), k = (uint64_t)c->k;
  MK(alloc(r.col_ptr, r.nf + 1));
  MK(alloc(r.xt_row, nnz));
  MK(alloc(r.xt_val, nnz));
  MK(alloc(r.row_ptr, (uint64_t)r.rows + 1));
  MK(alloc(r.col, nnz));
  MK(alloc(r.val, nnz));
  MK(alloc(r.inv_ptr, (uint64_t)r.rows + 1));
  MK(alloc(r.cache, (7 + k) * r.rows));
  MK(cudaMemcpyAsync(r.col_ptr.get(), h.col_ptr.data(), (r.nf + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
  MK(cudaMemcpyAsync(r.xt_row.get(), h.row.data(), nnz * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
  MK(cudaMemcpyAsync(r.xt_val.get(), h.val.data(), nnz * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  MK(cudaMemsetAsync(r.cache.get(), 0, (7 + k) * r.rows * sizeof(double), c->stream));
  for (int side = 0; side < 2; side++) {
    MK(alloc(r.join[side], h.join[side].size()));
    MK(cudaMemcpyAsync(r.join[side].get(), h.join[side].data(), h.join[side].size() * sizeof(uint32_t),
                       cudaMemcpyHostToDevice, c->stream));
  }
  DevPtr<uint32_t> key, pos;
  std::string err = sort_by_key(c, r.xt_row.get(), nnz, r.rows, key, pos);
  if (!err.empty()) return err;
  if (nnz > 0) {
    rel_rowmajor_kernel<<<grid_for(c, nnz), 256, 0, c->stream>>>(pos.get(), nnz, r.col_ptr.get(), r.nf, r.off,
                                                                 r.xt_val.get(), r.col.get(), r.val.get());
    c->launches++;
  }
  mcmc_colptr_kernel<<<grid_for(c, (uint64_t)r.rows + 1), 256, 0, c->stream>>>(key.get(), nnz, r.rows, r.row_ptr.get());
  c->launches++;
  if (r.rows > 0) {
    rel_dup_kernel<<<grid_for(c, r.rows), 256, 0, c->stream>>>(r.row_ptr.get(), r.col.get(), r.rows, s.dup.get());
    mcmc_prev_kernel<<<grid_for(c, r.rows), 256, 0, c->stream>>>(r.row_ptr.get(), r.col.get(), r.rows, prev_d);
    c->launches += 2;
  }
  err = sort_by_key(c, r.join[0].get(), h.join[0].size(), r.rows, key, r.inv_case);
  if (!err.empty()) return err;
  mcmc_colptr_kernel<<<grid_for(c, (uint64_t)r.rows + 1), 256, 0, c->stream>>>(key.get(), h.join[0].size(), r.rows,
                                                                                r.inv_ptr.get());
  rel_wnum_kernel<<<grid_for(c, r.rows), 256, 0, c->stream>>>(r.view());
  c->launches += 2;
  MK(cudaGetLastError());
  MK(cudaStreamSynchronize(c->stream));
  return "";
}

// One iteration's sweep with relations (draw_all, fm_learn_mcmc.h:438-640 after draw_w0): the main table's runs,
// then per block the unsync, its runs over its rows and the resync; per factor first the q rebuild of the blocks'
// rows and of the cases
std::string rel_sweep(fmb200_ctx* c, McmcState& s, const SweepArgs& a) {
  const uint64_t N = s.n_train;
  auto sweep = [&](const SweepArgs& sa, bool v, bool rel, uint32_t r_lo, uint32_t r_hi, int f) -> cudaError_t {
    if (r_lo >= r_hi) return cudaSuccess;
    void* args[] = {(void*)&sa, (void*)&r_lo, (void*)&r_hi, (void*)&f};
    const void* fn = v ? (rel ? (const void*)mcmc_block_sweep_kernel<true, true> : (const void*)mcmc_block_sweep_kernel<true>)
                       : (rel ? (const void*)mcmc_block_sweep_kernel<false, true> : (const void*)mcmc_block_sweep_kernel<false>);
    c->launches++;
    return cudaLaunchCooperativeKernel(fn, dim3(s.grid), dim3(256), args, 0, c->stream);
  };
  auto block_args = [&](const RelDev& r) {
    const RelView rv = r.view();
    SweepArgs b = a;
    b.col_ptr = rv.col_ptr;
    b.col_lo = r.off;
    b.col_hi = r.off + r.nf;
    b.cs_case = rv.xt_row;
    b.cs_x = rv.xt_val;
    b.q = rv.q;
    b.wnum = rv.wnum;
    b.we = rv.we;
    b.weq = rv.weq;
    b.wc = rv.wc;
    b.wc_sqr = rv.wc_sqr;
    b.y = rv.y;
    return b;
  };
  if (a.shift) {
    mcmc_shift_kernel<<<grid_for(c, N), 256, 0, c->stream>>>(a.e, N, a.e_shift);
    c->launches++;
  }
  const uint32_t R = (uint32_t)s.rel.size();
  if (a.use_w) {
    MK(sweep(a, false, false, 0, s.rel_run[0], 0));
    for (uint32_t r = 0; r < R; r++) {
      const RelView rv = s.rel[r].view();
      rel_unsync_kernel<false><<<grid_for(c, rv.rows), 256, 0, c->stream>>>(rv, a.e, a.q);
      c->launches++;
      MK(sweep(block_args(s.rel[r]), false, true, s.rel_run[r], s.rel_run[r + 1], 0));
      rel_resync_kernel<false><<<grid_for(c, N), 256, 0, c->stream>>>(rv, a.e, a.q, N);
      c->launches++;
    }
  }
  for (int f = 0; f < a.k; f++) {
    for (uint32_t r = 0; r < R; r++) {
      rel_row_kernel<REL_Q><<<grid_for(c, s.rel[r].rows), 256, 0, c->stream>>>(s.rel[r].view(), a.v, a.w, a.k, f, 0);
      c->launches++;
    }
    rel_case_q_kernel<<<grid_for(c, N), 256, 0, c->stream>>>(a, f, s.rel_d.get(), R);
    c->launches++;
    MK(sweep(a, true, false, 0, s.rel_run[0], f));
    for (uint32_t r = 0; r < R; r++) {
      const RelView rv = s.rel[r].view();
      rel_unsync_kernel<true><<<grid_for(c, rv.rows), 256, 0, c->stream>>>(rv, a.e, a.q);
      c->launches++;
      MK(sweep(block_args(s.rel[r]), true, true, s.rel_run[r], s.rel_run[r + 1], f));
      rel_resync_kernel<true><<<grid_for(c, N), 256, 0, c->stream>>>(rv, a.e, a.q, N);
      c->launches++;
    }
  }
  MK(cudaGetLastError());
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
  if (!rel.empty()) {
    if (train_xt || test_xt) return "relations are not streamed";
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
  std::unique_ptr<XtSet> xt[2];
  if (train_xt) {
    const std::string e = xt_open(c, *train_xt, "train", &xt[0]);
    if (!e.empty()) return e;
  }
  if (test_xt) {
    const std::string e = xt_open(c, *test_xt, "test", &xt[1]);
    if (!e.empty()) return e;
  }
  {  // no slot may serve two purposes
    std::vector<int> used;
    used.push_back(train_xt ? train_xt->slot[0] : train);
    if (train_xt) used.push_back(train_xt->slot[1]);
    if (test_xt) {
      used.push_back(test_xt->slot[0]);
      used.push_back(test_xt->slot[1]);
    } else if (test != train) {
      used.push_back(test);
    }
    for (size_t i = 0; i < used.size(); i++)
      for (size_t j = 0; j < i; j++)
        if (used[i] == used[j]) return "a streamed set's slots must differ from every other slot in use";
  }
  const DataSlot* d = train_xt ? nullptr : &c->slots[train];
  const DataSlot* dt = test_xt ? nullptr : &c->slots[test];
  const uint64_t n_train = d ? d->n_rows : train_xt->n_cases, n_test = dt ? dt->n_rows : test_xt->n_cases;
  if (n_train == 0) return "the training set is empty";
  if (d && (d->n_rows >= 0xffffffffull || d->nnz >= 0xffffffffull))
    return "training sets of 2^32 cases or entries and more are not supported";
  if (G == 0) return "n_groups must be >= 1";
  c->mcmc.reset(new McmcState());
  McmcState& s = *c->mcmc;
  const uint32_t n = c->n;
  const int k = c->k;
  s.train = train;
  s.test = test;
  s.xt[0] = std::move(xt[0]);
  s.xt[1] = std::move(xt[1]);
  s.n_train = n_train;
  s.n_test = n_test;
  s.train_gen = d ? d->upload_gen : 0;
  s.test_gen = dt ? dt->upload_gen : 0;
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
  s.y.resize(n_train);
  s.y_test.resize(n_test);
  s.e.resize(n_train);
  s.e_test.resize(n_test);
  s.pred_this.assign(n_test, 0.0);
  s.pred_all.assign(n_test, 0.0);
  s.pred_but5.assign(n_test, 0.0);
  if (d) {
    MK(alloc(s.col_ptr, n + 1));
    MK(alloc(s.cs_case, d->nnz));
    MK(alloc(s.cs_x, d->nnz));
  }
  MK(alloc(s.dup, n));
  MK(alloc(s.group_d, n));
  MK(alloc(s.e_d, n_train));
  MK(alloc(s.q_d, n_train));
  MK(alloc(s.e_test_d, n_test));
  MK(alloc(s.z_d, (size_t)(k + 1) * n));
  MK(alloc(s.hyp_d, 2 * G + 2 * (size_t)G * k));
  MK(alloc(s.flag_d, F_WORDS));
  if (d) {
    MK(cudaMemcpyAsync(s.y.data(), d->target.get(), n_train * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    s.y_dev = d->target.get();
  } else {
    std::copy(train_xt->target, train_xt->target + n_train, s.y.begin());
    MK(alloc(s.y_d, n_train));
    MK(alloc(s.q2_d, n_train));
    MK(cudaMemcpyAsync(s.y_d.get(), s.y.data(), n_train * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    s.y_dev = s.y_d.get();
  }
  if (dt) {
    if (n_test) MK(cudaMemcpyAsync(s.y_test.data(), dt->target.get(), n_test * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  } else {
    std::copy(test_xt->target, test_xt->target + n_test, s.y_test.begin());
    for (auto& acc : s.xt[1]->acc) MK(alloc(acc, n_test));
  }
  if (s.xt[0] || s.xt[1]) {  // the by-case sort of the largest block
    uint64_t max_nnz = 1;
    for (const auto& x : s.xt)
      if (x) max_nnz = std::max(max_nnz, *std::max_element(x->nnz.begin(), x->nnz.end()));
    MK(alloc(s.srt_key, max_nnz));
    MK(alloc(s.srt_pos, max_nnz));
    MK(alloc(s.iota, max_nnz));
    iota_kernel<<<grid_for(c, max_nnz), 256, 0, c->stream>>>(s.iota.get(), max_nnz);
    c->launches++;
    MK(cub::DeviceRadixSort::SortPairs(nullptr, s.srt_tmp_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                       (const uint32_t*)nullptr, (uint32_t*)nullptr, max_nnz, 0, 32, c->stream));
    MK(alloc(s.srt_tmp, s.srt_tmp_bytes ? s.srt_tmp_bytes : 1));
  }
  MK(cudaMemcpyAsync(s.group_d.get(), s.group.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
  MK(cudaMemsetAsync(s.dup.get(), 0, n * sizeof(uint32_t), c->stream));

  // transposed training data + feature runs, from the (id, entry) sort of the ORDERED index, or from one pass
  // over the streamed .xt
  std::vector<uint32_t> prev(n, 0u);
  if (s.xt[0]) {
    DevPtr<unsigned int> prev_d;
    DevPtr<uint32_t> last;
    MK(alloc(prev_d, n ? n : 1));
    MK(alloc(last, n_train));
    MK(cudaMemsetAsync(prev_d.get(), 0, n * sizeof(unsigned int), c->stream));
    MK(cudaMemsetAsync(last.get(), 0, n_train * sizeof(uint32_t), c->stream));
    const std::string err = xt_pass(c, *s.xt[0], [&](int slot, uint64_t b) -> std::string {
      const DataSlot& blk = c->slots[slot];
      if (blk.nnz == 0) return "";
      ChainArgs a;
      const std::string r = sort_block(c, s, blk, n_train, s.xt[0]->col_lo[b], &a);
      if (!r.empty()) return r;
      a.last = last.get();
      a.prev = prev_d.get();
      a.dup = s.dup.get();
      return chain<CH_PREV>(c, a);
    });
    if (!err.empty()) return err;
    MK(cudaMemcpyAsync(prev.data(), prev_d.get(), n * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
    MK(cudaStreamSynchronize(c->stream));
  } else if (d->nnz > 0) {
    DataSlot& dm = c->slots[train];
    SortedEntries se;
    MK(build_ordered_links(c, dm, &se));
    mcmc_csc_kernel<<<grid_for(c, dm.nnz), 256, 0, c->stream>>>(se.ids, se.ent, dm.nnz, dm.row_ptr.get(), dm.n_rows,
                                                                dm.val.get(), s.cs_case.get(), s.cs_x.get(), s.dup.get());
    mcmc_colptr_kernel<<<grid_for(c, (uint64_t)n + 1), 256, 0, c->stream>>>(se.ids, dm.nnz, n, s.col_ptr.get());
    DevPtr<unsigned int> prev_d;
    MK(alloc(prev_d, n));
    MK(cudaMemsetAsync(prev_d.get(), 0, n * sizeof(unsigned int), c->stream));
    mcmc_prev_kernel<<<grid_for(c, dm.n_rows), 256, 0, c->stream>>>(dm.row_ptr.get(), dm.col.get(), dm.n_rows, prev_d.get());
    c->launches += 3;
    MK(cudaGetLastError());
    MK(cudaMemcpyAsync(prev.data(), prev_d.get(), n * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
    MK(cudaStreamSynchronize(c->stream));
  } else {
    MK(cudaMemsetAsync(s.col_ptr.get(), 0, (n + 1) * sizeof(uint64_t), c->stream));
  }
  MK(cudaStreamSynchronize(c->stream));
  if (!rel.empty()) {  // the blocks' ids: prev from the blocks' rows
    DevPtr<unsigned int> prev_d;
    MK(alloc(prev_d, n));
    MK(cudaMemsetAsync(prev_d.get(), 0, n * sizeof(unsigned int), c->stream));
    s.rel.resize(rel.size());
    std::vector<RelView> views;
    for (size_t r = 0; r < rel.size(); r++) {
      const std::string err = rel_upload(c, s, rel[r], s.rel[r], prev_d.get());
      if (!err.empty()) return err;
      views.push_back(s.rel[r].view());
    }
    const uint32_t off0 = rel[0].attr_offset;
    MK(cudaMemcpyAsync(prev.data() + off0, prev_d.get() + off0, (n - off0) * sizeof(unsigned int),
                       cudaMemcpyDeviceToHost, c->stream));
    MK(alloc(s.rel_d, views.size()));
    MK(cudaMemcpyAsync(s.rel_d.get(), views.data(), views.size() * sizeof(RelView), cudaMemcpyHostToDevice, c->stream));
    MK(cudaStreamSynchronize(c->stream));
  }
  // cut greedily: j opens a new run when it shares a case with a feature of the current run; a streamed set
  // also cuts at every block start, so that a run never spans two blocks, and relational data at every relation
  // block's first id
  std::vector<bool> block_start(n, false);
  if (s.xt[0])
    for (uint64_t b = 1; b < s.xt[0]->n_blocks(); b++)
      if (s.xt[0]->col_lo[b] < n) block_start[s.xt[0]->col_lo[b]] = true;
  for (const RelationHost& h : rel)
    if (h.attr_offset < n) block_start[h.attr_offset] = true;
  s.runs.clear();
  if (n > 0) s.runs.push_back(0);
  for (uint32_t j = 1; j < n; j++)
    if ((prev[j] != 0 && prev[j] - 1 >= s.runs.back()) || block_start[j]) s.runs.push_back(j);
  s.runs.push_back(n);
  if (s.xt[0]) {  // block b sweeps the runs that start in its columns; the last block also the features after them
    XtSet& x = *s.xt[0];
    x.run_lo.resize(x.n_blocks() + 1);
    for (uint64_t b = 0; b < x.n_blocks(); b++)
      x.run_lo[b] = (uint32_t)(std::lower_bound(s.runs.begin(), s.runs.end() - 1, x.col_lo[b]) - s.runs.begin());
    x.run_lo[x.n_blocks()] = (uint32_t)s.runs.size() - 1;
  }
  for (const RelationHost& h : rel)
    s.rel_run.push_back((uint32_t)(std::lower_bound(s.runs.begin(), s.runs.end() - 1, h.attr_offset) - s.runs.begin()));
  if (!rel.empty()) s.rel_run.push_back((uint32_t)s.runs.size() - 1);
  MK(alloc(s.runs_d, s.runs.size()));
  MK(cudaMemcpyAsync(s.runs_d.get(), s.runs.data(), s.runs.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));

  int occ = 0, occ_w = 0, occ_v = 0;
  MK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, mcmc_sweep_kernel, 256, 0));
  MK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_w, mcmc_block_sweep_kernel<false>, 256, 0));
  MK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_v, mcmc_block_sweep_kernel<true>, 256, 0));
  if (s.xt[0] || !rel.empty()) occ = std::min(occ_w, occ_v);
  if (!rel.empty()) {
    int occ_wr = 0, occ_vr = 0;
    MK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_wr, mcmc_block_sweep_kernel<false, true>, 256, 0));
    MK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_vr, mcmc_block_sweep_kernel<true, true>, 256, 0));
    occ = std::min(occ, std::min(occ_wr, occ_vr));
  }
  if (occ < 1) return "the sweep kernel does not fit an SM";
  s.grid = occ * c->sm_count;

  // fm_learn_mcmc_simultaneous.h:69-86: predict, then e := prediction - target (both tasks)
  const std::string err = repredict(c, s);
  if (!err.empty()) return err;
  for (uint64_t i = 0; i < n_train; i++) s.e[i] = s.e[i] - s.y[i];
  MK(cudaMemcpyAsync(s.e_d.get(), s.e.data(), n_train * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  MK(cudaStreamSynchronize(c->stream));
  s.state.resize(c->p64.n_doubles);
  s.z.resize((size_t)(k + 1) * n);
  s.hyp.resize(2 * G + 2 * (size_t)G * k);
  return "";
}

std::string mcmc_iteration(fmb200_ctx* c, double* train_metric, uint32_t* counters) {
  McmcState& s = *c->mcmc;
  if ((!s.xt[0] && c->slots[s.train].upload_gen != s.train_gen) || (!s.xt[1] && c->slots[s.test].upload_gen != s.test_gen))
    return "the train or test slot was re-uploaded: call fmb200_mcmc_begin again";
  const uint32_t n = c->n, G = s.G;
  const int k = c->k;
  const uint64_t N = s.n_train, NT = s.n_test;
  const bool sample = s.sample, ml = s.multilevel;
  uint32_t* cnt = s.counters;  // nan, inf of: alpha, w0, w, v, w_mu, w_lambda, v_mu, v_lambda
  std::fill(cnt, cnt + 16, 0u);
  MK(cudaMemcpyAsync(s.state.data(), c->p64.base, s.state.size() * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  MK(cudaMemsetAsync(s.flag_d.get(), 0, F_SKIP * sizeof(unsigned int), c->stream));
  MK(cudaMemsetAsync(s.flag_d.get() + F_SKIP, 0xff, sizeof(unsigned int), c->stream));
  MK(cudaStreamSynchronize(c->stream));
  double& w0 = s.state[0];
  const double* w = s.state.data() + Params64::off_w;
  const double* v = s.state.data() + c->p64.off_v;  // [n][k]

  // draw_alpha, fm_learn_mcmc.h:911-939
  if (!ml) {
    s.alpha = kAlpha0;
  } else {
    const double alpha_n = kAlpha0 + N;
    double gamma_n = kGamma0;
    for (uint64_t i = 0; i < N; i++) gamma_n += s.e[i] * s.e[i];
    reject_nonfinite(s.alpha, ran_gamma(alpha_n / 2.0, gamma_n / 2.0), cnt, 0);
  }
  const double alpha = s.alpha;
  // draw_w0, :643-683
  bool shift = false;
  double e_shift = 0.0;
  if (c->k0) {
    double mean = 0;
    for (uint64_t i = 0; i < N; i++) mean += s.e[i] - w0;
    const double sig = (double)1.0 / (s.reg0 + alpha * N);
    mean = -sig * (alpha * mean - kW0Mean0 * s.reg0);
    const double old = w0;
    if (!reject_nonfinite(w0, sample ? ran_gaussian(mean, std::sqrt(sig)) : mean, cnt, 2)) {
      shift = true;
      e_shift = old - w0;
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

  // the sweep
  std::copy(s.w_mu.begin(), s.w_mu.end(), s.hyp.begin());
  std::copy(s.w_lambda.begin(), s.w_lambda.end(), s.hyp.begin() + G);
  std::copy(s.v_mu.begin(), s.v_mu.end(), s.hyp.begin() + 2 * G);
  std::copy(s.v_lambda.begin(), s.v_lambda.end(), s.hyp.begin() + 2 * G + (size_t)G * k);
  MK(cudaMemcpyAsync(c->p64.w0(), &w0, sizeof(double), cudaMemcpyHostToDevice, c->stream));
  MK(cudaMemcpyAsync(s.hyp_d.get(), s.hyp.data(), s.hyp.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  if (sample) MK(cudaMemcpyAsync(s.z_d.get(), s.z.data(), s.z.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  SweepArgs a{};
  if (!s.xt[0]) {
    const DataSlot& d = c->slots[s.train];
    a.col_ptr = s.col_ptr.get();
    a.col_lo = 0;
    a.col_hi = n;
    a.cs_case = s.cs_case.get();
    a.cs_x = s.cs_x.get();
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
  a.n_rows = N;
  a.e = s.e_d.get();
  a.q = s.q_d.get();
  a.w = c->p64.w();
  a.v = c->p64.v();
  a.k = k;
  a.use_w = c->k1;
  a.sample = sample;
  a.shift = shift;
  a.alpha = alpha;
  a.e_shift = e_shift;
  a.z = s.z_d.get();
  a.hyp = s.hyp_d.get();
  a.flag = s.flag_d.get();
  if (!s.rel.empty()) {
    const std::string err = rel_sweep(c, s, a);
    if (!err.empty()) return err;
  } else if (s.xt[0]) {
    if (shift) {
      mcmc_shift_kernel<<<grid_for(c, N), 256, 0, c->stream>>>(s.e_d.get(), N, e_shift);
      c->launches++;
    }
    const std::string err = xt_sweep(c, s, a);
    if (!err.empty()) return err;
  } else if (a.shift || a.use_w || k > 0) {
    void* args[] = {(void*)&a};
    MK(cudaLaunchCooperativeKernel((const void*)mcmc_sweep_kernel, dim3(s.grid), dim3(256), args, 0, c->stream));
    c->launches++;
  }
  unsigned int flag[F_WORDS];
  MK(cudaMemcpyAsync(flag, s.flag_d.get(), sizeof(flag), cudaMemcpyDeviceToHost, c->stream));
  MK(cudaStreamSynchronize(c->stream));
  cnt[4] = flag[F_NAN_W];
  cnt[5] = flag[F_INF_W];
  cnt[6] = flag[F_NAN_V];
  cnt[7] = flag[F_INF_V];
  if (flag[F_SKIP] != 0xffffffffu) {
    char buf[160];
    if (flag[F_SKIP] == 0) snprintf(buf, sizeof(buf), "iteration %u: a draw of w has a non-finite or zero posterior variance", s.iter);
    else snprintf(buf, sizeof(buf), "iteration %u: a draw of v[f=%u] has a non-finite or zero posterior variance", s.iter, flag[F_SKIP] - 1);
    return std::string(buf) + " (the model state diverged; sampling stops instead of desynchronising the random stream)";
  }

  // re-prediction and the target step, fm_learn_mcmc_simultaneous.h:122-200
  std::string err = repredict(c, s);
  if (!err.empty()) return err;
  const uint32_t i = s.iter;
  const double lo = c->hp.min_target, hi = c->hp.max_target;
  if (c->hp.task == FMB200_TASK_REGRESSION) {
    for (uint64_t t = 0; t < NT; t++) {
      double p = s.e_test[t];
      s.pred_this[t] = p;
      p = std::min(hi, p);
      p = std::max(lo, p);
      s.pred_all[t] += p;
      if (i >= 5) s.pred_but5[t] += p;
    }
    double rmse = 0.0;
    for (uint64_t t = 0; t < N; t++) {
      double p = s.e[t];
      p = std::min(hi, p);
      p = std::max(lo, p);
      const double er = p - s.y[t];
      rmse += er * er;
    }
    *train_metric = std::sqrt(rmse / N);
    mcmc_residual_kernel<<<grid_for(c, N), 256, 0, c->stream>>>(s.e_d.get(), s.y_dev, N);
    c->launches++;
    MK(cudaGetLastError());
    for (uint64_t t = 0; t < N; t++) s.e[t] = s.e[t] - s.y[t];
  } else {
    for (uint64_t t = 0; t < NT; t++) {
      const double p = cdf_gaussian(s.e_test[t]);
      s.pred_this[t] = p;
      s.pred_all[t] += p;
      if (i >= 5) s.pred_but5[t] += p;
    }
    uint64_t acc = 0;
    for (uint64_t t = 0; t < N; t++) {
      const double p = cdf_gaussian(s.e[t]);
      if (((p >= 0.5) && (s.y[t] > 0.0)) || ((p < 0.5) && (s.y[t] < 0.0))) acc++;
      const double mu = s.e[t];
      double st;
      if (s.y[t] >= 0.0) {
        if (sample) {
          st = ran_left_tgaussian(0.0, mu, 1.0);
        } else {
          const double phi = std::exp(-mu * mu / 2.0) / std::sqrt(3.141 * 2);
          st = mu + phi / (1 - cdf_gaussian(-mu));
        }
      } else {
        if (sample) {
          st = ran_right_tgaussian(0.0, mu, 1.0);
        } else {
          const double phi = std::exp(-mu * mu / 2.0) / std::sqrt(3.141 * 2);
          st = mu - phi / cdf_gaussian(-mu);
        }
      }
      s.e[t] = s.e[t] - st;
    }
    *train_metric = (double)acc / N;
    MK(cudaMemcpyAsync(s.e_d.get(), s.e.data(), N * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  }
  MK(cudaStreamSynchronize(c->stream));
  s.iter++;
  if (counters) std::copy(cnt, cnt + 16, counters);
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
