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
// Each draw needs one standard normal; the host draws them in the reference's order before the
// launch.  A sampled draw the reference would skip without consuming one (posterior variance
// not finite, or stdev 0) cannot arise from a finite state; the device flags it and the
// iteration fails instead of desynchronising the stream.
// This TU is compiled with --fmad=false: every product and sum rounds as the reference's do.
#include <cooperative_groups.h>

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

struct McmcState {
  int train = 0, test = 1;
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
  // device
  DevPtr<uint32_t> col_ptr, cs_case, dup, group_d, runs_d;
  DevPtr<float> cs_x;
  DevPtr<double> e_d, q_d, e_test_d, z_d, hyp_d;
  DevPtr<unsigned int> flag_d;
  int grid = 0;
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

__global__ void mcmc_colptr_kernel(const uint32_t* __restrict__ ids, uint64_t nnz, uint32_t n, uint32_t* col_ptr) {
  for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j <= n; j += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t lo = 0, hi = nnz;  // first position with id >= j
    while (lo < hi) {
      const uint64_t mid = (lo + hi) >> 1;
      if (ids[mid] < j) lo = mid + 1;
      else hi = mid;
    }
    col_ptr[j] = (uint32_t)lo;
  }
}

__global__ void mcmc_residual_kernel(double* e, const float* __restrict__ y, uint64_t n) {
  for (uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; c < n; c += (uint64_t)gridDim.x * blockDim.x)
    e[c] = e[c] - y[c];
}

// ---- device: the sweep -----------------------------------------------------------------------
struct SweepArgs {
  const uint32_t* col_ptr;
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
};

// draw_w (fm_learn_mcmc.h:685-732) / draw_v (:792-847) of feature j, one warp
template <bool V>
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
  const uint32_t beg = a.col_ptr[j], end = a.col_ptr[j + 1];
  double m = 0.0, s = 0.0;
  for (uint32_t b = beg; b < end; b += 32) {
    const uint32_t idx = b + lane;
    double tm = 0.0, ts = 0.0;
    if (idx < end) {
      const uint32_t c = a.cs_case[idx];
      const float x = a.cs_x[idx];
      const double xd = (double)x;
      if (V) {
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
  if (V) m -= old * s;
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
    if (V) {
      const double h = xd * (a.q[c] - xd * old);
      a.q[c] -= xd * d;
      a.e[c] -= h * d;
    } else {
      a.e[c] -= xd * d;
    }
  }
}

template <bool V>
__device__ void sweep_runs(const SweepArgs& a, cg::grid_group& grid, int f, uint32_t warp, uint32_t nwarp, int lane) {
  for (uint32_t r = 0; r < a.n_runs; r++) {
    const uint32_t j1 = a.runs[r + 1];
    for (uint32_t j = a.runs[r] + warp; j < j1; j += nwarp) draw_feature<V>(a, j, f, lane);
    grid.sync();
  }
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
  if (a.use_w) sweep_runs<false>(a, grid, 0, warp, nwarp, lane);
  for (int f = 0; f < a.k; f++) {
    for (uint64_t c = tid; c < a.n_rows; c += nth) {  // the q rebuild (add_main_q, :406-428)
      const uint64_t beg = a.row_ptr[c];
      RowOrder o;
      o.init(a.col + beg, (uint32_t)(a.row_ptr[c + 1] - beg));
      a.q[c] = row_q(o, a.v, a.k, f, a.val + beg);
    }
    grid.sync();
    sweep_runs<true>(a, grid, f, warp, nwarp, lane);
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

std::string repredict(fmb200_ctx* c, McmcState& s) {
  const DataSlot& tr = c->slots[s.train];
  const DataSlot& te = c->slots[s.test];
  MK(launch_mcmc_eterms(c, tr, s.e_d.get()));
  MK(launch_mcmc_eterms(c, te, s.e_test_d.get()));
  MK(cudaMemcpyAsync(s.e.data(), s.e_d.get(), tr.n_rows * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  if (te.n_rows) MK(cudaMemcpyAsync(s.e_test.data(), s.e_test_d.get(), te.n_rows * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  MK(cudaStreamSynchronize(c->stream));
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

}  // namespace

std::string mcmc_begin(fmb200_ctx* c, int train, int test, int do_sample, int do_multilevel, uint32_t G,
                       const uint32_t* attr_group, const uint32_t* attr_per_group, double reg0,
                       const double* w_lambda0, const double* v_lambda0) {
  DataSlot& d = c->slots[train];
  const DataSlot& dt = c->slots[test];
  if (d.n_rows == 0) return "the training set is empty";
  if (d.n_rows >= 0xffffffffull || d.nnz >= 0xffffffffull) return "training sets of 2^32 cases or entries and more are not supported";
  if (G == 0) return "n_groups must be >= 1";
  c->mcmc.reset(new McmcState());
  McmcState& s = *c->mcmc;
  const uint32_t n = c->n;
  const int k = c->k;
  s.train = train;
  s.test = test;
  s.train_gen = d.upload_gen;
  s.test_gen = dt.upload_gen;
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
  s.y.resize(d.n_rows);
  s.y_test.resize(dt.n_rows);
  s.e.resize(d.n_rows);
  s.e_test.resize(dt.n_rows);
  s.pred_this.assign(dt.n_rows, 0.0);
  s.pred_all.assign(dt.n_rows, 0.0);
  s.pred_but5.assign(dt.n_rows, 0.0);
  MK(alloc(s.col_ptr, n + 1));
  MK(alloc(s.cs_case, d.nnz));
  MK(alloc(s.cs_x, d.nnz));
  MK(alloc(s.dup, n));
  MK(alloc(s.group_d, n));
  MK(alloc(s.e_d, d.n_rows));
  MK(alloc(s.q_d, d.n_rows));
  MK(alloc(s.e_test_d, dt.n_rows));
  MK(alloc(s.z_d, (size_t)(k + 1) * n));
  MK(alloc(s.hyp_d, 2 * G + 2 * (size_t)G * k));
  MK(alloc(s.flag_d, F_WORDS));
  MK(cudaMemcpyAsync(s.y.data(), d.target.get(), d.n_rows * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  if (dt.n_rows) MK(cudaMemcpyAsync(s.y_test.data(), dt.target.get(), dt.n_rows * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  MK(cudaMemcpyAsync(s.group_d.get(), s.group.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
  MK(cudaMemsetAsync(s.dup.get(), 0, n * sizeof(uint32_t), c->stream));

  // transposed training data + feature runs, from the (id, entry) sort of the ORDERED index
  std::vector<uint32_t> prev(n, 0u);
  if (d.nnz > 0) {
    SortedEntries se;
    MK(build_ordered_links(c, d, &se));
    mcmc_csc_kernel<<<grid_for(c, d.nnz), 256, 0, c->stream>>>(se.ids, se.ent, d.nnz, d.row_ptr.get(), d.n_rows,
                                                               d.val.get(), s.cs_case.get(), s.cs_x.get(), s.dup.get());
    mcmc_colptr_kernel<<<grid_for(c, (uint64_t)n + 1), 256, 0, c->stream>>>(se.ids, d.nnz, n, s.col_ptr.get());
    DevPtr<unsigned int> prev_d;
    MK(alloc(prev_d, n));
    MK(cudaMemsetAsync(prev_d.get(), 0, n * sizeof(unsigned int), c->stream));
    mcmc_prev_kernel<<<grid_for(c, d.n_rows), 256, 0, c->stream>>>(d.row_ptr.get(), d.col.get(), d.n_rows, prev_d.get());
    c->launches += 3;
    MK(cudaGetLastError());
    MK(cudaMemcpyAsync(prev.data(), prev_d.get(), n * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
    MK(cudaStreamSynchronize(c->stream));
  } else {
    MK(cudaMemsetAsync(s.col_ptr.get(), 0, (n + 1) * sizeof(uint32_t), c->stream));
  }
  MK(cudaStreamSynchronize(c->stream));
  // cut greedily: j opens a new run when it shares a case with a feature of the current run
  s.runs.clear();
  if (n > 0) s.runs.push_back(0);
  for (uint32_t j = 1; j < n; j++)
    if (prev[j] != 0 && prev[j] - 1 >= s.runs.back()) s.runs.push_back(j);
  s.runs.push_back(n);
  MK(alloc(s.runs_d, s.runs.size()));
  MK(cudaMemcpyAsync(s.runs_d.get(), s.runs.data(), s.runs.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));

  int occ = 0;
  MK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, mcmc_sweep_kernel, 256, 0));
  if (occ < 1) return "the sweep kernel does not fit an SM";
  s.grid = occ * c->sm_count;

  // fm_learn_mcmc_simultaneous.h:69-86: predict, then e := prediction - target (both tasks)
  const std::string err = repredict(c, s);
  if (!err.empty()) return err;
  for (uint64_t i = 0; i < d.n_rows; i++) s.e[i] = s.e[i] - s.y[i];
  MK(cudaMemcpyAsync(s.e_d.get(), s.e.data(), d.n_rows * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  MK(cudaStreamSynchronize(c->stream));
  s.state.resize(c->p64.n_doubles);
  s.z.resize((size_t)(k + 1) * n);
  s.hyp.resize(2 * G + 2 * (size_t)G * k);
  return "";
}

std::string mcmc_iteration(fmb200_ctx* c, double* train_metric, uint32_t* counters) {
  McmcState& s = *c->mcmc;
  const DataSlot& d = c->slots[s.train];
  const DataSlot& dt = c->slots[s.test];
  if (d.upload_gen != s.train_gen || dt.upload_gen != s.test_gen)
    return "the train or test slot was re-uploaded: call fmb200_mcmc_begin again";
  const uint32_t n = c->n, G = s.G;
  const int k = c->k;
  const uint64_t N = d.n_rows;
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
  a.col_ptr = s.col_ptr.get();
  a.cs_case = s.cs_case.get();
  a.cs_x = s.cs_x.get();
  a.dup = s.dup.get();
  a.group = s.group_d.get();
  a.runs = s.runs_d.get();
  a.n_runs = (uint32_t)s.runs.size() - 1;
  a.n = n;
  a.G = G;
  a.row_ptr = d.row_ptr.get();
  a.col = d.col.get();
  a.val = d.val.get();
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
  if (a.shift || a.use_w || k > 0) {
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
    for (uint64_t t = 0; t < dt.n_rows; t++) {
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
    mcmc_residual_kernel<<<grid_for(c, N), 256, 0, c->stream>>>(s.e_d.get(), d.target.get(), N);
    c->launches++;
    MK(cudaGetLastError());
    for (uint64_t t = 0; t < N; t++) s.e[t] = s.e[t] - s.y[t];
  } else {
    for (uint64_t t = 0; t < dt.n_rows; t++) {
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
