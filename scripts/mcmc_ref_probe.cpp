// scripts/mcmc_ref_probe.cpp -- offline probe of the reference's MCMC / ALS learner, compiled by
// scripts/make_mcmc_golden.py against the UNMODIFIED reference headers (include path only; nothing
// of the reference is copied here).  It runs fm_learn_mcmc_simultaneous::learn on in-memory CSR data
// exactly as libfm.cpp:115-116,245-289,326-364 sets it up and returns the state after the last
// iteration: model, hyperparameters, NaN/Inf counters, the test prediction sums and the #Iter lines.
#include <stdint.h>

// include order matters: the reference headers are not self-contained
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iomanip>
#include <iostream>
#include <iterator>
#include <sstream>
#include <string>

#include "util/util.h"
#include "fm_core/fm_model.h"
#include "libfm/src/Data.h"
#include "libfm/src/fm_learn.h"
#include "libfm/src/fm_learn_mcmc_simultaneous.h"

namespace {

struct DataProbe : public Data {
  DataProbe() : Data(0, true, true) {}
  void make_t() { create_data_t(); }
};

// the test prediction sums are protected members
struct Learner : public fm_learn_mcmc_simultaneous {
  DVector<double>& p_this() { return pred_this; }
  DVector<double>& p_all() { return pred_sum_all; }
  DVector<double>& p_but5() { return pred_sum_all_but5; }
};

DataProbe* make_data(uint64_t n_rows, const uint64_t* rp, const uint32_t* col, const float* val, const float* y,
                     int num_feature) {
  DataProbe* d = new DataProbe();
  LargeSparseMatrixMemory<DATA_FLOAT>* m = new LargeSparseMatrixMemory<DATA_FLOAT>();
  d->data = m;
  const uint64_t nnz = rp[n_rows];
  sparse_entry<DATA_FLOAT>* ent = new sparse_entry<DATA_FLOAT>[nnz > 0 ? nnz : 1];
  for (uint64_t j = 0; j < nnz; j++) {
    ent[j].id = col[j];
    ent[j].value = val[j];
  }
  m->data.setSize(n_rows);
  for (uint64_t i = 0; i < n_rows; i++) {
    m->data.value[i].data = ent + rp[i];
    m->data.value[i].size = (uint)(rp[i + 1] - rp[i]);
  }
  m->num_cols = num_feature;
  m->num_values = nnz;
  d->target.setSize(n_rows);
  for (uint64_t i = 0; i < n_rows; i++) d->target.value[i] = y[i];
  d->num_feature = num_feature;
  d->num_cases = n_rows;
  d->make_t();
  return d;
}

}  // namespace

extern "C" int probe_mcmc(uint32_t n, int k, int k0, int k1, double init_stdev, long seed,
                          uint64_t n_tr, const uint64_t* tr_rp, const uint32_t* tr_col, const float* tr_val,
                          const float* tr_y, int tr_nf, uint64_t n_te, const uint64_t* te_rp, const uint32_t* te_col,
                          const float* te_val, const float* te_y, int te_nf, int task, int do_sample,
                          int do_multilevel, uint32_t G, const uint32_t* group, const uint32_t* per_group, double reg0,
                          const double* w_lambda0, const double* v_lambda0, int num_iter, double min_target,
                          double max_target, double* init_state, double* state, double* hyper, uint32_t* counters,
                          double* pred, char* out, int out_len) {
  std::ostringstream sink;
  std::streambuf* saved = std::cout.rdbuf(sink.rdbuf());
  int rc = 0;
  try {
    DataProbe* train = make_data(n_tr, tr_rp, tr_col, tr_val, tr_y, tr_nf);
    DataProbe* test = make_data(n_te, te_rp, te_col, te_val, te_y, te_nf);
    srand(seed);
    fm_model fm;
    fm.num_attribute = n;
    fm.init_stdev = init_stdev;
    fm.k0 = k0 != 0;
    fm.k1 = k1 != 0;
    fm.num_factor = k;
    fm.init();
    fm.w.init_normal(fm.init_mean, fm.init_stdev);
    // state layout: w0 | w[n] | v[k][n]
    init_state[0] = fm.w0;
    memcpy(init_state + 1, fm.w.value, sizeof(double) * n);
    if (k > 0) memcpy(init_state + 1 + n, fm.v.value[0], sizeof(double) * (size_t)n * k);
    DataMetaInfo meta(n);
    for (uint32_t i = 0; i < n; i++) meta.attr_group(i) = group[i];
    meta.num_attr_groups = G;
    meta.num_attr_per_group.setSize(G);
    for (uint32_t g = 0; g < G; g++) meta.num_attr_per_group(g) = per_group[g];
    meta.num_relations = 0;
    Learner l;
    l.fm = &fm;
    l.meta = &meta;
    l.validation = NULL;
    l.num_iter = num_iter;
    l.num_eval_cases = test->num_cases;
    l.do_sample = do_sample != 0;
    l.do_multilevel = do_multilevel != 0;
    l.max_target = max_target;
    l.min_target = min_target;
    l.task = task;
    l.log = NULL;
    l.init();
    fm.reg0 = reg0;
    for (uint32_t g = 0; g < G; g++) l.w_lambda(g) = w_lambda0[g];
    for (uint32_t g = 0; g < G; g++)
      for (int f = 0; f < k; f++) l.v_lambda(g, f) = v_lambda0[(size_t)g * k + f];
    l.learn(*train, *test);
    state[0] = fm.w0;
    memcpy(state + 1, fm.w.value, sizeof(double) * n);
    if (k > 0) memcpy(state + 1 + n, fm.v.value[0], sizeof(double) * (size_t)n * k);
    // hyper: alpha | w_mu[G] | w_lambda[G] | v_mu[G][k] | v_lambda[G][k]
    size_t o = 0;
    hyper[o++] = l.alpha;
    for (uint32_t g = 0; g < G; g++) hyper[o++] = l.w_mu(g);
    for (uint32_t g = 0; g < G; g++) hyper[o++] = l.w_lambda(g);
    for (uint32_t g = 0; g < G; g++)
      for (int f = 0; f < k; f++) hyper[o++] = l.v_mu(g, f);
    for (uint32_t g = 0; g < G; g++)
      for (int f = 0; f < k; f++) hyper[o++] = l.v_lambda(g, f);
    const uint32_t c[16] = {l.nan_cntr_alpha, l.inf_cntr_alpha, l.nan_cntr_w0, l.inf_cntr_w0, l.nan_cntr_w,
                            l.inf_cntr_w, l.nan_cntr_v, l.inf_cntr_v, l.nan_cntr_w_mu, l.inf_cntr_w_mu,
                            l.nan_cntr_w_lambda, l.inf_cntr_w_lambda, l.nan_cntr_v_mu, l.inf_cntr_v_mu,
                            l.nan_cntr_v_lambda, l.inf_cntr_v_lambda};
    memcpy(counters, c, sizeof(c));
    for (uint64_t t = 0; t < n_te; t++) {
      pred[t] = l.p_this()(t);
      pred[n_te + t] = l.p_all()(t);
      pred[2 * n_te + t] = l.p_but5()(t);
    }
  } catch (...) {
    rc = 1;
  }
  std::cout.rdbuf(saved);
  snprintf(out, out_len, "%s", sink.str().c_str());
  return rc;
}
