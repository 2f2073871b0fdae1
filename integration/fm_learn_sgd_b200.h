// fm_learn_sgd_b200.h -- the reference-side binding of libfmb200 (include/fmb200.h).
//
// Drop this header next to the reference's fm_learn_sgd_element.h and select the class
// at libfm.cpp:272 (`fml = new fm_learn_sgd_b200();`, see integration/build_patched.sh):
// the reference keeps its own main(), CMDLine, Data loader, RLog, fm_model and model /
// prediction writers; only the passes over the data move to the GPU.  It is written
// against the reference's own types (Data, DVector, LargeSparseMatrix*, fm_learn_sgd) and
// is compiled by oracle/Makefile against the unmodified sources in /root/reference to
// prove the ABI fits (oracle/_ref/libFM_b200; exercised by tests/test_cli_gpu.py).
//
// FMB200_MODE=inorder|ordered|hogwild (environment; default hogwild) picks the execution mode,
// FMB200_DEVICE the CUDA ordinal, FMB200_REPRODUCIBLE=1 the windowed HOGWILD epoch (fmb200_set_reproducible).
#ifndef FM_LEARN_SGD_B200_H_
#define FM_LEARN_SGD_B200_H_

#include <cstdlib>
#include <cstring>
#include <vector>
#include <ctime>

#include "fm_learn_sgd.h"

extern "C" {
#include "fmb200.h"
}

class fm_learn_sgd_b200 : public fm_learn_sgd {
 public:
  fm_learn_sgd_b200() : ctx(NULL), train_(NULL) {}
  virtual ~fm_learn_sgd_b200() {
    if (ctx) fmb200_destroy(ctx);
  }

  virtual void init() {
    fm_learn_sgd::init();
    if (log != NULL) log->addField("rmse_train", std::numeric_limits<double>::quiet_NaN());
    const char* dev = getenv("FMB200_DEVICE");
    ck(fmb200_create(&ctx, dev ? atoi(dev) : 0, fm->num_attribute, fm->num_factor, fm->k0, fm->k1));
    const char* mode = getenv("FMB200_MODE");
    ck(fmb200_set_mode(ctx, (mode && !strcmp(mode, "inorder")) ? FMB200_MODE_INORDER
                            : (mode && !strcmp(mode, "ordered")) ? FMB200_MODE_ORDERED
                                                                 : FMB200_MODE_HOGWILD));
    const char* repro = getenv("FMB200_REPRODUCIBLE");
    if (repro && !strcmp(repro, "1")) ck(fmb200_set_reproducible(ctx, 1, 0, 0));
  }

  // the row loop of fm_learn_sgd_element::learn (fm_learn_sgd_element.h:48-78), one
  // fmb200_sgd_epoch per iteration
  virtual void learn(Data& train, Data& test) {
    fm_learn_sgd::learn(train, test);
    std::cout << "SGD: DON'T FORGET TO SHUFFLE THE ROWS IN TRAINING DATA TO GET THE BEST RESULTS." << std::endl;
    ck(fmb200_set_hparams(ctx, task, learn_rate, fm->reg0, fm->regw, fm->regv, min_target, max_target));
    // DVector / DMatrix are one contiguous block each (util/matrix.h:165-170)
    ck(fmb200_set_params(ctx, fm->w0, fm->w.value, fm->num_factor ? fm->v.value[0] : NULL));
    train_ = &train;
    attach(train, 0);
    attach(test, 1);
    for (int i = 0; i < num_iter; i++) {
      double secs = 0;
      ck(fmb200_sgd_epoch(ctx, 0, &secs));
      double rmse_train = evaluate(train);
      double rmse_test = evaluate(test);
      std::cout << "#Iter=" << std::setw(3) << i << "\tTrain=" << rmse_train << "\tTest=" << rmse_test << std::endl;
      if (log != NULL) {
        log->log("rmse_train", rmse_train);
        log->log("time_learn", secs);
        log->newLine();
      }
    }
    // hand the state back: saveModel / the final evaluate / -out keep working unchanged
    ck(fmb200_get_params(ctx, &fm->w0, fm->w.value, fm->num_factor ? fm->v.value[0] : NULL));
  }

  // fm_learn_sgd::predict (fm_learn_sgd.h:76-90)
  virtual void predict(Data& data, DVector<double>& out) {
    assert(data.data->getNumRows() == out.dim);
    ck(fmb200_predict(ctx, slot_of(data), 1, out.value));
  }

 protected:
  // fm_learn::evaluate_regression / _classification (fm_learn.h:113-153)
  virtual double evaluate_regression(Data& data) {
    double sq = 0, ab = 0;
    uint64_t ok = 0;
    double t0 = wall_seconds();  // the pass runs on the GPU: user-CPU time would read ~0
    ck(fmb200_evaluate(ctx, slot_of(data), &sq, &ab, &ok));
    double n = data.data->getNumRows();
    if (log != NULL) {
      log->log("rmse", std::sqrt(sq / n));
      log->log("mae", ab / n);
      log->log("time_pred", wall_seconds() - t0);
    }
    return std::sqrt(sq / n);
  }
  virtual double evaluate_classification(Data& data) {
    double sq = 0, ab = 0;
    uint64_t ok = 0;
    double t0 = wall_seconds();
    ck(fmb200_evaluate(ctx, slot_of(data), &sq, &ab, &ok));
    double acc = (double)ok / (double)data.data->getNumRows();
    if (log != NULL) {
      log->log("accuracy", acc);
      log->log("time_pred", wall_seconds() - t0);
    }
    return acc;
  }

 private:
  fmb200_ctx* ctx;
  Data* train_;

  static void ck(int rc) {
    if (rc != 0) throw std::string(fmb200_last_error());
  }
  static double wall_seconds() {
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
  }
  int slot_of(Data& d) { return &d == train_ ? 0 : 1; }

  // Text input lives in LargeSparseMatrixMemory: hand its sparse_row[] to the library as
  // is (fmb200_upload_data_aos).  Binary input streams through the row cursor
  // (LargeSparseMatrixHD, util/fmatrix.h:68-101): assemble a CSR from it.
  void attach(Data& d, int slot) {
    LargeSparseMatrixMemory<DATA_FLOAT>* mem = dynamic_cast<LargeSparseMatrixMemory<DATA_FLOAT>*>(d.data);
    if (mem != NULL) {
      ck(fmb200_upload_data_aos(ctx, slot, mem->data.dim, mem->data.value, d.target.value));
      return;
    }
    std::vector<uint64_t> row_ptr(1, 0);
    std::vector<uint32_t> col;
    std::vector<float> val;
    for (d.data->begin(); !d.data->end(); d.data->next()) {
      sparse_row<DATA_FLOAT>& row = d.data->getRow();
      for (uint j = 0; j < row.size; j++) {
        col.push_back(row.data[j].id);
        val.push_back(row.data[j].value);
      }
      row_ptr.push_back(col.size());
    }
    col.push_back(0);  // keep .data() non-null for empty inputs
    val.push_back(0);
    ck(fmb200_upload_data(ctx, slot, row_ptr.size() - 1, row_ptr.back(), &row_ptr[0], &col[0], &val[0],
                          d.target.value));
  }
};

#endif /*FM_LEARN_SGD_B200_H_*/
