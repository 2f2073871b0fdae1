// fm_host.h -- host-side model image, R-style log and the SGD and MCMC/ALS learners
// of the drop-in command line.  The learners keep the reference's surface
// (init / learn / evaluate / predict; reference src/libfm/src/fm_learn.h:31-60)
// but every pass over the data is ONE call into libfmb200 (include/fmb200.h).
#pragma once
#include <sys/resource.h>

#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iomanip>
#include <iostream>
#include <limits>
#include <map>
#include <string>
#include <vector>

#include "../csrc/ref_random.h"
#include "fmb200.h"
#include "sparse_data.h"

#ifdef FMB200_WITH_NCCL
#include <cuda_runtime_api.h>
#include <nccl.h>
#endif

namespace host {

// RNG: libc rand() exactly as the reference consumes it (seeded by srand() at libfm.cpp:115-116)
using ref_random::ran_gaussian;

// ---- model image ------------------------------------------------------------
// v is factor-major [num_factor][num_attribute] like the reference's
// DMatrixDouble (util/matrix.h:152-175) so that the init draw order and the
// model file layout coincide with it.
struct HostModel {
  uint32_t num_attribute = 0;
  int num_factor = 0;
  bool k0 = true, k1 = true;
  double reg0 = 0, regw = 0, regv = 0;
  double init_mean = 0, init_stdev = 0.01;
  double w0 = 0;
  std::vector<double> w, v;

  double& V(int f, uint32_t i) { return v[(size_t)f * num_attribute + i]; }

  // one draw of DVector/DMatrix::init_normal (matrix.h:398-404)
  double draw() const {
    return (init_stdev == 0.0 || std::isnan(init_stdev)) ? init_mean : init_mean + init_stdev * ran_gaussian();
  }

  // fm_model::init, fm_core/fm_model.h:91-99
  void init() {
    w0 = 0;
    w.assign(num_attribute, 0.0);
    v.resize((size_t)num_factor * num_attribute);
    for (auto& x : v) x = draw();
  }

  void debug() const {  // fm_model.h:80-89
    std::cout << "num_attributes=" << num_attribute << std::endl;
    std::cout << "use w0=" << k0 << std::endl;
    std::cout << "use w1=" << k1 << std::endl;
    std::cout << "dim v =" << num_factor << std::endl;
    std::cout << "reg_w0=" << reg0 << std::endl;
    std::cout << "reg_w=" << regw << std::endl;
    std::cout << "reg_v=" << regv << std::endl;
    std::cout << "init ~ N(" << init_mean << "," << init_stdev << ")" << std::endl;
  }

  // text checkpoint, byte-compatible with fm_model::saveModel (fm_model.h:132-154)
  void save(const std::string& path) {
    std::ofstream out(path.c_str());
    if (k0) out << "#global bias W0" << std::endl << w0 << std::endl;
    if (k1) {
      out << "#unary interactions Wj" << std::endl;
      for (uint32_t i = 0; i < num_attribute; i++) out << w[i] << std::endl;
    }
    out << "#pairwise interactions Vj,f" << std::endl;
    for (uint32_t i = 0; i < num_attribute; i++) {
      for (int f = 0; f < num_factor; f++) {
        out << V(f, i);
        if (f != num_factor - 1) out << ' ';
      }
      out << std::endl;
    }
  }

  // fm_model::loadModel (fm_model.h:160-190): 1 = ok, 0 = malformed / missing.
  // Deviation: the reference's splitString yields no token for a line without a
  // blank, so num_factor == 1 files always read as malformed there; here they load.
  int load(const std::string& path) {
    std::ifstream in(path.c_str());
    if (!in.is_open()) return 0;
    std::string line;
    if (k0) {
      if (!std::getline(in, line)) return 0;
      if (!std::getline(in, line)) return 0;
      w0 = atof(line.c_str());
    }
    if (k1) {
      if (!std::getline(in, line)) return 0;
      for (uint32_t i = 0; i < num_attribute; i++) {
        if (!std::getline(in, line)) return 0;
        w[i] = atof(line.c_str());
      }
    }
    if (!std::getline(in, line)) return 0;
    for (uint32_t i = 0; i < num_attribute; i++) {
      if (!std::getline(in, line)) return 0;
      std::vector<std::string> tok;
      size_t a = 0;
      for (;;) {
        size_t b = line.find(' ', a);
        tok.push_back(line.substr(a, b == std::string::npos ? std::string::npos : b - a));
        if (b == std::string::npos) break;
        a = b + 1;
      }
      if ((int)tok.size() != num_factor) return 0;
      for (int f = 0; f < num_factor; f++) V(f, i) = atof(tok[f].c_str());
    }
    return 1;
  }
};

// ---- R-style measurement log (reference src/util/rlog.h:56-103) -------------
class RLog {
 public:
  explicit RLog(std::ostream* out) : out_(out) {}
  void add_field(const std::string& name, double dflt) {
    for (const auto& h : header_)
      if (h == name) throw "the field " + name + " already exists";
    header_.push_back(name);
    default_[name] = dflt;
  }
  void init() {
    write_row(true);
    reset();
  }
  void log(const std::string& field, double d) { value_[field] = d; }
  void new_line() {
    write_row(false);
    reset();
  }

 private:
  void reset() {
    value_.clear();
    for (const auto& h : header_) value_[h] = default_[h];
  }
  void write_row(bool names) {
    if (!out_) return;
    for (size_t i = 0; i < header_.size(); i++) {
      if (names) *out_ << header_[i];
      else *out_ << value_[header_[i]];
      *out_ << (i + 1 < header_.size() ? "\t" : "\n");
    }
    out_->flush();
  }
  std::ostream* out_;
  std::vector<std::string> header_;
  std::map<std::string, double> default_, value_;
};

inline double user_seconds() {  // util.h:71-81
  struct rusage ru;
  getrusage(RUSAGE_SELF, &ru);
  return (double)ru.ru_utime.tv_sec + (double)ru.ru_utime.tv_usec / 1e6;
}

// ---- the learners -------------------------------------------------------------
// What both share -- fm_learn (fm_learn.h:31-153) over one libfmb200 context per GPU: the model, the task and its
// target range, the log, and the data and parameters on the devices.
class GpuLearner {
 public:
  HostModel* fm = nullptr;
  double min_target = 0, max_target = 0;
  int task = FMB200_TASK_REGRESSION;
  int num_iter = 100;
  int mode = FMB200_MODE_HOGWILD;
  int num_gpus = 1;
  int first_device = 0;
  RLog* log = nullptr;

  GpuLearner() = default;
  GpuLearner(const GpuLearner&) = delete;
  GpuLearner& operator=(const GpuLearner&) = delete;
  ~GpuLearner() {
    for (auto c : ctx_) fmb200_destroy(c);
  }

  static void ck(int rc) {
    if (rc != 0) throw std::string(fmb200_last_error());
  }

  // slot 0 = the GPU's train shard (contiguous rows), slot 1 = test (GPU 0 only), slot 4 = SGDA's validation set.
  // A data set given as blocks (one GPU; .x blocks for -method sgd and sgda, .xt blocks for mcmc | als) is not
  // uploaded here: every pass over it streams its blocks through its two slots kSlot[which] (pass() here, or the
  // library's SGDA epoch), or through which + 2 and which + 4 (the library's MCMC passes).
  void attach(const SparseData& train, const SparseData& test, const BinaryBlocks* train_blocks = nullptr,
              const BinaryBlocks* test_blocks = nullptr) {
    const BinaryBlocks* blocks[2] = {train_blocks, test_blocks};
    for (int i = 0; i < 2; i++)
      if (blocks[i]) {
        streamed_[i].data = blocks[i];
        streamed_[i].reader.reset(new BlockReader(*blocks[i], pinned_alloc, pinned_free));
      }
    n_train_ = train_blocks ? train_blocks->num_cases() : train.num_cases();
    n_test_ = test_blocks ? test_blocks->num_cases() : test.num_cases();
    if (!train_blocks) attach_train(train);
    if (!test_blocks)
      ck(fmb200_upload_data(ctx_[0], 1, test.num_cases(), test.num_values(), test.row_ptr.data(), test.col.data(),
                            test.val.data(), test.target.data()));
  }

  void pull_state() { ck(fmb200_get_params(ctx_[0], &fm->w0, fm->w.data(), fm->v.data())); }

 protected:
  void attach_train(const SparseData& train) {
    const uint64_t n = train.num_cases();
    for (int g = 0; g < num_gpus; g++) {
      const uint64_t lo = n * g / num_gpus, hi = n * (g + 1) / num_gpus;
      std::vector<uint64_t> rp(hi - lo + 1);
      const uint64_t base = train.row_ptr[lo];
      for (uint64_t r = lo; r <= hi; r++) rp[r - lo] = train.row_ptr[r] - base;
      ck(fmb200_upload_data(ctx_[g], 0, hi - lo, rp.back(), rp.data(), train.col.data() + base,
                            train.val.data() + base, train.target.data() + lo));
    }
  }

  // the reader's two block buffers: page-locked, so the block uploads are asynchronous copies
  static void* pinned_alloc(uint64_t bytes) {
    void* p = nullptr;
    ck(fmb200_host_alloc(&p, bytes));
    return p;
  }
  static void pinned_free(void* p) { fmb200_host_free(p); }

  // fm_learn::init (fm_learn.h:73-91): the log fields every method writes
  void add_log_fields() {
    if (!log) return;
    const double nan = std::numeric_limits<double>::quiet_NaN();
    if (task == FMB200_TASK_REGRESSION) {
      log->add_field("rmse", nan);
      log->add_field("mae", nan);
    } else {
      log->add_field("accuracy", nan);
    }
    for (const char* f : {"time_pred", "time_learn", "time_learn2", "time_learn4"}) log->add_field(f, nan);
  }

  void create_contexts() {
    ctx_.resize(num_gpus, nullptr);
    for (int g = 0; g < num_gpus; g++) {
      ck(fmb200_create(&ctx_[g], first_device + g, fm->num_attribute, fm->num_factor, fm->k0, fm->k1));
      ck(fmb200_set_mode(ctx_[g], mode));
    }
  }

  void push_state(double learn_rate) {
    for (auto c : ctx_) {
      ck(fmb200_set_hparams(c, task, learn_rate, fm->reg0, fm->regw, fm->regv, min_target, max_target));
      ck(fmb200_set_params(c, fm->w0, fm->w.data(), fm->v.data()));
    }
  }

  // a data set read block by block (train = 0, test = 1, validation = 2); data == nullptr: resident in its slot
  struct Streamed {
    const BinaryBlocks* data = nullptr;
    std::unique_ptr<BlockReader> reader;
    std::string error;  // what the reader met while the library fetched a block (fetch_block)
  };

  // The two slots of each data set's .x blocks (train, test, validation); the first is its slot when resident
  static constexpr int kSlot[3][2] = {{0, 2}, {1, 3}, {4, 6}};

  // One pass over the streamed data set `which` (0 train, 1 test, 2 validation) in file order: use(slot, block)
  // once per block, in order.  Block b goes to slot kSlot[which][b % 2] on the copy stream, so the copy of block b + 1
  // runs while the work use() enqueued on block b does; use() waits for its block's upload itself (every
  // call on a slot does).  Before block b + 1 overwrites block b - 1's slot, the work on b - 1 has run.
  template <class F>
  void pass(int which, F use) {
    fmb200_ctx* const c = ctx_[0];
    const std::vector<BinaryBlocks::Block>& blocks = streamed_[which].data->blocks;
    BlockReader& rd = *streamed_[which].reader;
    auto slot = [&](size_t b) { return kSlot[which][b % 2]; };
    auto upload = [&](size_t b) {
      const BlockReader::Buffer buf = rd.wait(b);
      ck(fmb200_upload_xblock_async(c, slot(b), blocks[b].rows(), blocks[b].nnz, buf.x, buf.row_size, buf.target));
    };
    ck(fmb200_sync(c));  // the slots may hold blocks the previous pass still works on
    rd.start();
    upload(0);
    for (size_t b = 0; b < blocks.size(); b++) {
      if (b + 1 < blocks.size()) {
        if (b > 0) ck(fmb200_sync(c));
        upload(b + 1);
      }
      use(slot(b), blocks[b]);
      rd.release(b);  // its upload has finished: use() waited for it
    }
    rd.stop();
  }

  // The library's view of a streamed .xt or .x (`which` as in pass()): its block plan, and its blocks fetched from
  // the reader (page-locked buffers) through slots slot0 and slot1.  col_lo / nnz are filled here and must outlive
  // the library's use (the MCMC state, or the SGDA epoch).
  fmb200_xt_blocks file_blocks(int which, int slot0, int slot1, std::vector<uint32_t>& col_lo,
                               std::vector<uint64_t>& nnz) {
    const BinaryBlocks& d = *streamed_[which].data;
    col_lo.clear();
    nnz.clear();
    for (const auto& b : d.blocks) {
      col_lo.push_back((uint32_t)b.row_lo);
      nnz.push_back(b.nnz);
    }
    col_lo.push_back((uint32_t)d.blocks.back().row_hi);
    fmb200_xt_blocks x{};
    x.n_cases = d.num_cases();
    x.target = d.target.data();
    x.n_blocks = d.blocks.size();
    x.col_lo = col_lo.data();
    x.nnz = nnz.data();
    x.slot[0] = slot0;
    x.slot[1] = slot1;
    x.user = &streamed_[which];
    x.fetch = fetch_block;
    x.release = release_block;
    return x;
  }
  static int fetch_block(void* user, uint64_t b, const void** words, const uint32_t** col_size) {
    Streamed& s = *static_cast<Streamed*>(user);
    try {
      if (b == 0) s.reader->start();  // every pass reads the file from its start
      const BlockReader::Buffer buf = s.reader->wait(b);
      *words = buf.x;
      *col_size = buf.row_size;
      return 0;
    } catch (const std::string& e) {
      s.error = e;
      return 1;
    }
  }
  static void release_block(void* user, uint64_t b) { static_cast<Streamed*>(user)->reader->release(b); }
  // ck() for calls that stream: the reader's own error, when it had one, says more than the library's
  void ck_streamed(int rc) {
    if (rc == 0) return;
    for (const auto& s : streamed_)
      if (!s.error.empty()) throw s.error;
    ck(rc);
  }

  // (its buffers are freed after ~GpuLearner has destroyed the contexts, which ends every copy from them)
  Streamed streamed_[3];
  std::vector<fmb200_ctx*> ctx_;
  uint64_t n_train_ = 0, n_test_ = 0, n_val_ = 0;
};

// fm_learn_sgd_element over N GPUs: rows shard contiguously, one replica of
// w0|w|V per GPU, one NCCL all-reduce + 1/N scale per epoch.
class GpuSgdLearner : public GpuLearner {
 public:
  double learn_rate = 0;
  double learn_rates[3] = {0, 0, 0};

#ifdef FMB200_WITH_NCCL
  ~GpuSgdLearner() {
    for (auto c : comms_) ncclCommDestroy(c);
  }
#endif

  // fm_learn::init + fm_learn_sgd_element::init (fm_learn.h:73-91, fm_learn_sgd_element.h:40-46)
  void init() {
    add_log_fields();
    if (log) log->add_field("rmse_train", std::numeric_limits<double>::quiet_NaN());
    if (num_gpus > 1 && mode != FMB200_MODE_HOGWILD)
      throw std::string("-gpus > 1 requires -mode hogwild (the ordered / in-order epoch is one dependency chain)");
    create_contexts();
    // FMB200_REPRODUCIBLE=1: HOGWILD epochs as windows of a constant number of rows, the same model on every run
    // (per block with -cache_size, per shard with -gpus)
    const char* repro = getenv("FMB200_REPRODUCIBLE");
    if (repro && !strcmp(repro, "1"))
      for (auto c : ctx_) ck(fmb200_set_reproducible(c, 1, 0, 0));
    // per-epoch exchange: NVLink peer-memory averaging when the devices can map each
    // other, NCCL otherwise (or when FMB200_CLI_NCCL is set)
    if (num_gpus > 1 && getenv("FMB200_CLI_NCCL") == nullptr) {
      use_peer_ = true;
      for (int g = 0; g < num_gpus && use_peer_; g++)
        if (fmb200_peer_attach_local(ctx_[g], num_gpus, g, ctx_.data()) != 0) use_peer_ = false;
      if (!use_peer_) std::cerr << "note: peer access unavailable (" << fmb200_last_error() << "), using NCCL" << std::endl;
    }
    if (use_peer_) return;
#ifdef FMB200_WITH_NCCL
    if (num_gpus > 1) {
      std::vector<int> devs(num_gpus);
      for (int g = 0; g < num_gpus; g++) devs[g] = first_device + g;
      comms_.resize(num_gpus);
      if (ncclCommInitAll(comms_.data(), num_gpus, devs.data()) != ncclSuccess)
        throw std::string("ncclCommInitAll failed");
    }
#else
    if (num_gpus > 1) throw std::string("this build has no NCCL: -gpus must be 1");
#endif
  }

  // the body of fm_learn_sgd_element::learn's epoch (fm_learn_sgd_element.h:56-67)
  double epoch() {
    const auto t0 = std::chrono::steady_clock::now();
    if (streamed_[0].data)
      pass(0, [&](int slot, const BinaryBlocks::Block&) { ck(fmb200_sgd_epoch_async(ctx_[0], slot)); });
    else
      for (auto c : ctx_) ck(fmb200_sgd_epoch_async(c, 0));
    if (use_peer_)
      for (auto c : ctx_) ck(fmb200_allreduce_mean(c));
#ifdef FMB200_WITH_NCCL
    if (num_gpus > 1 && !use_peer_) {
      ncclGroupStart();
      for (int g = 0; g < num_gpus; g++) {
        void *buf = nullptr, *st = nullptr;
        uint64_t cnt = 0;
        ck(fmb200_params_device(ctx_[g], &buf, &cnt));
        ck(fmb200_stream(ctx_[g], &st));
        ncclAllReduce(buf, buf, cnt, ncclFloat, ncclSum, comms_[g], (cudaStream_t)st);
      }
      ncclGroupEnd();
      for (auto c : ctx_) ck(fmb200_scale_params(c, 1.0 / num_gpus));
    }
#endif
    for (auto c : ctx_) ck(fmb200_sync(c));
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  }

  // fm_learn::evaluate (fm_learn.h:93-153); which = 0 train (all shards), 1 test, 2 SGDA's validation set
  double evaluate(int which) {
    // wall clock: the pass runs on the GPU, user-CPU time (the reference's clock) would read ~0
    const auto t0 = std::chrono::steady_clock::now();
    double sq = 0, ab = 0;
    uint64_t ok = 0;
    auto add = [&](fmb200_ctx* ctx, int slot) {
      double a = 0, b = 0;
      uint64_t c = 0;
      ck(fmb200_evaluate(ctx, slot, &a, &b, &c));
      sq += a;
      ab += b;
      ok += c;
    };
    if (streamed_[which].data) {
      // The fp64 modes add the regression errors in row order (fm_learn.h:136-146): across the blocks too,
      // so the host adds them from the clamped predictions, err = p - y exactly as fmb200_evaluate forms it.
      const BinaryBlocks& d = *streamed_[which].data;
      const bool in_order = mode != FMB200_MODE_HOGWILD && task == FMB200_TASK_REGRESSION;
      std::vector<double> pred;
      pass(which, [&](int slot, const BinaryBlocks::Block& b) {
        if (!in_order) return add(ctx_[0], slot);
        pred.resize(b.rows());
        ck(fmb200_predict(ctx_[0], slot, 1, pred.data()));
        for (uint64_t i = 0; i < b.rows(); i++) {
          const double err = pred[i] - (double)d.target[b.row_lo + i];
          sq += err * err;
          ab += std::abs(err);
        }
      });
    } else {
      for (int g = 0; g < (which == 0 ? num_gpus : 1); g++) add(ctx_[g], kSlot[which][0]);
    }
    const double n = (double)(which == 0 ? n_train_ : which == 1 ? n_test_ : n_val_);
    const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    if (task == FMB200_TASK_REGRESSION) {
      const double rmse = std::sqrt(sq / n);
      if (log) {
        log->log("rmse", rmse);
        log->log("mae", ab / n);
        log->log("time_pred", dt);
      }
      return rmse;
    }
    const double acc = (double)ok / n;
    if (log) {
      log->log("accuracy", acc);
      log->log("time_pred", dt);
    }
    return acc;
  }

  // fm_learn_sgd::learn + fm_learn_sgd_element::learn (fm_learn_sgd.h:55-65, ..._element.h:48-78)
  void learn() {
    push_state(learn_rate);
    std::cout << "learnrate=" << learn_rate << std::endl;
    std::cout << "learnrates=" << learn_rates[0] << "," << learn_rates[1] << "," << learn_rates[2] << std::endl;
    std::cout << "#iterations=" << num_iter << std::endl;
    std::cout.flush();
    std::cout << "SGD: DON'T FORGET TO SHUFFLE THE ROWS IN TRAINING DATA TO GET THE BEST RESULTS." << std::endl;
    for (int i = 0; i < num_iter; i++) {
      const double dt = epoch();
      const double tr = evaluate(0);
      const double te = evaluate(1);
      std::cout << "#Iter=" << std::setw(3) << i << "\tTrain=" << tr << "\tTest=" << te << std::endl;
      if (log) {
        log->log("rmse_train", tr);
        log->log("time_learn", dt);
        log->new_line();
      }
    }
  }

  // fm_learn_sgd::predict (fm_learn_sgd.h:76-90) on the test slot
  void predict_test(std::vector<double>& out) {
    out.resize(n_test_);
    if (streamed_[1].data)
      pass(1, [&](int slot, const BinaryBlocks::Block& b) { ck(fmb200_predict(ctx_[0], slot, 1, out.data() + b.row_lo)); });
    else
      ck(fmb200_predict(ctx_[0], 1, 1, out.data()));
  }

  void debug() const {  // fm_learn_sgd.h:71-74 + fm_learn.h:107-111
    std::cout << "num_iter=" << num_iter << std::endl;
    std::cout << "task=" << task << std::endl;
    std::cout << "min_target=" << min_target << std::endl;
    std::cout << "max_target=" << max_target << std::endl;
  }

 private:
#ifdef FMB200_WITH_NCCL
  std::vector<ncclComm_t> comms_;
#endif
  bool use_peer_ = false;
};

// fm_learn_sgd_element_adapt_reg (SGDA, one GPU, fp64 modes): every epoch is one fmb200_sgda_epoch_x over the
// training set (slot 0, or its .x blocks) with the validation set (slot 4, or its .x blocks); this class prints and
// logs what the reference's learn does (fm_learn_sgd_element_adapt_reg.h:276-355).  Evaluation, -out and the Final
// line are the SGD learner's, streamed passes included.
class GpuSgdaLearner : public GpuSgdLearner {
 public:
  std::vector<uint32_t> attr_group;  // DataMetaInfo::attr_group
  uint32_t n_groups = 1;

  // fm_learn_sgd::init + fm_learn_sgd_element_adapt_reg::init (:80-134): fm_learn's fields, then these
  void init() {
    GpuSgdLearner::init();  // fm_learn's fields and rmse_train
    if (!log) return;
    const double nan = std::numeric_limits<double>::quiet_NaN();
    log->add_field("rmse_val", nan);
    log->add_field("wmean", nan);
    log->add_field("wvar", nan);
    for (int f = 0; f < fm->num_factor; f++) {
      log->add_field("vmean" + std::to_string(f), nan);
      log->add_field("vvar" + std::to_string(f), nan);
    }
    for (uint32_t g = 0; g < n_groups; g++) {
      log->add_field("regw[" + std::to_string(g) + "]", nan);
      for (int f = 0; f < fm->num_factor; f++)
        log->add_field("regv[" + std::to_string(g) + "," + std::to_string(f) + "]", nan);
    }
  }

  void attach_validation(const SparseData& val, const BinaryBlocks* blocks = nullptr) {
    if (blocks) {
      n_val_ = blocks->num_cases();
      streamed_[2].data = blocks;
      streamed_[2].reader.reset(new BlockReader(*blocks, pinned_alloc, pinned_free));
      return;
    }
    n_val_ = val.num_cases();
    ck(fmb200_upload_data(ctx_[0], kSlot[2][0], val.num_cases(), val.num_values(), val.row_ptr.data(),
                          val.col.data(), val.val.data(), val.target.data()));
  }

  void learn() {
    push_state(learn_rate);
    std::cout << "learnrate=" << learn_rate << std::endl;
    std::cout << "learnrates=" << learn_rates[0] << "," << learn_rates[1] << "," << learn_rates[2] << std::endl;
    std::cout << "#iterations=" << num_iter << std::endl;
    std::cout.flush();
    std::cout << "Training using self-adaptive-regularization SGD." << std::endl
              << "DON'T FORGET TO SHUFFLE THE ROWS IN TRAINING AND VALIDATION DATA TO GET THE BEST RESULTS."
              << std::endl;
    // :282-289: w = 0, the model's regularisation off, reg_w = reg_v = 0 (fmb200_sgda_begin zeroes w and reg)
    std::fill(fm->w.begin(), fm->w.end(), 0.0);
    fm->reg0 = fm->regw = fm->regv = 0;
    ck(fmb200_set_hparams(ctx_[0], task, learn_rate, 0.0, 0.0, 0.0, min_target, max_target));
    ck(fmb200_sgda_begin(ctx_[0], n_groups, n_groups > 1 ? attr_group.data() : nullptr));
    std::cout << "Using " << n_train_ << " rows for training model parameters and " << n_val_
              << " for training shrinkage." << std::endl;
    const int k = fm->num_factor;
    std::vector<double> var_v(k), reg_w(n_groups), reg_v((size_t)n_groups * k);
    fmb200_xt_blocks x[2];  // the training and validation sets' .x blocks, when streamed
    std::vector<uint32_t> row_lo[2];
    std::vector<uint64_t> nnz[2];
    const fmb200_xt_blocks* xp[2] = {nullptr, nullptr};
    for (int i = 0; i < 2; i++) {
      const int which = 2 * i;
      if (streamed_[which].data) {
        x[i] = file_blocks(which, kSlot[which][0], kSlot[which][1], row_lo[i], nnz[i]);
        xp[i] = &x[i];
      }
    }
    for (int i = 0; i < num_iter; i++) {
      const auto t0 = std::chrono::steady_clock::now();
      // no lambda-steps in the first epoch (:303)
      ck_streamed(fmb200_sgda_epoch_x(ctx_[0], kSlot[0][0], xp[0], kSlot[2][0], xp[1], i > 0, nullptr));
      const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      const double rmse_val = evaluate(2);
      const double rmse_train = evaluate(0);
      const double rmse_test = evaluate(1);
      std::cout << "#Iter=" << std::setw(3) << i << "\tTrain=" << rmse_train << "\tTest=" << rmse_test << std::endl;
      if (!log) continue;
      double var_w = 0;
      ck(fmb200_sgda_get_moments(ctx_[0], &var_w, var_v.data()));
      ck(fmb200_sgda_get_reg(ctx_[0], reg_w.data(), reg_v.data()));
      log->log("wmean", 0.0);  // update_means zeroes the means it logs (:270-273)
      log->log("wvar", var_w);
      for (int f = 0; f < k; f++) {
        log->log("vmean" + std::to_string(f), 0.0);
        log->log("vvar" + std::to_string(f), var_v[f]);
      }
      for (uint32_t g = 0; g < n_groups; g++) {
        log->log("regw[" + std::to_string(g) + "]", reg_w[g]);
        for (int f = 0; f < k; f++)
          log->log("regv[" + std::to_string(g) + "," + std::to_string(f) + "]", reg_v[(size_t)g * k + f]);
      }
      log->log("time_learn", dt);
      log->log("rmse_train", rmse_train);
      log->log("rmse_val", rmse_val);
      log->new_line();
    }
  }
};

// fm_learn_mcmc_simultaneous (MCMC / ALS, one GPU, relation blocks on resident data): every iteration is one
// fmb200_mcmc_iteration; this class prints and logs what the reference's _learn does
// (fm_learn_mcmc_simultaneous.h:88-270) and writes -out like fm_learn_mcmc::predict.
class GpuMcmcLearner : public GpuLearner {
 public:
  // a relation block and its joins of the train (0) and test (1) cases (libfm.cpp:176-197)
  struct Relation {
    RelationData data;
    RelationJoin join[2];
  };
  bool do_sample = true, do_multilevel = true;
  std::vector<uint32_t> attr_group;  // DataMetaInfo (Data.h:33-96), joined over the relation blocks
  std::vector<uint32_t> attr_per_group;
  std::vector<double> w_lambda, v_lambda;  // [G], [G][k]: what -regular sets (libfm.cpp:326-364)
  std::vector<Relation> relations;         // resident data only

  // fm_learn::init + fm_learn_mcmc::init (fm_learn.h:73-91, fm_learn_mcmc.h:1099-1158): the rlog fields
  void init() {
    const uint32_t G = (uint32_t)attr_per_group.size();
    add_log_fields();
    if (log) {
      const double nan = std::numeric_limits<double>::quiet_NaN();
      log->add_field("alpha", nan);
      const char* const* names = task == FMB200_TASK_REGRESSION ? reg_fields_ : cls_fields_;
      for (int i = 0; i < (task == FMB200_TASK_REGRESSION ? 3 : 6); i++) log->add_field(names[i], nan);
      for (uint32_t g = 0; g < G; g++) {
        log->add_field("wmu[" + std::to_string(g) + "]", nan);
        log->add_field("wlambda[" + std::to_string(g) + "]", nan);
        for (int f = 0; f < fm->num_factor; f++) {
          log->add_field("vmu[" + std::to_string(g) + "," + std::to_string(f) + "]", nan);
          log->add_field("vlambda[" + std::to_string(g) + "," + std::to_string(f) + "]", nan);
        }
      }
    }
    create_contexts();
  }

  // after attach(): test is the set in slot 1, its targets score the predictions
  // test_target: the targets of the test set (resident or streamed)
  void learn(const std::vector<float>& test) {
    push_state(0.0);
    fmb200_ctx* const ctx = ctx_[0];
    const uint32_t G = (uint32_t)attr_per_group.size();
    const int k = fm->num_factor;
    if (streamed_[0].data || streamed_[1].data) {  // a set larger than -cache_size streams from its .xt
      fmb200_xt_blocks xt[2];
      for (int i = 0; i < 2; i++)
        if (streamed_[i].data) xt[i] = file_blocks(i, i + 2, i + 4, xt_col_lo_[i], xt_nnz_[i]);
      ck_streamed(fmb200_mcmc_begin_xt(ctx, 0, streamed_[0].data ? &xt[0] : nullptr, 1,
                                       streamed_[1].data ? &xt[1] : nullptr, do_sample, do_multilevel, G,
                                       attr_group.data(), attr_per_group.data(), fm->reg0, w_lambda.data(),
                                       v_lambda.data()));
    } else {
      if (!relations.empty()) {  // the relations apply to the _begin that follows
        std::vector<fmb200_relation> rel;
        for (const Relation& r : relations) {
          const RelationData& d = r.data;
          rel.push_back(fmb200_relation{d.num_cases, d.num_feature, d.attr_offset, d.col_ptr.data(), d.row.data(),
                                        d.val.data(), r.join[0].rows.size(), r.join[1].rows.size(),
                                        r.join[0].rows.data(), r.join[1].rows.data()});
        }
        ck(fmb200_mcmc_set_relations(ctx, 0, 1, (uint32_t)rel.size(), rel.data()));
      }
      ck(fmb200_mcmc_begin(ctx, 0, 1, do_sample, do_multilevel, G, attr_group.data(), attr_per_group.data(),
                           fm->reg0, w_lambda.data(), v_lambda.data()));
    }
    const uint64_t nt = test.size();
    pred_this_.assign(nt, 0.0);
    pred_all_.assign(nt, 0.0);
    std::vector<double> but5(nt), w_mu(G), wl(G), v_mu((size_t)G * k), vl((size_t)G * k);
    static const char* cnt_names[8] = {"alpha", "w0", "w", "v", "w_mu", "w_lambda", "v_mu", "v_lambda"};
    for (uint32_t i = 0; i < (uint32_t)num_iter; i++) {
      const double t0 = user_seconds();
      const clock_t c0 = clock();
      const auto w0 = std::chrono::steady_clock::now();
      double train_metric = 0;
      uint32_t cnt[16];
      ck_streamed(fmb200_mcmc_iteration(ctx, &train_metric, cnt));
      for (int p = 0; p < 8; p++)  // fm_learn_mcmc_simultaneous.h:96-119
        if (cnt[2 * p] > 0 || cnt[2 * p + 1] > 0)
          std::cout << "#nans in " << cnt_names[p] << ":\t" << cnt[2 * p] << "\t#inf_in_" << cnt_names[p] << ":\t"
                    << cnt[2 * p + 1] << std::endl;
      double alpha = 0;
      ck(fmb200_mcmc_get_hyper(ctx, &alpha, w_mu.data(), wl.data(), v_mu.data(), vl.data()));
      ck(fmb200_mcmc_get_pred(ctx, pred_this_.data(), pred_all_.data(), but5.data()));
      if (log) {
        log->log("alpha", alpha);
        for (uint32_t g = 0; g < G; g++) {
          log->log("wmu[" + std::to_string(g) + "]", w_mu[g]);
          log->log("wlambda[" + std::to_string(g) + "]", wl[g]);
          for (int f = 0; f < k; f++) {
            log->log("vmu[" + std::to_string(g) + "," + std::to_string(f) + "]", v_mu[(size_t)g * k + f]);
            log->log("vlambda[" + std::to_string(g) + "," + std::to_string(f) + "]", vl[(size_t)g * k + f]);
          }
        }
        // the reference's clocks are user-CPU time; the iteration runs on the GPU, so wall time goes in too
        log->log("time_learn", user_seconds() - t0);
        log->log("time_learn2", (double)(clock() - c0) / CLOCKS_PER_SEC);
        log->log("time_learn4", std::chrono::duration<double>(std::chrono::steady_clock::now() - w0).count());
      }
      // the normalisers keep the reference's unsigned arithmetic: 1/(i-5+1) wraps for i < 4
      const double n_all = 1.0 / (i + 1), n_but5 = 1.0 / (uint32_t)(i - 5 + 1);
      if (task == FMB200_TASK_REGRESSION) {
        double r[3], m[3];
        eval_reg(pred_this_, test, 1.0, &r[0], &m[0]);
        eval_reg(pred_all_, test, n_all, &r[1], &m[1]);
        eval_reg(but5, test, n_but5, &r[2], &m[2]);
        std::cout << "#Iter=" << std::setw(3) << i << "\tTrain=" << train_metric << "\tTest=" << r[1] << std::endl;
        if (log) {
          log->log("rmse", r[1]);
          log->log("mae", m[1]);
          for (int q = 0; q < 3; q++) log->log(reg_fields_[q], r[q]);
          log->new_line();
        }
      } else {
        double a[3], ll[3];
        eval_cls(pred_this_, test, 1.0, &a[0], &ll[0]);
        eval_cls(pred_all_, test, n_all, &a[1], &ll[1]);
        eval_cls(but5, test, n_but5, &a[2], &ll[2]);
        std::cout << "#Iter=" << std::setw(3) << i << "\tTrain=" << train_metric << "\tTest=" << a[1]
                  << "\tTest(ll)=" << ll[1] << std::endl;
        if (log) {
          log->log("accuracy", a[1]);
          for (int q = 0; q < 3; q++) {
            log->log(cls_fields_[q], a[q]);
            log->log(cls_fields_[3 + q], ll[q]);
          }
          log->new_line();
        }
      }
    }
  }

  // fm_learn_mcmc::predict (fm_learn_mcmc.h:380-404)
  void predict_test(std::vector<double>& out) const {
    out.resize(pred_this_.size());
    for (size_t c = 0; c < out.size(); c++) {
      double p = do_sample ? pred_all_[c] / num_iter : pred_this_[c];
      if (task == FMB200_TASK_REGRESSION) {
        p = std::min(max_target, p);
        p = std::max(min_target, p);
      } else {
        p = std::min(1.0, p);
        p = std::max(0.0, p);
      }
      out[c] = p;
    }
  }

 private:
  // fm_learn_mcmc_simultaneous::_evaluate / _evaluate_class (:272-309) over all test cases
  void eval_reg(const std::vector<double>& pred, const std::vector<float>& t, double norm, double* rmse, double* mae) const {
    double r = 0, m = 0;
    uint32_t n = 0;
    for (size_t c = 0; c < pred.size(); c++) {
      double p = pred[c] * norm;
      p = std::min(max_target, p);
      p = std::max(min_target, p);
      const double err = p - t[c];
      r += err * err;
      m += std::abs((double)err);
      n++;
    }
    *rmse = std::sqrt(r / n);
    *mae = m / n;
  }
  void eval_cls(const std::vector<double>& pred, const std::vector<float>& t, double norm, double* acc, double* ll) const {
    double l = 0.0;
    uint32_t a = 0, n = 0;
    for (size_t c = 0; c < pred.size(); c++) {
      const double p = pred[c] * norm;
      if (((p >= 0.5) && (t[c] > 0.0)) || ((p < 0.5) && (t[c] < 0.0))) a++;
      const double m = (t[c] + 1.0) * 0.5;
      double pll = p;
      if (pll > 0.99) pll = 0.99;
      if (pll < 0.01) pll = 0.01;
      l -= m * log10(pll) + (1 - m) * log10(1 - pll);
      n++;
    }
    *ll = l / n;
    *acc = (double)a / n;
  }

  static constexpr const char* reg_fields_[3] = {"rmse_mcmc_this", "rmse_mcmc_all", "rmse_mcmc_all_but5"};
  static constexpr const char* cls_fields_[6] = {"acc_mcmc_this", "acc_mcmc_all", "acc_mcmc_all_but5",
                                                 "ll_mcmc_this",  "ll_mcmc_all",  "ll_mcmc_all_but5"};
  std::vector<double> pred_this_, pred_all_;
  std::vector<uint32_t> xt_col_lo_[2];
  std::vector<uint64_t> xt_nnz_[2];
};

}  // namespace host
