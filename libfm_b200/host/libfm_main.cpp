// libfm_main.cpp -- the drop-in `libFM` command line for the SGD path on H100.
//
// Keeps the reference's flags, defaults, stdout lines and file formats
// (reference src/libfm/libfm.cpp:62-441) and swaps the learner for one whose
// passes over the data run in libfmb200 (include/fmb200.h).  `-method sgd` runs in every mode;
// `-method mcmc|als` (data sets without relations, one GPU) run with -mode inorder or ordered, the
// fp64 state; sgda is refused with a clear error instead of silently doing something else.
//
// New, optional flags (old command lines are unaffected):
//   -mode hogwild|ordered|inorder   throughput (default); sequentially consistent fp64 (parallel over
//                           conflict-free runs, within rounding of the reference); bit-exact fp64
//   -gpus N                 row-shard the training set over N GPUs (hogwild)
//   -device D               first CUDA ordinal
#include <algorithm>
#include <cassert>
#include <chrono>
#include <cstdlib>
#include <ctime>
#include <fstream>
#include <iostream>
#include <string>
#include <vector>

#include "cli_flags.h"
#include "fm_host.h"

using namespace host;

// -method mcmc | als (libfm.cpp:135-139: ALS is MCMC without sampling and hyperparameter inference), following
// libfm.cpp:141-434 for data sets without relations
static int run_mcmc(const CmdLine& cmd, bool sample, int mode) {
  std::cout << "Loading train...\t" << std::endl;
  SparseData train;
  train.load(cmd.str("train"));
  std::cout << "Loading test... \t" << std::endl;
  SparseData test;
  test.load(cmd.str("test"));
  if (cmd.has("validation"))
    std::cout << "WARNING: Validation data is only used for SGDA. The data is ignored." << std::endl;
  std::cout << "#relations: " << 0 << std::endl;
  std::cout << "Loading meta data...\t" << std::endl;
  const uint32_t n = (uint32_t)std::max(train.num_feature, test.num_feature);  // :203
  // DataMetaInfo (Data.h:76-96): -meta holds one group id per attribute, read with >>; a value the file
  // lacks reads as 0 and is counted in group 0
  std::vector<uint32_t> group(n, 0u);
  uint32_t G = 1;
  if (cmd.has("meta")) {
    std::ifstream in(cmd.str("meta").c_str());
    if (!in.is_open()) throw "Unable to open file " + cmd.str("meta");
    G = 0;
    for (uint32_t i = 0; i < n; i++) {
      unsigned int v = 0;
      in >> v;
      group[i] = v;
      G = std::max(G, v + 1);
    }
  }
  std::vector<uint32_t> per_group(G, 0u);
  for (uint32_t i = 0; i < n; i++) per_group[group[i]]++;

  HostModel fm;  // :245-283
  fm.num_attribute = n;
  fm.init_stdev = cmd.num("init_stdev", 0.1);
  {
    std::vector<int> dim = cmd.int_list("dim");
    if (dim.size() != 3) throw "-dim needs three values 'k0,k1,k2'";
    fm.k0 = dim[0] != 0;
    fm.k1 = dim[1] != 0;
    fm.num_factor = dim[2];
  }
  fm.init();
  if (cmd.has("load_model")) {  // ALS only: MCMC returned above
    std::cout << "Reading FM model... \t" << std::endl;
    if (!fm.load(cmd.str("load_model"))) {
      std::cout << "WARNING: malformed model file. Nothing will be loaded." << std::endl;
      fm.init();
    }
  }
  for (uint32_t i = 0; i < n; i++)  // fm.w.init_normal: overwrites a loaded w, as the reference does
    fm.w[i] = (fm.init_stdev == 0.0 || std::isnan(fm.init_stdev)) ? fm.init_mean
                                                                   : fm.init_mean + fm.init_stdev * ran_gaussian();

  GpuMcmcLearner fml;
  fml.fm = &fm;
  fml.num_iter = (int)cmd.integer("iter", 100);
  fml.do_sample = fml.do_multilevel = sample;
  fml.mode = mode;
  fml.max_target = train.max_target;
  fml.min_target = train.min_target;
  const std::string task = cmd.str("task");
  if (task == "r") {
    fml.task = FMB200_TASK_REGRESSION;
  } else if (task == "c") {
    fml.task = FMB200_TASK_CLASSIFICATION;
    train.binarize_targets();
    test.binarize_targets();
  } else {
    throw "unknown task";
  }
  RLog* rlog = nullptr;
  std::ofstream* rlog_file = nullptr;
  if (cmd.has("rlog")) {
    const std::string f = cmd.str("rlog");
    rlog_file = new std::ofstream(f.c_str());
    if (!rlog_file->is_open()) throw "Unable to open file " + f;
    std::cout << "logging to " << f << std::endl;
    rlog = new RLog(rlog_file);
  }
  fml.log = rlog;
  fml.attr_group = group;
  fml.attr_per_group = per_group;
  const int k = fm.num_factor;
  if (getenv("CUDA_VISIBLE_DEVICES") == nullptr) {
    setenv("CUDA_VISIBLE_DEVICES", std::to_string(cmd.integer("device", 0)).c_str(), 1);
  } else {
    fml.device = (int)cmd.integer("device", 0);
  }
  fml.init();
  {  // regularisation per group, :326-364
    std::vector<double> reg = cmd.num_list("regular");
    if (!(reg.size() == 0 || reg.size() == 1 || reg.size() == 3 || reg.size() == 1 + 2 * (size_t)G))
      throw "-regular needs 0, 1, 3 or 1+2*#groups values";  // assert at :330
    fml.w_lambda.assign(G, 0.0);
    fml.v_lambda.assign((size_t)G * k, 0.0);
    if (reg.size() == 1 || reg.size() == 3) {
      fm.reg0 = reg[0];
      fm.regw = reg.size() == 1 ? reg[0] : reg[1];
      fm.regv = reg.size() == 1 ? reg[0] : reg[2];
      fml.w_lambda.assign(G, fm.regw);
      fml.v_lambda.assign((size_t)G * k, fm.regv);
    } else if (reg.size() == 1 + 2 * (size_t)G && reg.size() > 3) {
      fm.reg0 = reg[0];
      for (uint32_t g = 0; g < G; g++) fml.w_lambda[g] = reg[1 + g];
      for (uint32_t g = 0; g < G; g++)
        for (int f = 0; f < k; f++) fml.v_lambda[(size_t)g * k + f] = reg[1 + G + g];
    }
  }
  if (rlog) rlog->init();
  if (cmd.integer("verbosity", 0) > 0) fm.debug();
  fml.learn(train, test);
  // no Final line for MCMC / ALS (:417-420)
  if (cmd.has("out")) {
    std::vector<double> pred;
    fml.predict_test(pred);
    std::ofstream out(cmd.str("out").c_str());
    if (out.is_open()) {
      for (double p : pred) out << p << std::endl;
    } else {
      std::cout << "Unable to open file " << cmd.str("out");
    }
  }
  if (cmd.has("save_model")) {  // ALS only
    std::cout << "Writing FM model to " << cmd.str("save_model") << std::endl;
    fm.save(cmd.str("save_model"));
  }
  delete rlog;
  delete rlog_file;
  return 0;
}

int main(int argc, char** argv) {
  const auto t_start = std::chrono::steady_clock::now();
  auto since = [&](std::chrono::steady_clock::time_point t) {
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t).count();
  };
  try {
    CmdLine cmd(argc, argv);
    const char* bar = "----------------------------------------------------------------------------";
    std::cout << bar << std::endl;
    std::cout << "libFM (libfm_b200: H100-native SGD path)" << std::endl;
    std::cout << "  CLI-compatible with libFM 1.4.4 for -method sgd; see INTEGRATION.md" << std::endl;
    std::cout << bar << std::endl;

    // the reference's 20 flags, libfm.cpp:76-102
    const std::string p_task = cmd.add("task", "r=regression, c=binary classification [MANDATORY]");
    const std::string p_meta = cmd.add("meta", "filename for meta information about data set");
    const std::string p_train = cmd.add("train", "filename for training data [MANDATORY]");
    const std::string p_test = cmd.add("test", "filename for test data [MANDATORY]");
    const std::string p_val = cmd.add("validation", "filename for validation data (only for SGDA)");
    const std::string p_out = cmd.add("out", "filename for output");
    const std::string p_dim = cmd.add("dim", "'k0,k1,k2': k0=use bias, k1=use 1-way interactions, k2=dim of 2-way interactions; default=1,1,8");
    const std::string p_reg = cmd.add("regular", "'r0,r1,r2' for SGD and ALS: r0=bias regularization, r1=1-way regularization, r2=2-way regularization");
    const std::string p_stdev = cmd.add("init_stdev", "stdev for initialization of 2-way factors; default=0.1");
    const std::string p_iter = cmd.add("iter", "number of iterations; default=100");
    const std::string p_lr = cmd.add("learn_rate", "learn_rate for SGD; default=0.1");
    const std::string p_method = cmd.add("method", "learning method (SGD, SGDA, ALS, MCMC); default=MCMC");
    const std::string p_verb = cmd.add("verbosity", "how much infos to print; default=0");
    const std::string p_rlog = cmd.add("rlog", "write measurements within iterations to a file; default=''");
    const std::string p_seed = cmd.add("seed", "integer value, default=None");
    const std::string p_help = cmd.add("help", "this screen");
    const std::string p_rel = cmd.add("relation", "BS: filenames for the relations, default=''");
    const std::string p_cache = cmd.add("cache_size", "cache size for data storage (only applicable if data is in binary format), default=infty");
    const std::string p_save = cmd.add("save_model", "filename for writing the FM model");
    const std::string p_load = cmd.add("load_model", "filename for reading the FM model");
    // additions
    const std::string p_mode = cmd.add("mode", "GPU execution mode: hogwild (throughput, default), ordered (the reference's update order, fp64, parallel over independent rows) or inorder (bit-exact fp64, one row at a time)");
    const std::string p_gpus = cmd.add("gpus", "number of GPUs to shard the training rows over; default=1");
    const std::string p_dev = cmd.add("device", "first CUDA device ordinal; default=0");

    if (cmd.has(p_help) || argc == 1) {
      cmd.print_help();
      return 0;
    }
    cmd.check();

    // libfm.cpp:115-120
    long seed = cmd.integer(p_seed, (long)time(NULL));
    srand((unsigned)seed);
    if (!cmd.has(p_method)) cmd.set(p_method, "mcmc");
    if (!cmd.has(p_stdev)) cmd.set(p_stdev, "0.1");
    if (!cmd.has(p_dim)) cmd.set(p_dim, "1,1,8");

    const std::string method = cmd.str(p_method);
    // libfm.cpp:123-133: MCMC keeps no model file
    if (method == "mcmc" && cmd.has(p_save)) {
      std::cout << "WARNING: -save_model enabled only for SGD and ALS." << std::endl;
      return 0;
    }
    if (method == "mcmc" && cmd.has(p_load)) {
      std::cout << "WARNING: -load_model enabled only for SGD and ALS." << std::endl;
      return 0;
    }
    if (method == "mcmc" || method == "als") {
      const std::string mode = cmd.str(p_mode, "hogwild");
      if (mode != "inorder" && mode != "ordered")
        throw std::string("method '" + method + "' is outside the libfm_b200 scope in -mode " + mode +
                          " (the fp32 SGD path); use -mode inorder");
      if (cmd.integer(p_gpus, 1) != 1) throw std::string("-method " + method + " runs on one GPU: -gpus must be 1");
      if (!cmd.list(p_rel).empty()) throw std::string("relations (-relation) are not supported with -method " + method);
      return run_mcmc(cmd, method == "mcmc", mode == "inorder" ? FMB200_MODE_INORDER : FMB200_MODE_ORDERED);
    }
    if (method != "sgd") {
      if (method == "mcmc" || method == "als" || method == "sgda")
        throw std::string("method '" + method + "' is outside the libfm_b200 scope (SGD hot path only); use -method sgd");
      throw "unknown method";  // libfm.cpp:291-293
    }
    if (!cmd.list(p_rel).empty()) throw "relations are not supported with SGD";  // fm_learn_sgd.h:61-63

    // (1) data, libfm.cpp:141-157
    std::cout << "Loading train...\t" << std::endl;
    SparseData train;
    train.load(cmd.str(p_train));
    std::cout << "Loading test... \t" << std::endl;
    SparseData test;
    test.load(cmd.str(p_test));
    if (cmd.has(p_val))
      std::cout << "WARNING: Validation data is only used for SGDA. The data is ignored." << std::endl;
    std::cout << "#relations: " << 0 << std::endl;
    std::cout << "Loading meta data...\t" << std::endl;
    const uint32_t num_all_attribute = (uint32_t)std::max(train.num_feature, test.num_feature);  // :203

    // (2) model, libfm.cpp:244-268
    HostModel fm;
    fm.num_attribute = num_all_attribute;
    fm.init_stdev = cmd.num(p_stdev, 0.1);
    {
      std::vector<int> dim = cmd.int_list(p_dim);
      if (dim.size() != 3) throw "-dim needs three values 'k0,k1,k2'";  // assert at :252
      fm.k0 = dim[0] != 0;
      fm.k1 = dim[1] != 0;
      fm.num_factor = dim[2];
    }
    fm.init();
    if (cmd.has(p_load)) {
      std::cout << "Reading FM model... \t" << std::endl;
      if (!fm.load(cmd.str(p_load))) {
        std::cout << "WARNING: malformed model file. Nothing will be loaded." << std::endl;
        fm.init();
      }
    }

    // (3) learner, libfm.cpp:270-309
    GpuSgdLearner fml;
    fml.fm = &fm;
    fml.num_iter = (int)cmd.integer(p_iter, 100);
    fml.max_target = train.max_target;
    fml.min_target = train.min_target;
    const std::string task = cmd.str(p_task);
    if (task == "r") {
      fml.task = FMB200_TASK_REGRESSION;
    } else if (task == "c") {
      fml.task = FMB200_TASK_CLASSIFICATION;
      train.binarize_targets();
      test.binarize_targets();
    } else {
      throw "unknown task";
    }
    const std::string mode = cmd.str(p_mode, "hogwild");
    if (mode == "hogwild") fml.mode = FMB200_MODE_HOGWILD;
    else if (mode == "inorder") fml.mode = FMB200_MODE_INORDER;
    else if (mode == "ordered") fml.mode = FMB200_MODE_ORDERED;
    else throw std::string("unknown -mode " + mode);
    fml.num_gpus = (int)cmd.integer(p_gpus, 1);
    fml.first_device = (int)cmd.integer(p_dev, 0);
    if (fml.num_gpus < 1) throw "-gpus must be >= 1";

    // (4) logging, libfm.cpp:311-324
    RLog* rlog = nullptr;
    std::ofstream* rlog_file = nullptr;
    if (cmd.has(p_rlog)) {
      const std::string f = cmd.str(p_rlog);
      rlog_file = new std::ofstream(f.c_str());
      if (!rlog_file->is_open()) throw "Unable to open file " + f;
      std::cout << "logging to " << f << std::endl;
      rlog = new RLog(rlog_file);
    }
    fml.log = rlog;
    // A single-GPU run on a multi-GPU host: expose only that device to the CUDA driver
    // (initialising eight 180 GB devices costs seconds a short job never earns back).
    if (fml.num_gpus == 1 && getenv("CUDA_VISIBLE_DEVICES") == nullptr) {
      setenv("CUDA_VISIBLE_DEVICES", std::to_string(fml.first_device).c_str(), 1);
      fml.first_device = 0;
    }
    const double t_loaded = since(t_start);
    fml.init();
    const double t_init = since(t_start);

    // regularisation, libfm.cpp:366-384
    {
      std::vector<double> reg = cmd.num_list(p_reg);
      if (!(reg.size() == 0 || reg.size() == 1 || reg.size() == 3))
        throw "-regular needs 0, 1 or 3 values";  // assert at :370
      if (reg.size() == 1) fm.reg0 = fm.regw = fm.regv = reg[0];
      if (reg.size() == 3) {
        fm.reg0 = reg[0];
        fm.regw = reg[1];
        fm.regv = reg[2];
      }
    }
    // learning rate, libfm.cpp:386-404.  Three values set the scalar rate to 0
    // (the per-layer rates are printed but never used by fm_SGD) -- kept as is.
    {
      std::vector<double> lr = cmd.num_list(p_lr);
      if (!(lr.size() == 1 || lr.size() == 3)) throw "-learn_rate needs 1 or 3 values";  // assert at :392
      if (lr.size() == 1) {
        fml.learn_rate = lr[0];
        fml.learn_rates[0] = fml.learn_rates[1] = fml.learn_rates[2] = lr[0];
      } else {
        fml.learn_rate = 0;
        for (int i = 0; i < 3; i++) fml.learn_rates[i] = lr[i];
      }
    }
    if (rlog) rlog->init();
    if (cmd.integer(p_verb, 0) > 0) {
      fm.debug();
      fml.debug();
    }

    // learn, libfm.cpp:414-420
    fml.attach(train, test);
    const double t_attached = since(t_start);
    fml.push_state();
    fml.learn();
    if (cmd.integer(p_verb, 0) > 0)
      std::cout << "time: load " << t_loaded << " s, gpu init " << (t_init - t_loaded) << " s, upload "
                << (t_attached - t_init) << " s, learn+evaluate " << (since(t_start) - t_attached) << " s" << std::endl;
    std::cout << "Final\t" << "Train=" << fml.evaluate(0) << "\tTest=" << fml.evaluate(1) << std::endl;

    // -out, libfm.cpp:422-428 (DVector::save: one value per line, matrix.h:332-342)
    if (cmd.has(p_out)) {
      std::vector<double> pred;
      fml.predict_test(pred);
      std::ofstream out(cmd.str(p_out).c_str());
      if (out.is_open()) {
        for (double p : pred) out << p << std::endl;
      } else {
        std::cout << "Unable to open file " << cmd.str(p_out);
      }
    }
    // -save_model, libfm.cpp:430-434
    if (cmd.has(p_save)) {
      std::cout << "Writing FM model to " << cmd.str(p_save) << std::endl;
      fml.pull_state();
      fm.save(cmd.str(p_save));
    }
    delete rlog;
    delete rlog_file;
    return 0;
  } catch (std::string& e) {
    std::cerr << std::endl << "ERROR: " << e << std::endl;
  } catch (char const*& e) {
    std::cerr << std::endl << "ERROR: " << e << std::endl;
  } catch (const std::exception& e) {  // e.g. bad_alloc on a corrupt size field
    std::cerr << std::endl << "ERROR: " << e.what() << std::endl;
  }
  return 1;  // the reference falls off main with 0 here; a non-zero status is the one deliberate change
}
