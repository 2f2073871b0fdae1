// libfm_main.cpp -- the drop-in `libFM` command line for the SGD path on H100.
//
// Keeps the reference's flags, defaults, stdout lines and file formats
// (reference src/libfm/libfm.cpp:62-441) and swaps the learner for one whose
// passes over the data run in libfmb200 (include/fmb200.h).  `-method sgd` runs in every mode;
// `-method mcmc|als` (one GPU, with -relation blocks on resident data) run with -mode inorder or ordered, the
// fp64 state, and so does `-method sgda` with its -validation set, which also runs in -mode hogwild as the
// windowed fp32 epoch (resident data, one GPU).
// -cache_size streams a binary data set larger than it through the GPU block by block (one GPU): -method sgd
// and sgda its .x (sgda its validation set too), -method mcmc|als its transposed .xt (as the reference's
// data_t); text input loads the data whole.
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
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "cli_flags.h"
#include "fm_host.h"

using namespace host;

// -mode and -gpus: SGD runs in every mode on one or more GPUs, MCMC and ALS in the fp64 modes on one
struct Exec {
  int mode, num_gpus;
};
static Exec exec_of(const CmdLine& cmd, const std::string& method) {
  const std::string name = cmd.str("mode", "hogwild");
  const int mode = name == "hogwild"   ? FMB200_MODE_HOGWILD
                   : name == "inorder" ? FMB200_MODE_INORDER
                   : name == "ordered" ? FMB200_MODE_ORDERED
                                       : -1;
  const int num_gpus = (int)cmd.integer("gpus", 1);
  if (method == "sgd") {
    if (mode < 0) throw std::string("unknown -mode " + name);
    if (num_gpus < 1) throw "-gpus must be >= 1";
  } else {
    // SGDA also runs in -mode hogwild, as the windowed fp32 epoch (fm_sgda_hogwild.cu)
    if (mode != FMB200_MODE_INORDER && mode != FMB200_MODE_ORDERED && !(method == "sgda" && mode == FMB200_MODE_HOGWILD))
      throw std::string("method '" + method + "' is outside the libfm_b200 scope in -mode " + name +
                        " (the fp32 SGD path); use -mode inorder");
    if (num_gpus != 1) throw std::string("-method " + method + " runs on one GPU: -gpus must be 1");
  }
  return {mode, num_gpus};
}

// libfm.cpp:141-434 for data sets without relations.  Learner is GpuSgdLearner for -method sgd, GpuSgdaLearner
// for sgda and GpuMcmcLearner for mcmc | als (libfm.cpp:135-139: ALS is MCMC without sampling and
// hyperparameter inference).
template <class Learner>
static int run(const CmdLine& cmd, const std::string& method, std::chrono::steady_clock::time_point t_start) {
  constexpr bool sgd = std::is_same<Learner, GpuSgdLearner>::value;
  constexpr bool sgda = std::is_same<Learner, GpuSgdaLearner>::value;
  constexpr bool mcmc = !sgd && !sgda;
  auto since_start = [&] {
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count();
  };

  // (1) data, libfm.cpp:141-157.  -cache_size (bytes; 0 or absent: everything resident, the reference's
  // unlimited), on one GPU: with -method sgd or sgda, a binary data set whose rows exceed one block of
  // cache_size / 2 bytes is read and trained on block by block (BinaryBlocks; SGDA's validation set too); with
  // -method mcmc | als, one whose transposed file <file>.xt exists and whose columns exceed such a block is
  // streamed from .xt and .y alone, .x unread (BinaryBlocks::open_xt; SGDA, MCMC and ALS run in -mode inorder |
  // ordered on one GPU, checked before loading).  Train, test and validation decide independently.  Text input
  // ignores the flag, as in the reference.
  const long long cache_size = cmd.integer("gpus", 1) == 1 ? cmd.integer64("cache_size", 0) : 0;
  auto load = [&](const std::string& file, SparseData& d) {
    std::unique_ptr<BinaryBlocks> b;
    if (cache_size > 0)
      b = mcmc ? BinaryBlocks::open_xt(file, (uint64_t)cache_size) : BinaryBlocks::open(file, (uint64_t)cache_size);
    if (b) b->print();
    else d.load(file);
    return b;
  };
  std::cout << "Loading train...\t" << std::endl;
  SparseData train;
  const std::unique_ptr<BinaryBlocks> train_blocks = load(cmd.str("train"), train);
  std::cout << "Loading test... \t" << std::endl;
  SparseData test;
  const std::unique_ptr<BinaryBlocks> test_blocks = load(cmd.str("test"), test);
  SparseData validation;  // libfm.cpp:159-173
  std::unique_ptr<BinaryBlocks> validation_blocks;
  if (cmd.has("validation") && !sgda)
    std::cout << "WARNING: Validation data is only used for SGDA. The data is ignored." << std::endl;
  if (sgda) {
    std::cout << "Loading validation set...\t" << std::endl;
    validation_blocks = load(cmd.str("validation"), validation);
  }
  // relation blocks (MCMC and ALS; the others have refused -relation), libfm.cpp:176-197: each block's .xt and
  // .groups, then its joins of the train and test cases
  const std::vector<std::string> rel_stems = cmd.list("relation");
  std::cout << "#relations: " << rel_stems.size() << std::endl;
  std::vector<GpuMcmcLearner::Relation> rel(rel_stems.size());
  for (size_t r = 0; r < rel.size(); r++) {
    rel[r].data.load(rel_stems[r]);
    rel[r].join[0].load(rel_stems[r] + ".train", train.num_cases());
    rel[r].join[1].load(rel_stems[r] + ".test", test.num_cases());
  }
  std::cout << "Loading meta data...\t" << std::endl;
  uint32_t n = (uint32_t)std::max(train_blocks ? train_blocks->num_feature : train.num_feature,
                                  test_blocks ? test_blocks->num_feature : test.num_feature);  // :203
  if (sgda)  // :204-206
    n = std::max(n, (uint32_t)(validation_blocks ? validation_blocks->num_feature : validation.num_feature));

  HostModel fm;
  Learner fml;
  fml.fm = &fm;
  if constexpr (!sgd) {
    // DataMetaInfo (Data.h:76-96), used by SGDA, MCMC and ALS (the reference also reads it for SGD, which ignores
    // it): -meta holds one group id per attribute, read with >>; a value the file lacks reads as 0 and is
    // counted in group 0
    fml.attr_group.assign(n, 0u);
    uint32_t G = 1;
    if (cmd.has("meta")) G = read_groups(cmd.str("meta"), n, fml.attr_group);
    if constexpr (sgda) {
      fml.n_groups = G;
    } else {
      // the joined meta table, libfm.cpp:212-241: the blocks' attributes follow the main table's, each block's
      // groups follow the groups before it
      for (GpuMcmcLearner::Relation& b : rel) {
        b.data.attr_offset = n;
        n += b.data.num_feature;
        for (uint32_t g : b.data.attr_group) fml.attr_group.push_back(G + g);
        G += b.data.num_groups;
      }
      fml.attr_per_group.assign(G, 0u);
      for (uint32_t i = 0; i < n; i++) fml.attr_per_group[fml.attr_group[i]]++;
      fml.relations = std::move(rel);
    }
  }

  // (2) model, libfm.cpp:244-283
  fm.num_attribute = n;
  fm.init_stdev = cmd.num("init_stdev", 0.1);
  {
    std::vector<int> dim = cmd.int_list("dim");
    if (dim.size() != 3) throw "-dim needs three values 'k0,k1,k2'";  // assert at :252
    fm.k0 = dim[0] != 0;
    fm.k1 = dim[1] != 0;
    fm.num_factor = dim[2];
  }
  fm.init();
  if (cmd.has("load_model")) {  // SGD and ALS: MCMC has refused it
    std::cout << "Reading FM model... \t" << std::endl;
    if (!fm.load(cmd.str("load_model"))) {
      std::cout << "WARNING: malformed model file. Nothing will be loaded." << std::endl;
      fm.init();
    }
  }
  if (mcmc)  // fm.w.init_normal (:283): overwrites a loaded w, as the reference does
    for (auto& x : fm.w) x = fm.draw();

  // (3) learner, libfm.cpp:270-309
  fml.num_iter = (int)cmd.integer("iter", 100);
  fml.max_target = train_blocks ? train_blocks->max_target : train.max_target;
  fml.min_target = train_blocks ? train_blocks->min_target : train.min_target;
  const std::string task = cmd.str("task");
  if (task == "r") {
    fml.task = FMB200_TASK_REGRESSION;
  } else if (task == "c") {
    fml.task = FMB200_TASK_CLASSIFICATION;
    train.binarize_targets();
    test.binarize_targets();
    validation.binarize_targets();  // :304-305
    if (train_blocks) train_blocks->binarize_targets();
    if (test_blocks) test_blocks->binarize_targets();
    if (validation_blocks) validation_blocks->binarize_targets();
  } else {
    throw "unknown task";
  }
  if constexpr (mcmc) fml.do_sample = fml.do_multilevel = method == "mcmc";
  const Exec exec = exec_of(cmd, method);  // SGDA, MCMC and ALS have passed it before loading
  fml.mode = exec.mode;
  fml.num_gpus = exec.num_gpus;
  fml.first_device = (int)cmd.integer("device", 0);

  // (4) logging, libfm.cpp:311-324
  std::ofstream rlog_file;
  std::unique_ptr<RLog> rlog;
  if (cmd.has("rlog")) {
    const std::string f = cmd.str("rlog");
    rlog_file.open(f.c_str());
    if (!rlog_file.is_open()) throw "Unable to open file " + f;
    std::cout << "logging to " << f << std::endl;
    rlog = std::make_unique<RLog>(&rlog_file);
  }
  fml.log = rlog.get();
  // A single-GPU run on a multi-GPU host: expose only that device to the CUDA driver
  // (initialising eight 180 GB devices costs seconds a short job never earns back).
  if (fml.num_gpus == 1 && getenv("CUDA_VISIBLE_DEVICES") == nullptr) {
    setenv("CUDA_VISIBLE_DEVICES", std::to_string(fml.first_device).c_str(), 1);
    fml.first_device = 0;
  }
  const double t_loaded = since_start();
  fml.init();
  const double t_init = since_start();

  // regularisation, libfm.cpp:326-384: r0,r1,r2 for every method; MCMC and ALS also take r0 and then
  // one r1 and one r2 per attribute group
  {
    const std::vector<double> reg = cmd.num_list("regular");
    const size_t s = reg.size();
    if constexpr (!mcmc) {
      if (!(s == 0 || s == 1 || s == 3)) throw "-regular needs 0, 1 or 3 values";  // assert at :370
    } else {
      if (!(s == 0 || s == 1 || s == 3 || s == 1 + 2 * fml.attr_per_group.size()))
        throw "-regular needs 0, 1, 3 or 1+2*#groups values";  // assert at :330
    }
    if (s == 1) fm.reg0 = fm.regw = fm.regv = reg[0];
    if (s == 3) {
      fm.reg0 = reg[0];
      fm.regw = reg[1];
      fm.regv = reg[2];
    }
    if constexpr (mcmc) {
      const uint32_t G = (uint32_t)fml.attr_per_group.size();
      const int k = fm.num_factor;
      fml.w_lambda.assign(G, fm.regw);
      fml.v_lambda.assign((size_t)G * k, fm.regv);
      if (s == 1 + 2 * (size_t)G && s > 3) {
        fm.reg0 = reg[0];
        for (uint32_t g = 0; g < G; g++) fml.w_lambda[g] = reg[1 + g];
        for (uint32_t g = 0; g < G; g++)
          for (int f = 0; f < k; f++) fml.v_lambda[(size_t)g * k + f] = reg[1 + G + g];
      }
    }
  }
  // learning rate, libfm.cpp:386-404.  Three values set the scalar rate to 0
  // (the per-layer rates are printed but never used by fm_SGD) -- kept as is.
  if constexpr (!mcmc) {
    std::vector<double> lr = cmd.num_list("learn_rate");
    if (!(lr.size() == 1 || lr.size() == 3)) throw "-learn_rate needs 1 or 3 values";  // assert at :392
    if (lr.size() == 1) {
      fml.learn_rate = lr[0];
      fml.learn_rates[0] = fml.learn_rates[1] = fml.learn_rates[2] = lr[0];
    } else {
      fml.learn_rate = 0;
      for (int i = 0; i < 3; i++) fml.learn_rates[i] = lr[i];
    }
  }
  const bool verbose = cmd.integer("verbosity", 0) > 0;
  if (rlog) rlog->init();
  if (verbose) {
    fm.debug();
    if constexpr (!mcmc) fml.debug();
  }

  // learn, libfm.cpp:414-420
  fml.attach(train, test, train_blocks.get(), test_blocks.get());
  if constexpr (sgda) fml.attach_validation(validation, validation_blocks.get());
  const double t_attached = since_start();
  if constexpr (!mcmc) {
    fml.learn();
    if (verbose)
      std::cout << "time: load " << t_loaded << " s, gpu init " << (t_init - t_loaded) << " s, upload "
                << (t_attached - t_init) << " s, learn+evaluate " << (since_start() - t_attached) << " s"
                << std::endl;
    std::cout << "Final\t" << "Train=" << fml.evaluate(0) << "\tTest=" << fml.evaluate(1) << std::endl;
  } else {
    fml.learn(test_blocks ? test_blocks->target : test.target);  // no Final line for MCMC / ALS (:417-420)
  }

  // -out, libfm.cpp:422-428 (DVector::save: one value per line, matrix.h:332-342)
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
  // -save_model, libfm.cpp:430-434
  if (cmd.has("save_model")) {
    std::cout << "Writing FM model to " << cmd.str("save_model") << std::endl;
    fml.pull_state();
    fm.save(cmd.str("save_model"));
  }
  return 0;
}

int main(int argc, char** argv) {
  const auto t_start = std::chrono::steady_clock::now();
  try {
    CmdLine cmd(argc, argv);
    const char* bar = "----------------------------------------------------------------------------";
    std::cout << bar << std::endl;
    std::cout << "libFM (libfm_b200: H100-native SGD path)" << std::endl;
    std::cout << "  CLI-compatible with libFM 1.4.4 for -method sgd; see INTEGRATION.md" << std::endl;
    std::cout << bar << std::endl;

    // the reference's 20 flags, libfm.cpp:76-102
    cmd.add("task", "r=regression, c=binary classification [MANDATORY]");
    cmd.add("meta", "filename for meta information about data set");
    cmd.add("train", "filename for training data [MANDATORY]");
    cmd.add("test", "filename for test data [MANDATORY]");
    cmd.add("validation", "filename for validation data (only for SGDA)");
    cmd.add("out", "filename for output");
    cmd.add("dim", "'k0,k1,k2': k0=use bias, k1=use 1-way interactions, k2=dim of 2-way interactions; default=1,1,8");
    cmd.add("regular", "'r0,r1,r2' for SGD and ALS: r0=bias regularization, r1=1-way regularization, r2=2-way regularization");
    cmd.add("init_stdev", "stdev for initialization of 2-way factors; default=0.1");
    cmd.add("iter", "number of iterations; default=100");
    cmd.add("learn_rate", "learn_rate for SGD; default=0.1");
    cmd.add("method", "learning method (SGD, SGDA, ALS, MCMC); default=MCMC");
    cmd.add("verbosity", "how much infos to print; default=0");
    cmd.add("rlog", "write measurements within iterations to a file; default=''");
    cmd.add("seed", "integer value, default=None");
    cmd.add("help", "this screen");
    cmd.add("relation", "BS: filenames for the relations, default=''");
    cmd.add("cache_size", "cache size for data storage (only applicable if data is in binary format), default=infty");
    cmd.add("save_model", "filename for writing the FM model");
    cmd.add("load_model", "filename for reading the FM model");
    // additions
    cmd.add("mode", "GPU execution mode: hogwild (throughput, default), ordered (the reference's update order, fp64, parallel over independent rows) or inorder (bit-exact fp64, one row at a time)");
    cmd.add("gpus", "number of GPUs to shard the training rows over; default=1");
    cmd.add("device", "first CUDA device ordinal; default=0");

    if (cmd.has("help") || argc == 1) {
      cmd.print_help();
      return 0;
    }
    cmd.check();

    // libfm.cpp:115-120
    long seed = cmd.integer("seed", (long)time(NULL));
    srand((unsigned)seed);
    if (!cmd.has("method")) cmd.set("method", "mcmc");
    if (!cmd.has("init_stdev")) cmd.set("init_stdev", "0.1");
    if (!cmd.has("dim")) cmd.set("dim", "1,1,8");

    const std::string method = cmd.str("method");
    // libfm.cpp:123-133: MCMC keeps no model file
    if (method == "mcmc" && cmd.has("save_model")) {
      std::cout << "WARNING: -save_model enabled only for SGD and ALS." << std::endl;
      return 0;
    }
    if (method == "mcmc" && cmd.has("load_model")) {
      std::cout << "WARNING: -load_model enabled only for SGD and ALS." << std::endl;
      return 0;
    }
    if (method == "sgda") {  // the fp64 modes, and -mode hogwild with a validation set (the windowed epoch)
      const std::string mode = cmd.str("mode", "hogwild");
      if (mode != "inorder" && mode != "ordered" && !(mode == "hogwild" && cmd.has("validation")))
        throw std::string("method '" + method + "' is outside the libfm_b200 scope (SGD hot path only); use -method sgd");
      if (!cmd.has("validation"))  // the reference asserts (libfm.cpp:277)
        throw "-method sgda needs a validation set (-validation) to learn the regularisation values on";
      if (mode == "hogwild" && cmd.integer64("cache_size", 0) > 0) {  // checked before loading
        std::string fx, fy;
        for (const char* f : {"train", "test", "validation"})
          if (SparseData::binary_pair(cmd.str(f), &fx, &fy))
            throw "-method sgda in -mode hogwild trains on resident data: -cache_size streams binary data in -mode "
                  "inorder or ordered; use -mode inorder";
      }
    }
    if (method != "sgd" && method != "sgda" && method != "mcmc" && method != "als")
      throw "unknown method";  // libfm.cpp:291-293
    // SGDA, MCMC and ALS refuse an out-of-scope -mode or -gpus before loading anything; SGD checks them after its model
    if (method != "sgd") exec_of(cmd, method);
    if (!cmd.list("relation").empty()) {  // MCMC and ALS: resident relation blocks, -mode inorder | ordered, one GPU
      if (method == "sgd") throw "relations are not supported with SGD";  // fm_learn_sgd.h:61-63
      if (method == "sgda") throw std::string("relations (-relation) are not supported with -method " + method);
      if (cmd.integer64("cache_size", 0) > 0)
        throw "relations (-relation) are not supported with -cache_size: the relation blocks and the data sets are "
              "held on the GPU whole; drop -cache_size";
      // a block is read from its transposed binary file <stem>.xt alone (RelationData); a stem without one is
      // refused as before, before the data sets are read.  The other files of a block are checked as they load,
      // each error naming its file.
      for (const std::string& stem : cmd.list("relation"))
        if (!SparseData::file_exists(stem + ".xt"))
          throw std::string("relations (-relation) are not supported with -method " + method);
    }
    if (method == "sgd") return run<GpuSgdLearner>(cmd, method, t_start);
    if (method == "sgda") return run<GpuSgdaLearner>(cmd, method, t_start);
    return run<GpuMcmcLearner>(cmd, method, t_start);
  } catch (std::string& e) {
    std::cerr << std::endl << "ERROR: " << e << std::endl;
  } catch (char const*& e) {
    std::cerr << std::endl << "ERROR: " << e << std::endl;
  } catch (const std::exception& e) {  // e.g. bad_alloc on a corrupt size field
    std::cerr << std::endl << "ERROR: " << e.what() << std::endl;
  }
  return 1;  // the reference falls off main with 0 here; a non-zero status is the one deliberate change
}
