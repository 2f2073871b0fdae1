// scripts/mcmc_relation_probe.cpp -- offline probe of the reference's MCMC / ALS learner on relational data,
// compiled by scripts/make_relation_golden.py against the UNMODIFIED reference headers (include path only;
// nothing of the reference is copied here).  The main tables are in-memory CSR (mcmc_ref_probe.cpp); the
// relation blocks are loaded from files with the reference's own RelationData::load and RelationJoin::load, and
// train.relation / test.relation and the joined meta table are set up as libfm.cpp:175-240 does.  Returns the
// state after the last iteration, the joined group table and the loader's lines.
#include "mcmc_ref_probe.cpp"

extern "C" int probe_mcmc_relation(int k, int k0, int k1, long seed, uint64_t n_tr, const uint64_t* tr_rp,
                                   const uint32_t* tr_col, const float* tr_val, const float* tr_y, int tr_nf,
                                   uint64_t n_te, const uint64_t* te_rp, const uint32_t* te_col, const float* te_val,
                                   const float* te_y, int te_nf, const char* stems, int n_rel, const char* meta_file,
                                   int task, int do_sample, int do_multilevel, const double* reg, int n_reg,
                                   int num_iter, double min_target, double max_target, uint32_t* n_out,
                                   uint32_t* G_out, uint32_t* group, uint32_t* per_group, int cap, double* init_state,
                                   double* state, double* hyper, int hyper_cap, uint32_t* counters, double* pred,
                                   char* out, int out_len) {
  std::ostringstream sink;
  std::streambuf* saved = std::cout.rdbuf(sink.rdbuf());
  int rc = 0;
  try {
    DataProbe* train = make_data(n_tr, tr_rp, tr_col, tr_val, tr_y, tr_nf);
    DataProbe* test = make_data(n_te, te_rp, te_col, te_val, te_y, te_nf);
    // libfm.cpp:175-198
    std::vector<std::string> rel;
    {
      std::istringstream in(stems);
      std::string s;
      while (std::getline(in, s))
        if (!s.empty()) rel.push_back(s);
    }
    if ((int)rel.size() != n_rel) throw "stems";
    DVector<RelationData*> relation;
    relation.setSize(rel.size());
    train->relation.setSize(rel.size());
    test->relation.setSize(rel.size());
    for (uint i = 0; i < rel.size(); i++) {
      relation(i) = new RelationData(0, false, true);  // -method mcmc: no .x, the .xt
      relation(i)->load(rel[i]);
      train->relation(i).data = relation(i);
      test->relation(i).data = relation(i);
      train->relation(i).load(rel[i] + ".train", train->num_cases);
      test->relation(i).load(rel[i] + ".test", test->num_cases);
    }
    // libfm.cpp:204-240
    uint num_all_attribute = std::max(train->num_feature, test->num_feature);
    DataMetaInfo meta_main(num_all_attribute);
    if (meta_file[0]) meta_main.loadGroupsFromFile(meta_file);
    for (uint r = 0; r < train->relation.dim; r++) {
      train->relation(r).data->attr_offset = num_all_attribute;
      num_all_attribute += train->relation(r).data->num_feature;
    }
    DataMetaInfo meta(num_all_attribute);
    meta.num_attr_groups = meta_main.num_attr_groups;
    for (uint r = 0; r < relation.dim; r++) meta.num_attr_groups += relation(r)->meta->num_attr_groups;
    meta.num_attr_per_group.setSize(meta.num_attr_groups);
    meta.num_attr_per_group.init(0);
    for (uint i = 0; i < meta_main.attr_group.dim; i++) {
      meta.attr_group(i) = meta_main.attr_group(i);
      meta.num_attr_per_group(meta.attr_group(i))++;
    }
    uint attr_cntr = meta_main.attr_group.dim;
    uint attr_group_cntr = meta_main.num_attr_groups;
    for (uint r = 0; r < relation.dim; r++) {
      for (uint i = 0; i < relation(r)->meta->attr_group.dim; i++) {
        meta.attr_group(i + attr_cntr) = attr_group_cntr + relation(r)->meta->attr_group(i);
        meta.num_attr_per_group(attr_group_cntr + relation(r)->meta->attr_group(i))++;
      }
      attr_cntr += relation(r)->meta->attr_group.dim;
      attr_group_cntr += relation(r)->meta->num_attr_groups;
    }
    meta.num_relations = train->relation.dim;
    const uint32_t n = num_all_attribute, G = meta.num_attr_groups;
    if ((int)n > cap || (int)G > cap || (int)(1 + 2 * G + 2 * G * k) > hyper_cap) throw "cap";
    *n_out = n;
    *G_out = G;
    for (uint32_t i = 0; i < n; i++) group[i] = meta.attr_group(i);
    for (uint32_t g = 0; g < G; g++) per_group[g] = meta.num_attr_per_group(g);
    // libfm.cpp:115-116, 245-283
    srand(seed);
    fm_model fm;
    fm.num_attribute = n;
    fm.init_stdev = 0.1;
    fm.k0 = k0 != 0;
    fm.k1 = k1 != 0;
    fm.num_factor = k;
    fm.init();
    fm.w.init_normal(fm.init_mean, fm.init_stdev);
    init_state[0] = fm.w0;
    memcpy(init_state + 1, fm.w.value, sizeof(double) * n);
    if (k > 0) memcpy(init_state + 1 + n, fm.v.value[0], sizeof(double) * (size_t)n * k);
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
    // -regular, libfm.cpp:326-364
    if (n_reg == 0) {
      fm.reg0 = 0.0;
      l.w_lambda.init(0.0);
      l.v_lambda.init(0.0);
    } else if (n_reg == 1) {
      fm.reg0 = reg[0];
      l.w_lambda.init(reg[0]);
      l.v_lambda.init(reg[0]);
    } else if (n_reg == 3) {
      fm.reg0 = reg[0];
      l.w_lambda.init(reg[1]);
      l.v_lambda.init(reg[2]);
    } else {
      if (n_reg != (int)(1 + 2 * G)) throw "reg";
      fm.reg0 = reg[0];
      for (uint32_t g = 0; g < G; g++) l.w_lambda(g) = reg[1 + g];
      for (uint32_t g = 0; g < G; g++)
        for (int f = 0; f < k; f++) l.v_lambda(g, f) = reg[1 + G + g];
    }
    l.learn(*train, *test);
    state[0] = fm.w0;
    memcpy(state + 1, fm.w.value, sizeof(double) * n);
    if (k > 0) memcpy(state + 1 + n, fm.v.value[0], sizeof(double) * (size_t)n * k);
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
