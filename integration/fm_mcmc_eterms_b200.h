// fm_mcmc_eterms_b200.h -- reference-side binding of fmb200_mcmc_eterms (include/fmb200.h).
//
// The MCMC / ALS learner re-predicts train and test once per iteration through
// fm_learn_mcmc::predict_data_and_write_to_eterms (fm_learn_mcmc.h:148-378; called at
// fm_learn_mcmc_simultaneous.h:69 and :122).  That member is not virtual, so a maintainer swaps
// the two call sites:
//
//   -  predict_data_and_write_to_eterms(main_data, main_cache);
//   +  b200_predict_data_and_write_to_eterms(fm, main_data, main_cache);
//
// (integration/build_patched.sh does exactly that on a temporary copy of the header and builds
// oracle/_ref/libFM_b200; with FMB200_MCMC_ETERMS=1 in the environment `-method mcmc|als` then
// runs its e-term pass on the GPU and prints the same per-iteration lines as the stock binary,
// tests/test_cli_gpu.py).  The Gibbs draws stay the reference's own code; the model crosses PCIe
// once per iteration (fmb200_set_params), the e-terms come back as one array per data set.
// Limits: data sets without relations, held in memory in row-major form (text input).
#ifndef FM_MCMC_ETERMS_B200_H_
#define FM_MCMC_ETERMS_B200_H_

#include <cstdlib>
#include <string>
#include <vector>

extern "C" {
#include "fmb200.h"
}

inline bool b200_eterms_enabled() {
  const char* e = getenv("FMB200_MCMC_ETERMS");
  return e != NULL && e[0] == '1';
}

inline void b200_predict_data_and_write_to_eterms(fm_model* fm, DVector<Data*>& main_data,
                                                  DVector<e_q_term*>& main_cache) {
  static fmb200_ctx* ctx = NULL;
  static std::vector<Data*> slots;  // slot i holds *slots[i]
  struct ck {
    static void rc(int r) {
      if (r != 0) throw std::string(fmb200_last_error());
    }
  };
  if (main_data.dim == 0) return;
  if (ctx == NULL) {
    const char* dev = getenv("FMB200_DEVICE");
    ck::rc(fmb200_create(&ctx, dev ? atoi(dev) : 0, fm->num_attribute, fm->num_factor, fm->k0, fm->k1));
    ck::rc(fmb200_set_mode(ctx, FMB200_MODE_INORDER));  // the fp64 state
  }
  // draw_all() has moved w0 / w / v on the host since the last pass
  ck::rc(fmb200_set_params(ctx, fm->w0, fm->w.value, fm->num_factor ? fm->v.value[0] : NULL));
  std::vector<double> e;
  for (uint ds = 0; ds < main_data.dim; ds++) {
    Data* d = main_data(ds);
    if (d->relation.dim != 0) throw "the GPU e-term pass does not handle relations";
    LargeSparseMatrixMemory<DATA_FLOAT>* mem = dynamic_cast<LargeSparseMatrixMemory<DATA_FLOAT>*>(d->data);
    if (mem == NULL) throw "the GPU e-term pass needs the row-major data in memory (text input)";
    int slot = -1;
    for (size_t i = 0; i < slots.size(); i++)
      if (slots[i] == d) slot = (int)i;
    if (slot < 0) {
      slot = (int)slots.size();
      slots.push_back(d);
      ck::rc(fmb200_upload_data_aos(ctx, slot, d->num_cases, mem->data.value, d->target.value));
    }
    e.resize(d->num_cases > 0 ? d->num_cases : 1);
    ck::rc(fmb200_mcmc_eterms(ctx, slot, e.data()));
    e_q_term* cache = main_cache(ds);
    for (uint c = 0; c < d->num_cases; c++) {
      cache[c].e = e[c];
      cache[c].q = 0.0;  // fm_learn_mcmc.h:361
    }
  }
}

#endif /* FM_MCMC_ETERMS_B200_H_ */
