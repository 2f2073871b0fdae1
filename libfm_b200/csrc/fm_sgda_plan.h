// fm_sgda_plan.h -- the launches of one SGDA epoch (fm_learn_sgd_element_adapt_reg.h:295-311), resident or
// streamed in blocks.  Plain C++ without CUDA: the library and tests/sgda_plan_dump.cpp both compile it.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

namespace fmb {

// The step t* whose lambda-step follows the epoch's last update_means (:298, :302-307), 0 when that call
// is the one at the epoch's start: the cursor over V validation rows restarts before the lambda-steps
// t = V, 2V, ... of an epoch of N theta-steps.
inline uint64_t sgda_last_moments_step(uint64_t n_train, uint64_t n_val, bool lambda_steps) {
  if (!lambda_steps || n_val == 0 || n_train <= n_val) return 0;
  return (n_train - 1) / n_val * n_val;
}

// One launch of the epoch: the half-steps [h_begin, h_end) -- half-step 2t is the theta-step on training row t,
// 2t + 1 the lambda-step after it, on validation row t mod V -- with vc0 the validation cursor at h_begin (V when
// the restart is due).  train_block / val_block: the block of each set the launch reads, -1 when that set is
// resident or the launch reads none of it.  moments: the moments kernel runs before the launch.
struct SgdaLaunch {
  uint64_t h_begin, h_end, vc0;
  int64_t train_block, val_block;
  bool moments;
};

// The launches of an epoch of N training and V validation rows.  train_lo[nbt + 1] / val_lo[nbv + 1]: the first
// row of every block, then the row count; nbt / nbv = 0 for a set resident in one slot.  Cuts:
//  - at every training block start T (half-step 2T): a launch reads one training block;
//  - with lambda-steps and a validation set streamed in two blocks or more, before every lambda-step whose row
//    starts a block, the cursor's restart at row 0 included (half-step 2t + 1, t >= 1): a launch reads one
//    validation block and never wraps inside it.  A single block holds rows [0, V) as a resident set does, so
//    its launches wrap as the resident ones do;
//  - before the lambda-step t* (half-step 2t* + 1) when t* > 0, the moments being taken there; with a streamed
//    validation set t* is already a restart cut.
// The resident epoch, and one whose sets come in one block each, is one launch, or two around t*.  A cut only
// splits the chain of steps between two launches: every step still runs once, in order, with the arithmetic of
// the uncut launch.
inline std::vector<SgdaLaunch> sgda_plan(uint64_t N, uint64_t V, bool lambda_steps, const uint32_t* train_lo,
                                         uint64_t nbt, const uint32_t* val_lo, uint64_t nbv) {
  const bool lam = lambda_steps && V > 0;
  const uint64_t t_star = sgda_last_moments_step(N, V, lam);
  std::vector<uint64_t> cut = {0, 2 * N};
  for (uint64_t b = 1; b < nbt; b++) cut.push_back(2 * (uint64_t)train_lo[b]);
  if (lam && nbv > 1)
    for (uint64_t m = 0; m * V < N; m++)
      for (uint64_t b = 0; b < nbv; b++) {
        const uint64_t t = m * V + val_lo[b];
        if (t >= 1 && t < N) cut.push_back(2 * t + 1);
      }
  if (t_star > 0) cut.push_back(2 * t_star + 1);
  std::sort(cut.begin(), cut.end());
  cut.erase(std::unique(cut.begin(), cut.end()), cut.end());
  auto block_of = [](const uint32_t* lo, uint64_t nb, uint64_t row) -> int64_t {
    if (nb == 0) return -1;
    return (int64_t)(std::upper_bound(lo, lo + nb, (uint32_t)row) - lo) - 1;
  };
  std::vector<SgdaLaunch> plan;
  if (N == 0) plan.push_back(SgdaLaunch{0, 0, 0, -1, -1, true});  // the moments alone
  for (size_t i = 0; i + 1 < cut.size(); i++) {
    const uint64_t h0 = cut[i], pair = h0 / 2;  // pair: the first step the launch touches
    SgdaLaunch l;
    l.h_begin = h0;
    l.h_end = cut[i + 1];
    l.vc0 = (!lam || pair == 0) ? 0 : (pair - 1) % V + 1;  // `pair` lambda-steps have run
    l.train_block = block_of(train_lo, nbt, pair);
    l.val_block = lam ? block_of(val_lo, nbv, pair % V) : -1;
    l.moments = t_star == 0 ? h0 == 0 : h0 == 2 * t_star + 1;
    plan.push_back(l);
  }
  return plan;
}

}  // namespace fmb
