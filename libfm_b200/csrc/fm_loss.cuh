// fm_loss.cuh -- the loss rules of the fp64 in-order epochs (SGD and SGDA), and the target clamp.
// Included by fm_inorder.cu (compiled with --fmad=false) and by the wavefront headers, which
// tests/simt/ also compiles for the host.
#pragma once
#include <math.h>

#include "fmb200_internal.h"

namespace fmb {

// the score clipped to the target range (fm_learn_sgd_element.h:58-59, fm_learn.h:138-139)
__device__ __forceinline__ double clamp_target(double p, const HParams& hp) {
  p = fmin(hp.max_target, p);
  return fmax(hp.min_target, p);
}

// d loss / d score of the SGD learner for classification (fm_learn_sgd_element.h:62-64)
__device__ __forceinline__ double sgd_mult_logistic(double p, double y) {
  return -y * (1.0 - 1.0 / (1.0 + exp(-y * p)));
}

// d loss / d score of the SGD learner (fm_learn_sgd_element.h:58-65)
__device__ __forceinline__ double sgd_mult(const HParams& hp, double p, double y) {
  if (hp.task == FMB200_TASK_REGRESSION) return -(y - clamp_target(p, hp));
  return sgd_mult_logistic(p, y);
}

// sgd_mult with the task known at compile time, for a chain that waits on every operation after
// the score.  Regression: the two comparisons and the unclamped difference all start from p at
// once and one select picks among three candidates (two of them known before p), instead of
// compare -> select -> compare -> select -> subtract in series.  Same values as clamp_target's
// fmin(max, .) then fmax(min, .): a NaN or too-large score takes max_target, then anything below
// min_target takes min_target, also when the bounds are inverted.
template <int TASK>
__device__ __forceinline__ double sgd_mult_select(const HParams& hp, double p, double y) {
  if (TASK != FMB200_TASK_REGRESSION) return sgd_mult_logistic(p, y);
  const double m_lo = -(y - hp.min_target), m_hi = -(y - hp.max_target);
  const bool hi = !(p <= hp.max_target);
  const bool lo = hi ? hp.max_target < hp.min_target : (p < hp.min_target);
  const double m_mid = -(y - p);
  return lo ? m_lo : (hi ? m_hi : m_mid);
}

// d loss / d score of the SGDA learner (fm_learn_sgd_element_adapt_reg.h:151-157, :206-211)
__device__ __forceinline__ double sgda_grad_loss(const HParams& hp, double p, double t) {
  if (hp.task == FMB200_TASK_REGRESSION) return 2 * (clamp_target(p, hp) - t);
  return t * ((1.0 / (1.0 + exp(-t * p))) - 1.0);
}

}  // namespace fmb
