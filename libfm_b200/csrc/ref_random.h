// ref_random.h -- the reference's samplers (util/random.h), restated: same algorithms, same
// operations, all drawing from the process-wide libc rand() stream.  Plain C++: the MCMC / ALS
// learner (fm_mcmc.cu) and the command line's model initialisation (host/fm_host.h) consume the
// same stream, so they share this one copy.
// Leva's ratio-of-uniforms normal; Marsaglia-Tsang gamma; Robert's exponential-proposal
// truncated normal; the Abramowitz-Stegun 7.1.26 erf.
#pragma once
#include <cmath>
#include <cstdlib>

namespace ref_random {

inline double ran_uniform() { return rand() / ((double)RAND_MAX + 1); }

inline double ran_gaussian() {
  double u, v, x, y, Q;
  do {
    do {
      u = ran_uniform();
    } while (u == 0.0);
    v = 1.7156 * (ran_uniform() - 0.5);
    x = u - 0.449871;
    y = std::abs(v) + 0.386595;
    Q = x * x + y * (0.19600 * y - 0.25472 * x);
    if (Q < 0.27597) break;
  } while ((Q > 0.27846) || ((v * v) > (-4.0 * u * u * std::log(u))));
  return v / u;
}

inline double ran_gaussian(double mean, double stdev) {
  if ((stdev == 0.0) || std::isnan(stdev)) return mean;
  return mean + stdev * ran_gaussian();
}

inline double ran_gamma(double a) {
  if (a < 1.0) {
    double u;
    do {
      u = ran_uniform();
    } while (u == 0.0);
    return ran_gamma(a + 1.0) * std::pow(u, 1.0 / a);
  }
  const double d = a - 1.0 / 3.0;
  const double c = 1.0 / std::sqrt(9.0 * d);
  double x, v, u;
  do {
    do {
      x = ran_gaussian();
      v = 1.0 + c * x;
    } while (v <= 0.0);
    v = v * v * v;
    u = ran_uniform();
  } while ((u >= (1.0 - 0.0331 * (x * x) * (x * x))) && (std::log(u) >= (0.5 * x * x + d * (1.0 - v + std::log(v)))));
  return d * v;
}

inline double ran_gamma(double a, double b) { return ran_gamma(a) / b; }

inline double ran_exp() { return -std::log(1 - ran_uniform()); }

inline double ran_left_tgaussian(double left) {
  if (left <= 0.0) {
    double r;
    do {
      r = ran_gaussian();
    } while (r < left);
    return r;
  }
  const double alpha_star = 0.5 * (left + std::sqrt(left * left + 4.0));
  for (;;) {
    const double z = ran_exp() / alpha_star + left;
    double d = z - alpha_star;
    d = std::exp(-(d * d) / 2);
    const double u = ran_uniform();
    if (u < d) return z;
  }
}

inline double ran_left_tgaussian(double left, double mean, double stdev) {
  return mean + stdev * ran_left_tgaussian((left - mean) / stdev);
}

inline double ran_right_tgaussian(double right, double mean, double stdev) {
  return mean + stdev * -ran_left_tgaussian(-((right - mean) / stdev));
}

inline double as_erf(double x) {
  const double t = x >= 0 ? 1.0 / (1.0 + 0.3275911 * x) : 1.0 / (1.0 - 0.3275911 * x);
  const double r = 1.0 - (t * (0.254829592 + t * (-0.284496736 + t * (1.421413741 + t * (-1.453152027 + t * 1.061405429))))) *
                             std::exp(-x * x);
  return x >= 0 ? r : -r;
}

inline double cdf_gaussian(double x) { return 0.5 + 0.5 * as_erf(0.707106781 * x); }

}  // namespace ref_random
