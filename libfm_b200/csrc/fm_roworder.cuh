// fm_roworder.cuh -- a case's entries in (feature id, position) order, the order in which the
// MCMC / ALS learner reaches them through the transposed data (reference Data.h:292-341).
// Used by the e-term pass and the q rebuild of the Gibbs sweep (fm_mcmc.cu), with
// row_of, the entry -> case lookup of the index builds (fm_ordered.cu, fm_mcmc.cu).
#pragma once
#include <stdint.h>

namespace fmb {

// Rows whose ids are not ascending are visited through a per-thread order array (rows of
// <= ET_LOCAL entries) or by repeated selection (longer rows).
constexpr int ET_LOCAL = 64;

struct RowOrder {
  const uint32_t* c;
  uint32_t size;
  bool sorted;
  unsigned short ord[ET_LOCAL];
  __device__ __forceinline__ void init(const uint32_t* col, uint32_t n) {
    c = col;
    size = n;
    sorted = true;
    for (uint32_t i = 1; i < n; i++)
      if (col[i] < col[i - 1]) sorted = false;
    if (!sorted && n <= (uint32_t)ET_LOCAL) {  // stable insertion sort by id
      for (uint32_t i = 0; i < n; i++) ord[i] = (unsigned short)i;
      for (uint32_t i = 1; i < n; i++) {
        const unsigned short o = ord[i];
        uint32_t j = i;
        while (j > 0 && col[ord[j - 1]] > col[o]) {
          ord[j] = ord[j - 1];
          j--;
        }
        ord[j] = o;
      }
    }
  }
  // position of the i-th entry in (id, position) order; `prev` = position of the (i-1)-th
  __device__ __forceinline__ uint32_t at(uint32_t i, uint32_t prev) const {
    if (sorted) return i;
    if (size <= (uint32_t)ET_LOCAL) return ord[i];
    // selection: the smallest (id, position) greater than (c[prev], prev)
    uint32_t best = 0xffffffffu;
    for (uint32_t j = 0; j < size; j++) {
      const bool after = (i == 0) || c[j] > c[prev] || (c[j] == c[prev] && j > prev);
      if (!after) continue;
      if (best == 0xffffffffu || c[j] < c[best]) best = j;
    }
    return best;
  }
  // fn(pos) for every entry, in (id, position) order
  template <class F>
  __device__ __forceinline__ void for_each(F&& fn) const {
    uint32_t pos = 0;
    for (uint32_t i = 0; i < size; i++) {
      pos = at(i, pos);
      fn(pos);
    }
  }
};

// q_f of a case: 0 + sum of v[id][f] * x over its entries in (id, position) order (fm_learn_mcmc.h:172-252,
// add_main_q :406-428); v is attribute-major [n][k], x the case's values
__device__ __forceinline__ double row_q(const RowOrder& o, const double* v, int k, int f, const float* x) {
  double q = 0.0;
  o.for_each([&](uint32_t pos) { q += v[(size_t)o.c[pos] * k + f] * (double)x[pos]; });
  return q;
}

// The e-term of one case (fm_learn_mcmc.h:172-362), every operation in the reference's order:
//   e = sum_f 0.5 q_f^2 ;  q = sum_f sum_i -0.5 v_if^2 x_i^2  (+ sum_i w_i x_i) ;  e = (e + q) + w0
// rel_f(f, q_f) adds the relation blocks' q_f of the case to q_f before it is squared (:227-240), rel(q) their
// q to q before the merge (:352-368); without relations both leave their argument alone.
template <class RF, class R>
__device__ __forceinline__ double case_eterm(const RowOrder& o, const double* v, const double* w, int k, int use_w,
                                             int use_w0, double w0, const float* x, RF&& rel_f, R&& rel) {
  double e = 0.0;
  for (int f = 0; f < k; f++) {  // :172-252
    double q = row_q(o, v, k, f, x);
    rel_f(f, q);
    e += 0.5 * q * q;
  }
  double q = 0.0;
  for (int f = 0; f < k; f++)  // :255-306
    o.for_each([&](uint32_t pos) {
      const double vif = v[(size_t)o.c[pos] * k + f];
      const float xi = x[pos];
      q -= 0.5 * vif * vif * xi * xi;  // (((0.5*v)*v)*x)*x, x promoted to double per factor
    });
  if (use_w) o.for_each([&](uint32_t pos) { q += w[o.c[pos]] * (double)x[pos]; });  // :309-346
  rel(q);
  e = e + q;  // :350-362
  if (use_w0) e += w0;
  return e;
}

// row containing entry e: the last r with row_ptr[r] <= e (empty rows skipped by construction)
__device__ __forceinline__ uint64_t row_of(const uint64_t* __restrict__ rp, uint64_t n_rows, uint64_t e) {
  uint64_t lo = 0, hi = n_rows;  // invariant: rp[lo] <= e < rp[hi]
  while (hi - lo > 1) {
    const uint64_t mid = (lo + hi) >> 1;
    if (rp[mid] <= e) lo = mid;
    else hi = mid;
  }
  return lo;
}

}  // namespace fmb
