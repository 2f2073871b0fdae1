// fm_sgda_wavefront.cuh -- the SGDA epoch (fm_learn_sgd_element_adapt_reg.h:295-311): the one-warp
// kernel's arguments, and the wavefront schedule for short rows and small k, built from the window
// pieces of fm_inorder_wavefront.cuh.  Included by fm_inorder.cu (compiled with --fmad=false); also
// compiled for the host by tests/simt/ (FMB_SIMT_HOST).
#pragma once
#include "fm_inorder_wavefront.cuh"
#include "fm_loss.cuh"
#include "fmb200_internal.h"

namespace fmb {

// One launch runs the half-steps [h_begin, h_end) of an epoch: half-step 2t is the theta-step on
// training row t, 2t + 1 the lambda-step that follows it (skipped when lambda_steps == 0).  The
// epoch is cut in two where the reference takes its last moments (update_means, :304-307), between
// a theta-step and its lambda-step.  vc0 is the validation cursor at h_begin (v_rows = at the end).
struct SgdaArgs {
  Params64 p;
  double* grad_w;        // [n]
  double* grad_v;        // [n][k] attribute-major
  double* reg_w;         // [G]
  double* reg_v;         // [G][k]
  const uint32_t* group; // [n]
  uint32_t n_groups;
  int k, use_w0, use_w, lambda_steps;
  HParams hp;
  uint64_t n_rows, v_rows;
  uint64_t h_begin, h_end, vc0;
  const uint64_t *row_ptr, *v_row_ptr;
  const uint32_t *col, *v_col;
  const float *val, *v_val, *target, *v_target;
};

// ---------------------------------------------------------------------------------------
// Wavefront schedule of the SGDA epoch (k <= WF_K, train and validation rows of <= WF_Z entries).
//
// Step t is the pair (theta_t on train row r_t, lambda_t on validation row s_t).  theta_t writes w,
// v, grad_w, grad_v of r_t's features; lambda_t reads those of s_t's features and writes only
// reg_w / reg_v.  So a window of consecutive pairs reads, at its start, everything its steps read,
// as long as no feature of r_t appears in r_t' (t' > t) or in s_t' (t' >= t).  Validation rows may
// share features with each other; hash collisions only shorten a window; the cursor restart may
// fall anywhere inside one.  A pair whose validation row meets its own train row at the head of a
// window is split: the window ends after its theta-step, and the next one starts with its lambda-step.
//
// One warp.  Per window:
//   1. lane = pair: load the pair's two rows, find the conflict-free prefix P (WfHash: r_t is marked,
//      s_t only looked up);
//   2. lanes < P gather w / V (and for s_t grad_w / grad_v) and form the theta score's addends
//      a_i = w_i x_i, b_f = 0.5 (sum_f^2 - sumsq_f) -- they read nothing the chain moves;
//   3. the chain walks t = 0..P-1 with the one-warp kernel's arithmetic, lane = factor:
//      theta score ((w0 + a_1) + ...) + b_k, loss, w0; a snapshot of the reg values theta_t's update
//      reads; lambda score through w' / v' on the current reg; the reg_w / reg_v updates of all G
//      groups.  Only this part is serial;
//   4. lane = pair: the theta updates of w, v, grad_w, grad_v (WfGather::scatter).
// Bit-identical to fm_sgda_epoch_kernel (tests/test_sgda_wavefront_gpu.py).
struct SgdaWindow {
  static constexpr int NA = WF_Z + WF_K;  // addends of a theta score
  double ta[32][NA];                      // theta addends, -0.0 (the identity of +) in unused slots
  double rw[32][WF_Z];                    // reg_w of each theta entry's group as theta_t reads it
  double rv[32][WF_Z][WF_K];              // reg_v likewise
  double lw[32][WF_Z], lgw[32][WF_Z];     // lambda row: w, grad_w
  double lv[32][WF_Z][WF_K], lgv[32][WF_Z][WF_K];
  double mult[32];                        // theta_t's loss gradient
  uint32_t tg[32][WF_Z], lg[32][WF_Z];    // groups of the entries
  float lx[32][WF_Z];
  float ty[32], ly[32];
  int tsize[32], lsize[32];               // -1: the pair has no theta- / lambda-step in this window
  unsigned int hash[WF_HASH];             // WfHash's table, marked with the r_t
};

__global__ void __launch_bounds__(32, 1) fm_sgda_wavefront_kernel(const SgdaArgs a) {
  __shared__ SgdaWindow s;
#ifdef FMB_SIMT_HOST
  double* const sw_smem = simt::dynamic_smem;
#else
  extern __shared__ double sw_smem[];  // reg_w[G] | reg_v[G][k]
#endif
  const int lane = threadIdx.x;
  const unsigned full = 0xffffffffu;
  const int k = a.k;
  const uint32_t G = a.n_groups;
  const bool k0 = a.use_w0 != 0, k1 = a.use_w != 0;
  double* s_reg_w = sw_smem;
  double* s_reg_v = s_reg_w + G;
  for (uint32_t i = lane; i < G; i += 32) s_reg_w[i] = a.reg_w[i];
  for (uint32_t i = lane; i < G * (uint32_t)k; i += 32) s_reg_v[i] = a.reg_v[i];
  WfHash hash(s.hash, lane);
  __syncwarp();
  double* w = a.p.w();
  double* v = a.p.v();
  double w0 = *a.p.w0();
  const double lr = a.hp.lr;
  const bool lam = a.lambda_steps && a.v_rows > 0;
  const uint64_t vstart = (a.vc0 >= a.v_rows) ? 0 : a.vc0;  // the first lambda-step restarts a full cursor
  const uint64_t p_first = a.h_begin / 2;

  uint64_t hs = a.h_begin;
  while (hs < a.h_end) {
    // (1) the window's pairs and their conflict-free prefix
    const uint64_t p = hs / 2 + lane;
    const bool valid = 2 * p < a.h_end;
    const bool has_theta = valid && 2 * p >= hs;
    bool has_lambda = valid && lam && 2 * p + 1 < a.h_end;
    uint64_t beg = 0, end = 0;
    float ty = 0.f, ly = 0.f;
    if (has_theta) {
      beg = a.row_ptr[p];
      end = a.row_ptr[p + 1];
      ty = a.target[p];
    }
    WfRow trow;
    trow.load(a.col, a.val, beg, end);
    beg = end = 0;
    if (has_lambda) {
      const uint64_t s_row = (vstart + (p - p_first)) % a.v_rows;  // :302-305
      beg = a.v_row_ptr[s_row];
      end = a.v_row_ptr[s_row + 1];
      ly = a.v_target[s_row];
    }
    WfRow lrow;
    lrow.load(a.v_col, a.v_val, beg, end);
    const bool dup = trow.names_a_feature_twice();
    hash.next_window(lane);
    hash.mark(trow);
    // r_t' with t' < t has one of r_t's features, or r_t' with t' <= t one of s_t's
    int P = wf_prefix(hash.earlier_has(trow, lane) | hash.this_or_earlier_has(lrow, lane) | !valid);
    // Lane 0 conflicts only through its own pair: split it (theta now, lambda heads the next window).
    const bool split = P == 0;
    if (split) {
      P = 1;
      if (lane == 0) has_lambda = false, lrow.size = 0;
    }
    const bool active = lane < P;

    // (2) gathers and theta addends
    WfGather gat;
    if (active) {
      s.tsize[lane] = has_theta ? trow.size : -1;
      s.lsize[lane] = has_lambda ? lrow.size : -1;
      s.ty[lane] = ty;
      s.ly[lane] = ly;
#pragma unroll
      for (int j = 0; j < WF_Z; j++) {
        const uint32_t id = lrow.id[j];
        double lwj = 0, lgwj = 0;
        uint32_t g = 0;
        if (j < lrow.size) {
          g = a.group[id];
          if (k1) {
            lwj = w[id];
            lgwj = a.grad_w[id];
          }
        }
        s.lg[lane][j] = g;
        s.lx[lane][j] = lrow.x[j];
        s.lw[lane][j] = lwj;
        s.lgw[lane][j] = lgwj;
#pragma unroll
        for (int f = 0; f < WF_K; f++) {
          double a_v = 0, a_g = 0;
          if (j < lrow.size && f < k) {
            a_v = v[(size_t)id * k + f];
            a_g = a.grad_v[(size_t)id * k + f];
          }
          s.lv[lane][j][f] = a_v;
          s.lgv[lane][j][f] = a_g;
        }
      }
      gat.gather(trow, w, v, k, k1);
#pragma unroll
      for (int j = 0; j < WF_Z; j++) s.tg[lane][j] = (j < trow.size) ? a.group[trow.id[j]] : 0;
      gat.addends(trow, k, k1, s.ta[lane]);
    }
    __syncwarp();
    // (3) the chain, lane = factor
    for (int t = 0; t < P; t++) {
      const int ts = s.tsize[t];
      if (ts >= 0) {  // ---- theta score, loss, w0 (:137-152) ----
        double pr = 0.0;
        if (k0) pr += w0;
#pragma unroll
        for (int q = 0; q < SgdaWindow::NA; q++) pr += s.ta[t][q];
        const double mult = sgda_grad_loss(a.hp, pr, (double)s.ty[t]);
        if (k0) w0 -= lr * (mult + 2 * 0.0 * w0);  // reg_0 stays 0 (:60,79)
        if (lane == 0) s.mult[t] = mult;
        // the reg values theta_t's w / v updates read (:158, :166): those after lambda_{t-1}
        for (int j = 0; j < ts; j++) {
          const uint32_t g = s.tg[t][j];
          if (lane == 0) s.rw[t][j] = s_reg_w[g];
          if (lane < k) s.rv[t][j][lane] = s_reg_v[(size_t)g * k + lane];
        }
      }
      const int ls = s.lsize[t];
      if (ls >= 0) {  // ---- lambda-step (:201-248) on w' / v' (:171-199) ----
        double pr = 0.0;
        if (k0) pr += w0;
        if (k1)
          for (int j = 0; j < ls; j++) {
            const double wj = s.lw[t][j];
            const double wd = wj - lr * (s.lgw[t][j] + 2 * s_reg_w[s.lg[t][j]] * wj);
            pr += wd * (double)s.lx[t][j];
          }
        double vd[WF_Z];
        double term = -0.0;
        if (lane < k) {
          double sf = 0, ss = 0;
#pragma unroll
          for (int j = 0; j < WF_Z; j++)
            if (j < ls) {
              const double vj = s.lv[t][j][lane];
              vd[j] = vj - lr * (s.lgv[t][j][lane] + 2 * s_reg_v[(size_t)s.lg[t][j] * k + lane] * vj);
              const double d = vd[j] * (double)s.lx[t][j];
              sf += d;
              ss += d * d;
            }
          term = 0.5 * (sf * sf - ss);
        }
#pragma unroll
        for (int f = 0; f < WF_K; f++) pr += __shfl_sync(full, term, f);  // lanes >= k hold -0.0
        const double grad_loss = sgda_grad_loss(a.hp, pr, (double)s.ly[t]);
        __syncwarp();  // every lane has read the reg values of the score before any is replaced
        if (k1) {      // :212-223, lane g owns group g, g + 32, ...
          for (uint32_t g = lane; g < G; g += 32) {
            double acc = 0.0;
            for (int j = 0; j < ls; j++)
              if (s.lg[t][j] == g) acc += s.lx[t][j] * s.lw[t][j];
            acc = -2 * lr * acc;
            const double rw = s_reg_w[g] - lr * grad_loss * acc;
            s_reg_w[g] = (0.0 < rw) ? rw : 0.0;  // std::max(0.0, .)
          }
        }
        if (lane < k) {  // :224-247
          double sum_f_dash = 0.0;
#pragma unroll
          for (int j = 0; j < WF_Z; j++)
            if (j < ls) sum_f_dash += vd[j] * s.lx[t][j];
          for (uint32_t g = 0; g < G; g++) {
            double sf = 0.0, sdf = 0.0;
#pragma unroll
            for (int j = 0; j < WF_Z; j++)
              if (j < ls && s.lg[t][j] == g) {
                const double vj = s.lv[t][j][lane];
                sf += vj * s.lx[t][j];
                sdf += vd[j] * s.lx[t][j] * vj * s.lx[t][j];
              }
            const double lvg = -2 * lr * (sum_f_dash * sf - sdf);
            const double rv = s_reg_v[(size_t)g * k + lane] - lr * grad_loss * lvg;
            s_reg_v[(size_t)g * k + lane] = (0.0 < rv) ? rv : 0.0;
          }
        }
        __syncwarp();
      }
    }
    __syncwarp();  // mult and the reg snapshots reach the scatter

    // (4) the theta updates, lane = pair (:153-168)
    if (active && has_theta) {
      const double mult = s.mult[lane];
      gat.scatter(
          trow, dup, w, v, k, k1,
          [&](int j, uint32_t at, double c) {
            const double gw = mult * trow.x[j];
            a.grad_w[at] = gw;
            return c - lr * (gw + 2 * s.rw[lane][j] * c);
          },
          [&](int j, int f, size_t at, double c) {
            const double x = trow.x[j];
            const double gv = mult * (x * (gat.sum[f] - c * x));
            a.grad_v[at] = gv;
            return c - lr * (gv + 2 * s.rv[lane][j][f] * c);
          });
    }
    __syncwarp();  // the next window's gathers (other lanes) must see these stores
    hs = split ? 2 * (hs / 2) + 1 : 2 * (hs / 2 + P);
  }
  if (lane == 0 && k0) *a.p.w0() = w0;
  for (uint32_t i = lane; i < G; i += 32) a.reg_w[i] = s_reg_w[i];
  for (uint32_t i = lane; i < G * (uint32_t)k; i += 32) a.reg_v[i] = s_reg_v[i];
}

}  // namespace fmb
