// fm_inorder.cu -- sequential-equivalent fp64 path (FMB200_MODE_INORDER).
//
// This translation unit is compiled with --fmad=false: the reference is built
// by g++ -O3 for baseline x86-64 (no FMA contraction), and the parity gate for
// this mode is bit-level agreement of w0/w/V with fm_learn_sgd_element::learn
// (reference src/libfm/src/fm_learn_sgd_element.h:56-67) for regression.
//
// Mapping: ONE warp walks the rows strictly in file order (example t must see
// every update of examples < t, including the bias w0 that every example
// touches -- fm_sgd.h:34-37 -- so the epoch is one serial dependency chain and
// no parallel schedule is sequentially equivalent).  Within a row the warp
// parallelises across factors: lane l owns factors l, l+32, ...  All
// floating-point sums are formed in the reference's order:
//   result = w0 ; += w[id_i]*x_i (i ascending) ; += 0.5*(sum_f^2 - sumsq_f) (f ascending)
//   sum_f  = ((0 + d_0) + d_1) + ...                       (fm_model.h:105-127)
// V is attribute-major fp64 [n][k] here (lane-contiguous, coalesced), versus
// the reference's factor-major layout; only the addressing differs.
#include "fm_device.cuh"
#include "fmb200_internal.h"
#include "fm_inorder_wavefront.cuh"
#include "fm_loss.cuh"
#include "fm_roworder.cuh"
#include "fm_sgda_wavefront.cuh"

namespace fmb {

struct RowCtx {
  int k;
  bool k0, k1;
  const double* w;
  const double* v;
  __device__ RowCtx(const Params64& p, int n_factor, int use_w0, int use_w)
      : k(n_factor), k0(use_w0 != 0), k1(use_w != 0), w(p.w()), v(p.v()) {}
};

// Exact fm_model::predict for one row, executed by a full warp.  Returns the
// score in every lane; sum[j] holds sum_f for f = lane + 32*j.
// KF = factors per lane (1, 2, 4 or 8): the single warp of the in-order epoch has no
// other warp to hide behind, so dead predicated code for unused factor slots (and the
// instruction-cache misses it causes) is paid in full -- the kernels are instantiated per KF.
// w_at(id) and v_at(id, f) read the weights the score uses (SGDA's lambda-step scores with
// stepped-ahead weights); the overload without them reads the state as it is.  VCACHE: short rows
// gather their v_at values into registers first.  That pays for plain reads; SGDA's lambda-step,
// whose every v_at is a computation over four loads, ran 10% slower with it (k = 5, H100).
template <int KF, bool VCACHE, class WAt, class VAt>
__device__ __forceinline__ double predict_row_exact(const RowCtx& m, double w0,
                                                    const uint32_t* __restrict__ col,
                                                    const float* __restrict__ val, uint32_t size,
                                                    double (&sum)[KF], int lane, WAt w_at, VAt v_at) {
  // Issue this lane's factor gathers BEFORE lane 0 walks the linear weights: both are
  // L2 round trips, and the warp would otherwise serialise them (lane 0's branch runs
  // first).  Short rows of models with k <= 32 keep the values in registers.
  constexpr int VC = 8;
  const bool cached = VCACHE && size <= (uint32_t)VC && m.k <= 32;
  double vcache[VC];
  if (cached && lane < m.k) {
#pragma unroll
    for (int i = 0; i < VC; i++)
      if ((uint32_t)i < size) vcache[i] = v_at(col[i], lane);
  }
  double result = 0;
  if (lane == 0) {
    if (m.k0) result += w0;
    if (m.k1) {
      for (uint32_t i = 0; i < size; i++) {
        result += w_at(col[i]) * (double)val[i];
      }
    }
  }
  result = __shfl_sync(0xffffffffu, result, 0);
  double term[KF];
#pragma unroll
  for (int j = 0; j < KF; j++) {
    int f = lane + 32 * j;
    double s = 0, ss = 0;
    if (f < m.k) {
      if (cached) {  // j == 0 only (k <= 32)
#pragma unroll
        for (int i = 0; i < VC; i++) {
          if ((uint32_t)i < size) {
            double d = vcache[i] * (double)val[i];
            s += d;
            ss += d * d;
          }
        }
      } else {
        for (uint32_t i = 0; i < size; i++) {
          double d = v_at(col[i], f) * (double)val[i];
          s += d;
          ss += d * d;
        }
      }
    }
    sum[j] = s;
    term[j] = 0.5 * (s * s - ss);
  }
  // ordered accumulation over f = 0..k-1 (all lanes redundantly, same ops)
#pragma unroll
  for (int j = 0; j < KF; j++) {
    int fbase = 32 * j;
    if (fbase < m.k) {
      int cnt = min(32, m.k - fbase);
      for (int l = 0; l < cnt; l++) {
        double t = __shfl_sync(0xffffffffu, term[j], l);
        result += t;
      }
    }
  }
  return result;
}

template <int KF>
__device__ __forceinline__ double predict_row_exact(const RowCtx& m, double w0,
                                                    const uint32_t* __restrict__ col,
                                                    const float* __restrict__ val, uint32_t size,
                                                    double (&sum)[KF], int lane) {
  return predict_row_exact<KF, true>(
      m, w0, col, val, size, sum, lane, [&](uint32_t id) { return m.w[id]; },
      [&](uint32_t id, int f) { return m.v[(size_t)id * m.k + f]; });
}

template <int KF>
__global__ void __launch_bounds__(32, 1)
    fm_sgd_inorder_kernel(Params64 p, int n_factor, int use_w0, int use_w, HParams hp,
                          uint64_t n_rows, const uint64_t* __restrict__ row_ptr,
                          const uint32_t* __restrict__ col, const float* __restrict__ val,
                          const float* __restrict__ target) {
  const int lane = threadIdx.x;
  const RowCtx m(p, n_factor, use_w0, use_w);
  double* w = p.w();
  double* v = p.v();
  double w0 = *p.w0();
  const double lr = hp.lr, reg0 = hp.reg0, regw = hp.regw, regv = hp.regv;
  double sum[KF];

  for (uint64_t r0 = 0; r0 < n_rows; r0 += 32) {
    // the CSR is immutable: fetch 32 rows' bounds and targets at once
    uint64_t rr = r0 + lane;
    uint64_t my_beg = 0, my_end = 0;
    float my_y = 0.f;
    if (rr < n_rows) {
      my_beg = row_ptr[rr];
      my_end = row_ptr[rr + 1];
      my_y = target[rr];
    }
    int cnt = (int)min((uint64_t)32, n_rows - r0);
    for (int q = 0; q < cnt; q++) {
      uint64_t beg = __shfl_sync(0xffffffffu, my_beg, q);
      uint64_t end = __shfl_sync(0xffffffffu, my_end, q);
      double y = (double)__shfl_sync(0xffffffffu, my_y, q);
      uint32_t size = (uint32_t)(end - beg);
      const uint32_t* c = col + beg;
      const float* x = val + beg;

      const double mult = sgd_mult(hp, predict_row_exact<KF>(m, w0, c, x, size, sum, lane), y);
      // fm_sgd.h:34-37 (replicated in every lane, identical arithmetic)
      if (m.k0) w0 -= lr * (mult + reg0 * w0);
      // fm_sgd.h:38-43 (lane 0 is the only reader/writer of w)
      if (m.k1 && lane == 0) {
        for (uint32_t i = 0; i < size; i++) {
          double* wi = &w[c[i]];
          double cur = *wi;
          cur -= lr * (mult * (double)x[i] + regw * cur);
          *wi = cur;
        }
      }
      // fm_sgd.h:44-50 (lane f%32 is the only reader/writer of V[:, f])
#pragma unroll
      for (int j = 0; j < KF; j++) {
        int f = lane + 32 * j;
        if (f < m.k) {
          for (uint32_t i = 0; i < size; i++) {
            double* vp = &v[(size_t)c[i] * m.k + f];
            double xv = (double)x[i];
            double cur = *vp;
            double grad = sum[j] * xv - cur * xv * xv;
            cur -= lr * (mult * grad + regv * cur);
            *vp = cur;
          }
        }
      }
    }
  }
  if (lane == 0 && m.k0) *p.w0() = w0;
}

// Exact fp64 scores: one warp per row; optional metric partials per block in
// fixed (deterministic) order: each block reduces its warps in warp order.
template <int KF>
__global__ void __launch_bounds__(256)
    fm_predict64_kernel(Params64 p, int n_factor, int use_w0, int use_w, HParams hp, int transform,
                        uint64_t n_rows, const uint64_t* __restrict__ row_ptr,
                        const uint32_t* __restrict__ col, const float* __restrict__ val,
                        const float* __restrict__ target, double* __restrict__ out_pred,
                        double* __restrict__ partials) {
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nwarp = blockDim.x >> 5;
  const RowCtx m(p, n_factor, use_w0, use_w);
  const double w0 = *p.w0();
  double sum[KF];
  double sq = 0, ab = 0, ok = 0;
  // contiguous row ranges per warp keep the reduction order a pure function of
  // (n_rows, grid, block)
  uint64_t total_warps = (uint64_t)gridDim.x * nwarp;
  uint64_t gw = (uint64_t)blockIdx.x * nwarp + warp;
  uint64_t per = (n_rows + total_warps - 1) / total_warps;
  uint64_t rbeg = gw * per, rend = min(n_rows, rbeg + per);
  for (uint64_t r = rbeg; r < rend; r++) {
    uint64_t beg = row_ptr[r], end = row_ptr[r + 1];
    double pr = predict_row_exact<KF>(m, w0, col + beg, val + beg, (uint32_t)(end - beg), sum, lane);
    double y = (double)target[r];
    if (hp.task == FMB200_TASK_REGRESSION) {
      // fm_learn.h:138-142
      const double pc = clamp_target(pr, hp);
      double err = pc - y;
      sq += err * err;
      ab += fabs(err);
      if (transform == 1) pr = pc;
      if (transform == 2) pr = err;  // evaluate in row order on the host (fm_learn.h:139)
    } else {
      // fm_learn.h:118-120
      if (((pr >= 0) && (y >= 0)) || ((pr < 0) && (y < 0))) ok += 1;
      if (transform == 1) pr = 1.0 / (1.0 + exp(-pr));  // fm_learn_sgd.h:84
    }
    if (out_pred != nullptr && lane == 0) out_pred[r] = pr;
  }
  if (partials != nullptr) {
    __shared__ double s_part[8][3];
    if (lane == 0) {
      s_part[warp][0] = sq;
      s_part[warp][1] = ab;
      s_part[warp][2] = ok;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double a = 0, b = 0, c = 0;
      for (int i = 0; i < nwarp; i++) {
        a += s_part[i][0];
        b += s_part[i][1];
        c += s_part[i][2];
      }
      partials[3 * blockIdx.x + 0] = a;
      partials[3 * blockIdx.x + 1] = b;
      partials[3 * blockIdx.x + 2] = c;
    }
  }
}

// MCMC / ALS e-term pass (reference libfm/src/fm_learn_mcmc.h:148-378, no relations): the
// learner re-predicts every case once per iteration through the TRANSPOSED copy of the data, so
// each case accumulates its terms in ascending feature id (ties in row order) and in a different
// association than fm_model::predict:
//   e = sum_f 0.5 q_f^2 ;  q = sum_f sum_i -0.5 v_if^2 x_i^2  (+ sum_i w_i x_i) ;  e = (e + q) + w0
// One thread per case, every operation in that order (this TU is compiled with --fmad=false):
// bit-identical e-terms.  RowOrder (fm_roworder.cuh) gives that order for unsorted rows.
__global__ void __launch_bounds__(128)
    fm_eterm64_kernel(Params64 p, int k, int use_w0, int use_w, uint64_t n_rows,
                      const uint64_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
                      const float* __restrict__ val, double* __restrict__ e_out) {
  const double* w = p.w();
  const double* v = p.v();
  const double w0 = *p.w0();
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rows;
       r += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t beg = row_ptr[r];
    const uint32_t size = (uint32_t)(row_ptr[r + 1] - beg);
    const uint32_t* c = col + beg;
    const float* x = val + beg;
    RowOrder o;
    o.init(c, size);
    double e = 0.0;
    for (int f = 0; f < k; f++) {  // fm_learn_mcmc.h:172-252
      const double q = row_q(o, v, k, f, x);
      e += 0.5 * q * q;
    }
    double q = 0.0;
    for (int f = 0; f < k; f++)  // :255-306
      o.for_each([&](uint32_t pos) {
        const double vif = v[(size_t)c[pos] * k + f];
        const float xi = x[pos];
        q -= 0.5 * vif * vif * xi * xi;  // (((0.5*v)*v)*x)*x, x promoted to double per factor
      });
    if (use_w) o.for_each([&](uint32_t pos) { q += w[c[pos]] * (double)x[pos]; });  // :309-346
    e = e + q;  // :350-362
    if (use_w0) e += w0;
    e_out[r] = e;
  }
}

cudaError_t launch_mcmc_eterms(fmb200_ctx* c, const DataSlot& d, double* e_out) {
  if (d.n_rows == 0) return cudaSuccess;
  const uint64_t blocks = (d.n_rows + 127) / 128;
  const int grid = (int)(blocks < (uint64_t)c->sm_count * 16 ? blocks : (uint64_t)c->sm_count * 16);
  fm_eterm64_kernel<<<grid, 128, 0, c->stream>>>(c->p64, c->k, c->k0, c->k1, d.n_rows, d.row_ptr.get(), d.col.get(),
                                                 d.val.get(), e_out);
  c->launches++;
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------
// SGDA: SGD with self-adaptive regularisation (reference
// libfm/src/fm_learn_sgd_element_adapt_reg.h).  Every training row's theta-step (:136-169) is
// followed by a lambda-step on the next validation row (:201-248) that moves the per-group
// regularisation values; both touch state every later step reads (w0, reg_w, reg_v), so the
// epoch is one chain like the plain in-order epoch and runs the same way: one warp, lane =
// factor, every operation in the reference's order (--fmad=false): bit-identical parameters and
// regularisation values.  Per-group accumulators of a lambda-step live in shared memory
// ([group][factor], one column per lane: no two lanes share a word).  Runs the half-steps
// [h_begin, h_end) of SgdaArgs (fm_sgda_wavefront.cuh).
template <int KF>
__global__ void __launch_bounds__(32, 1) fm_sgda_epoch_kernel(const SgdaArgs a) {
  extern __shared__ double sg_smem[];  // reg_w[G] | reg_v[G][k] | sum_f[G][k] | sum_f_dash_f[G][k] | lwg[G]
  const int lane = threadIdx.x;
  const int k = a.k;
  const uint32_t G = a.n_groups;
  double* s_reg_w = sg_smem;
  double* s_reg_v = s_reg_w + G;
  double* s_sum_f = s_reg_v + (size_t)G * k;
  double* s_sdf = s_sum_f + (size_t)G * k;
  double* s_lwg = s_sdf + (size_t)G * k;
  for (uint32_t i = lane; i < G; i += 32) s_reg_w[i] = a.reg_w[i];
  for (uint32_t i = lane; i < G * (uint32_t)k; i += 32) s_reg_v[i] = a.reg_v[i];
  __syncwarp();
  const RowCtx m(a.p, k, a.use_w0, a.use_w);
  double* w = a.p.w();
  double* v = a.p.v();
  double w0 = *a.p.w0();
  const double lr = a.hp.lr;
  // w' and v' of the lambda-step (:171-199): one theta-step ahead with the stored gradient
  auto w_dash = [&](uint32_t id) {
    const double wv = w[id];
    return wv - lr * (a.grad_w[id] + 2 * s_reg_w[a.group[id]] * wv);
  };
  auto v_dash = [&](uint32_t id, int f) {
    const double vv = v[(size_t)id * k + f];
    return vv - lr * (a.grad_v[(size_t)id * k + f] + 2 * s_reg_v[(size_t)a.group[id] * k + f] * vv);
  };
  double sum[KF];
  uint64_t vc = a.vc0;
  for (uint64_t r = a.h_begin / 2; 2 * r < a.h_end; r++) {
    if (2 * r >= a.h_begin) {  // ---- sgd_theta_step, :136-169 ----
      const uint64_t beg = a.row_ptr[r];
      const uint32_t size = (uint32_t)(a.row_ptr[r + 1] - beg);
      const uint32_t* c = a.col + beg;
      const float* x = a.val + beg;
      const float target = a.target[r];
      const double mult = sgda_grad_loss(a.hp, predict_row_exact<KF>(m, w0, c, x, size, sum, lane), target);
      if (m.k0) w0 -= lr * (mult + 2 * 0.0 * w0);  // reg_0 stays 0 (:60,79)
      if (m.k1 && lane == 0) {
        for (uint32_t i = 0; i < size; i++) {
          const uint32_t id = c[i];
          const uint32_t g = a.group[id];
          double cur = w[id];
          const double gw = mult * x[i];
          a.grad_w[id] = gw;
          cur -= lr * (gw + 2 * s_reg_w[g] * cur);
          w[id] = cur;
        }
      }
#pragma unroll
      for (int j = 0; j < KF; j++) {
        const int f = lane + 32 * j;
        if (f < k) {
          for (uint32_t i = 0; i < size; i++) {
            const uint32_t id = c[i];
            const uint32_t g = a.group[id];
            double* vp = &v[(size_t)id * k + f];
            double cur = *vp;
            const double gv = mult * (x[i] * (sum[j] - cur * x[i]));
            a.grad_v[(size_t)id * k + f] = gv;
            cur -= lr * (gv + 2 * s_reg_v[(size_t)g * k + f] * cur);
            *vp = cur;
          }
        }
      }
      __syncwarp();
    }
    if (a.lambda_steps && a.v_rows > 0 && 2 * r + 1 < a.h_end) {  // ---- sgd_lambda_step, :201-248 ----
      if (vc == a.v_rows) vc = 0;  // :302-305
      const uint64_t beg = a.v_row_ptr[vc];
      const uint32_t size = (uint32_t)(a.v_row_ptr[vc + 1] - beg);
      const uint32_t* c = a.v_col + beg;
      const float* x = a.v_val + beg;
      const float target = a.v_target[vc];
      vc++;
      const double grad_loss =
          sgda_grad_loss(a.hp, predict_row_exact<KF, false>(m, w0, c, x, size, sum, lane, w_dash, v_dash), target);
      if (m.k1) {  // :213-223: lane g owns group g, g+32, ...
        for (uint32_t g = lane; g < G; g += 32) {
          double acc = 0.0;
          for (uint32_t i = 0; i < size; i++)
            if (a.group[c[i]] == g) acc += x[i] * w[c[i]];
          acc = -2 * lr * acc;
          double rw = s_reg_w[g] - lr * grad_loss * acc;
          s_reg_w[g] = (0.0 < rw) ? rw : 0.0;  // std::max(0.0, .)
        }
      }
#pragma unroll
      for (int j = 0; j < KF; j++) {  // :224-247
        const int f = lane + 32 * j;
        if (f < k) {
          double sum_f_dash = 0.0;
          for (uint32_t g = 0; g < G; g++) {
            s_sum_f[(size_t)g * k + f] = 0.0;
            s_sdf[(size_t)g * k + f] = 0.0;
          }
          for (uint32_t i = 0; i < size; i++) {
            const uint32_t id = c[i];
            const uint32_t g = a.group[id];
            const double vv = v[(size_t)id * k + f];
            const double vd = v_dash(id, f);
            sum_f_dash += vd * x[i];
            s_sum_f[(size_t)g * k + f] += vv * x[i];
            s_sdf[(size_t)g * k + f] += vd * x[i] * vv * x[i];
          }
          for (uint32_t g = 0; g < G; g++) {
            const double lvg = -2 * lr * (sum_f_dash * s_sum_f[(size_t)g * k + f] - s_sdf[(size_t)g * k + f]);
            const double rv = s_reg_v[(size_t)g * k + f] - lr * grad_loss * lvg;
            s_reg_v[(size_t)g * k + f] = (0.0 < rv) ? rv : 0.0;
          }
        }
      }
      __syncwarp();
    }
  }
  (void)s_lwg;
  if (lane == 0 && m.k0) *a.p.w0() = w0;
  for (uint32_t i = lane; i < G; i += 32) a.reg_w[i] = s_reg_w[i];
  for (uint32_t i = lane; i < G * (uint32_t)k; i += 32) a.reg_v[i] = s_reg_v[i];
}

// Factors per lane of the one-warp kernels: body(kf) runs with kf.value = KF in {1, 2, 4, 8}, the
// smallest with 32 * KF >= k.  Lane l owns factors l, l + 32, ..., so k is at most 256.
template <class Body>
cudaError_t with_kf(int k, Body&& body) {
  if (k > 32 * 8) return cudaErrorInvalidValue;
  const int kf = (k + 31) / 32;
  if (kf <= 1) return body(std::integral_constant<int, 1>());
  if (kf <= 2) return body(std::integral_constant<int, 2>());
  if (kf <= 4) return body(std::integral_constant<int, 4>());
  return body(std::integral_constant<int, 8>());
}

// update_means (fm_learn_sgd_element_adapt_reg.h:250-274) over the fp64 state: thread 0 walks w, thread
// 1 + f factor f, each one serial chain over j = 0..n-1.  The means it returns are zeroed (:270-273), so
// only the variances are kept: out = [var_w | var_v[k]].
__global__ void fm_sgda_moments_kernel(Params64 p, uint32_t n, int k, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > k) return;
  const double* w = p.w();
  const double* v = p.v();
  double mean = 0, var = 0;
  for (uint32_t j = 0; j < n; j++) {
    const double x = (i == 0) ? w[j] : v[(size_t)j * k + (i - 1)];
    mean += x;
    var += x * x;
  }
  mean /= (double)n;
  out[i] = var / n - mean * mean;
}

cudaError_t launch_sgda_epoch(fmb200_ctx* c, const DataSlot& tr, const DataSlot& va, int lambda_steps) {
  SgdaArgs a;
  a.p = c->p64;
  a.grad_w = c->sgda_grad_w.get();
  a.grad_v = c->sgda_grad_v.get();
  a.reg_w = c->sgda_reg_w.get();
  a.reg_v = c->sgda_reg_v.get();
  a.group = c->sgda_group.get();
  a.n_groups = c->sgda_groups;
  a.k = c->k;
  a.use_w0 = c->k0;
  a.use_w = c->k1;
  a.lambda_steps = lambda_steps;
  a.hp = c->hp;
  a.n_rows = tr.n_rows;
  a.row_ptr = tr.row_ptr.get();
  a.col = tr.col.get();
  a.val = tr.val.get();
  a.target = tr.target.get();
  a.v_rows = va.n_rows;
  a.v_row_ptr = va.row_ptr.get();
  a.v_col = va.col.get();
  a.v_val = va.val.get();
  a.v_target = va.target.get();
  // The wavefront schedule is the default for eligible shapes (bit-identical to the one-warp kernel,
  // tests/test_sgda_wavefront_gpu.py); variant 1 forces the one-warp kernel.
  const bool lam = lambda_steps && va.n_rows > 0;
  const size_t wf_smem = sizeof(double) * (size_t)c->sgda_groups * (1 + (size_t)c->k);
  const bool wavefront = c->tune_variant != 1 &&
                         wavefront_fits(c->k, tr.max_row_nnz) && (!lam || wavefront_fits(c->k, va.max_row_nnz)) &&
                         sizeof(SgdaWindow) + wf_smem <= (size_t)c->max_smem_optin;
  const size_t smem = wavefront ? wf_smem : sgda_smem_bytes(c->sgda_groups, c->k);
  if (smem > (size_t)c->max_smem_optin) return cudaErrorInvalidConfiguration;  // fmb200_sgda_begin refuses it
  auto run = [&](uint64_t h_begin, uint64_t h_end, uint64_t vc0) -> cudaError_t {
    if (h_begin >= h_end) return cudaSuccess;
    a.h_begin = h_begin;
    a.h_end = h_end;
    a.vc0 = vc0;
    if (wavefront) {
      const cudaError_t e =
          cudaFuncSetAttribute(fm_sgda_wavefront_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return e;
      fm_sgda_wavefront_kernel<<<1, 32, smem, c->stream>>>(a);
    } else {
      const cudaError_t e = with_kf(c->k, [&](auto kf) {
        auto kernel = fm_sgda_epoch_kernel<decltype(kf)::value>;
        const cudaError_t e_ = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e_ != cudaSuccess) return e_;
        kernel<<<1, 32, smem, c->stream>>>(a);
        return cudaSuccess;
      });
      if (e != cudaSuccess) return e;
    }
    c->launches++;
    return cudaGetLastError();
  };
  auto moments = [&]() -> cudaError_t {
    fm_sgda_moments_kernel<<<(c->k + 32) / 32, 32, 0, c->stream>>>(c->p64, c->n, c->k, c->sgda_moments.get());
    c->launches++;
    return cudaGetLastError();
  };
  // The epoch's last update_means (:298, :304-307) comes at its start, or, when the validation cursor
  // wraps, between theta-step t* = floor((N - 1) / V) * V and its lambda-step: the launch is cut there.
  const uint64_t N = tr.n_rows, V = va.n_rows;
  const uint64_t t_star = sgda_last_moments_step(N, V, lam);
  cudaError_t e = cudaSuccess;
  if (t_star == 0) {
    if ((e = moments()) != cudaSuccess || (e = run(0, 2 * N, 0)) != cudaSuccess) return e;
  } else if ((e = run(0, 2 * t_star + 1, 0)) != cudaSuccess || (e = moments()) != cudaSuccess ||
             (e = run(2 * t_star + 1, 2 * N, V)) != cudaSuccess) {
    return e;
  }
  c->last_cfg =
      wavefront ? wavefront_config((int)(sizeof(SgdaWindow) + smem)) : EpochConfig{32, 1, 1, 1, 32, (int)smem, 0};
  return cudaSuccess;
}

cudaError_t launch_sgd_inorder(fmb200_ctx* c, const DataSlot& d) {
  // The wavefront schedule (k <= 8, rows of <= 4 entries) is the default for eligible shapes:
  // bit-identical to the row-at-a-time kernel on the device (tests/test_wavefront_gpu.py, r02) and
  // 6.7x faster on C2 (0.210 s vs 1.416 s per epoch).  variant 1 forces the row-at-a-time kernel.
  if (c->tune_variant != 1 && wavefront_fits(c->k, d.max_row_nnz) && d.n_rows > 0) {
#define FMB_WAVEFRONT(K0, TASK)                                                                       \
  fm_sgd_inorder_wavefront_kernel<K0, TASK><<<1, 32, 0, c->stream>>>(c->p64, c->k, c->k0, c->k1, c->hp, \
                                                                     d.n_rows, d.row_ptr.get(), d.col.get(),  \
                                                                     d.val.get(), d.target.get())
    const bool reg = c->hp.task == FMB200_TASK_REGRESSION;
    if (c->k0 && reg) FMB_WAVEFRONT(true, FMB200_TASK_REGRESSION);
    else if (c->k0) FMB_WAVEFRONT(true, FMB200_TASK_CLASSIFICATION);
    else if (reg) FMB_WAVEFRONT(false, FMB200_TASK_REGRESSION);
    else FMB_WAVEFRONT(false, FMB200_TASK_CLASSIFICATION);
#undef FMB_WAVEFRONT
    c->launches++;
    c->last_cfg = wavefront_config(0);
    return cudaGetLastError();
  }
  const cudaError_t e = with_kf(c->k, [&](auto kf) {
    fm_sgd_inorder_kernel<decltype(kf)::value><<<1, 32, 0, c->stream>>>(
        c->p64, c->k, c->k0, c->k1, c->hp, d.n_rows, d.row_ptr.get(), d.col.get(), d.val.get(), d.target.get());
    return cudaSuccess;
  });
  if (e != cudaSuccess) return e;
  c->launches++;
  c->last_cfg = EpochConfig{32, 1, 1, 1, 32, 0};
  return cudaGetLastError();
}

cudaError_t launch_predict64(fmb200_ctx* c, const DataSlot& d, int transform, double* out_pred,
                             double* partials, int n_blocks) {
  const cudaError_t e = with_kf(c->k, [&](auto kf) {
    fm_predict64_kernel<decltype(kf)::value><<<n_blocks, 256, 0, c->stream>>>(
        c->p64, c->k, c->k0, c->k1, c->hp, transform, d.n_rows, d.row_ptr.get(), d.col.get(), d.val.get(),
        d.target.get(), out_pred, partials);
    return cudaSuccess;
  });
  if (e != cudaSuccess) return e;
  c->launches++;
  return cudaGetLastError();
}

}  // namespace fmb
