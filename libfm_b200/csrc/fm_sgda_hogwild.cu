// fm_sgda_hogwild.cu -- SGDA (fm_learn_sgd_element_adapt_reg.h) in HOGWILD mode: the windowed fp32 epoch.
//
// The epoch is cut into windows of W consecutive training rows (W a library constant, kSgdaWindowRows, not the
// grid), the first at row 0.  One cooperative launch walks the windows; each is up to four phases behind grid
// barriers:
//   theta   a warp per training row (lanes over factors) scores the row from the state as the window found
//           it, takes the reference's theta-step (:136-169) with reg as the previous window left it -- a
//           feature the row names twice is stepped twice in a row, from where its first step ended --, damps
//           each step by the row-lane epoch's gamma(c, u) and adds it to the fixed-point accumulator
//           (fm_hogwild_common.cuh: acc_add, 2^-32, exact in any order).  Each row's gradient of a feature (the
//           one its last entry of the feature left) goes to a second accumulator, and the feature's stamp
//           records the window.
//   fold    every element of a feature the window stamped: state += its steps, stored gradient := its
//           gradients' sum; both accumulators back to zero.  A step that was not finite or not below 2^11 set
//           the flag, and then the whole state turns NaN.
//   lambda  (lambda_steps) a warp per lambda-step, on validation row (global step) mod V, in fp64 from the
//           folded fp32 state and stored gradients and the reg the theta-phase read: sgd_lambda_step's per-group
//           terms (:201-248), one row of G * (k + 1) doubles per step.
//   reg     warp e sums column e of those rows over the row index in a fixed order and sets
//           reg <- max(0, reg + sum), once per window.
// The moments (update_means, :250-274) are a fixed-order reduction per column of the state the lambda-steps
// read in the window that holds the epoch's last cursor restart (the epoch's start when there is none).
// Which warp takes which row only decides the order in which integers are added, so the result is the same
// bits on every run and at every grid size.  tests/test_sgda_hogwild_gpu.py holds it to an fp64 statement of the
// windows (DESIGN.md section 3.5).  The stamp table and the cooperative launch are fm_window.cuh's,
// shared with the reproducible SGD epoch.  Its windows are short (4096 rows): measured on an H100, the SGD epoch's
// touched-feature list and fold (window_touch, window_fold) made this epoch 1.1-1.3 ms slower on C2, so it scans.
#include "fm_window.cuh"

namespace fmb {

namespace {

constexpr int kSgdaThreads = 256;

struct SgdaHwArgs {
  const uint64_t* row_ptr;
  const uint32_t* col;
  const float* val;
  const float* target;
  uint64_t n_rows;
  const uint64_t* v_row_ptr;
  const uint32_t* v_col;
  const float* v_val;
  const float* v_target;
  uint64_t v_rows;
  const float* feat_cnt;  // occurrences of each feature in the training set
  float conc_scale;       // min(W, N) / N: count -> concurrency
  float w0_conc;          // min(W, N): the bias's concurrency
  float* state;           // packed fp32 state (Params32)
  float* grad;            // stored gradients, element for element beside the state
  unsigned long long* acc;   // steps [n_floats], then the divergence flag
  unsigned long long* gacc;  // gradients [n_floats]
  uint64_t n_floats, off_w, off_v;
  int ws, kp, k;
  uint32_t n;
  uint32_t* stamp;  // [n]: the stamp of the last window that named the feature
  uint32_t stamp0;  // stamp of this epoch's window 0
  uint32_t* list;           // the SGD epoch's list and count words: set by launch_windows, not used here
  unsigned long long* aux;
  double* reg_w;    // [G]
  double* reg_v;    // [G][k]
  const uint32_t* group;
  uint32_t G;
  double* part;     // [W][G * (k + 1)]: the lambda-steps' terms, v then w per group
  double* moments;  // var_w | var_v[k]
  uint64_t W;
  int64_t moments_window;  // -1: the epoch's start
  int use_w0, use_w, task, lambda, damp;
  float lr, min_target, max_target;
  unsigned int* gbar;
  uint32_t gbar_base;
};

__device__ __forceinline__ float ldf(const float* p) { return __ldcg(p); }
__device__ __forceinline__ double ldd(const double* p) { return __ldcg(p); }

// the gradient sum an accumulated element stores
__device__ __forceinline__ float acc_value(unsigned long long u) {
  return (float)((double)(long long)u * (1.0 / (double)kAccScale));
}

// whether another entry of row [beg, beg + size) names feature id: before entry i (prev), after it (!last)
__device__ __forceinline__ void occurrences(const uint32_t* col, uint64_t beg, uint32_t size, uint32_t i, uint32_t id,
                                            bool* prev, bool* last) {
  bool p = false, l = true;
  for (uint32_t j = 0; j < size; j++)
    if (j != i && __ldg(col + beg + j) == id) {
      if (j < i) p = true;
      else l = false;
    }
  *prev = p;
  *last = l;
}

// update_means of the columns (w, v_0 .. v_{k-1}): warp `gw` of `GW` takes columns gw, gw + GW, ...; lane l sums
// features l, l + 32, ... and the warp adds the lanes in a fixed tree
__device__ void sgda_moments(const SgdaHwArgs& a, int gw, int GW, int lane) {
  for (int c = gw; c <= a.k; c += GW) {
    double s = 0.0, q = 0.0;
    for (uint32_t i = lane; i < a.n; i += 32) {
      const double x = c == 0 ? ldf(a.state + a.off_w + (uint64_t)i * a.ws)
                              : ldf(a.state + a.off_v + (uint64_t)i * a.kp + (c - 1));
      s += x;
      q += x * x;
    }
    s = warp_sum_d(s);
    q = warp_sum_d(q);
    if (lane == 0) {
      const double mean = s / a.n;
      a.moments[c] = q / a.n - mean * mean;
    }
  }
}

template <int KF>
__device__ void theta_row(const SgdaHwArgs& a, uint64_t r, uint32_t stamp, int lane, long long* w0_sum) {
  const uint64_t beg = __ldg(a.row_ptr + r);
  const uint32_t size = (uint32_t)(__ldg(a.row_ptr + r + 1) - beg);
  const float y = __ldg(a.target + r);
  const int k = a.k;
  const float* w = a.state + a.off_w;
  const float* v = a.state + a.off_v;
  unsigned long long* bad = a.acc + a.n_floats;
  // ---- the score from the window's state ----
  float s[KF], q = 0.f, lin = 0.f, xx = 0.f;
#pragma unroll
  for (int j = 0; j < KF; j++) s[j] = 0.f;
  for (uint32_t i = 0; i < size; i++) {
    const uint32_t id = __ldg(a.col + beg + i);
    const float x = __ldg(a.val + beg + i);
    if (a.use_w) lin += ldf(w + (uint64_t)id * a.ws) * x;
    xx += x * x;
#pragma unroll
    for (int j = 0; j < KF; j++) {
      const int f = lane + 32 * j;
      if (f < k) {
        const float vx = ldf(v + (uint64_t)id * a.kp + f) * x;
        s[j] += vx;
        q += vx * vx;
      }
    }
  }
  float s2 = 0.f;
#pragma unroll
  for (int j = 0; j < KF; j++) s2 += s[j] * s[j];
  s2 = warp_sum(s2);
  const float sq = warp_sum(q);
  const float p = (a.use_w0 ? ldf(a.state) : 0.f) + lin + 0.5f * (s2 - sq);
  const LossStep l = loss_step(a.task, a.min_target, a.max_target, p, y);
  const float scale = a.task == FMB200_TASK_REGRESSION ? 2.f : 1.f;  // SGDA's loss is (p - y)^2
  const float mult = scale * l.mult, hc = scale * l.curv;
  const float hrow = (a.use_w ? xx : 0.f) + fmaxf((xx - 2.f) * s2 + sq, 0.f);
  const float hjoint = a.damp ? hc * ((a.use_w0 ? 1.f : 0.f) + hrow) : hc;
  const float lr = a.lr;
  if (a.use_w0 && lane == 0) {
    const float gb = a.damp ? gamma_scale(a.w0_conc, lr * hjoint) : 1.f;
    *w0_sum += (long long)acc_quantise(-lr * gb * mult, bad);
  }
  // ---- the steps, entry by entry as the reference takes them ----
  for (uint32_t i = 0; i < size; i++) {
    const uint32_t id = __ldg(a.col + beg + i);
    const float x = __ldg(a.val + beg + i);
    bool prev, last;
    occurrences(a.col, beg, size, i, id, &prev, &last);
    const uint32_t g = __ldg(a.group + id);
    const float c = __ldg(a.feat_cnt + id) * a.conc_scale;
    const bool damped = a.damp && c > 1.f;
    if (lane == 0) a.stamp[id] = stamp;
    if (a.use_w && lane == 0) {
      const float rw = (float)ldd(a.reg_w + g);
      const uint64_t e = a.off_w + (uint64_t)id * a.ws;
      float cur = ldf(a.state + e);
      if (prev)  // the row's earlier entries of this feature stepped it first
        for (uint32_t j = 0; j < i; j++)
          if (__ldg(a.col + beg + j) == id) cur += -lr * (mult * __ldg(a.val + beg + j) + 2.f * rw * cur);
      const float step = -lr * (mult * x + 2.f * rw * cur);
      const float gm = damped ? gamma_scale(c, lr * (hjoint + 2.f * rw)) : 1.f;
      acc_add(a.acc + e, gm * step, bad);
      if (last) acc_add(a.gacc + e, mult * x, bad);
    }
#pragma unroll
    for (int j = 0; j < KF; j++) {
      const int f = lane + 32 * j;
      if (f < k) {
        const float rv = (float)ldd(a.reg_v + (uint64_t)g * k + f);
        const uint64_t e = a.off_v + (uint64_t)id * a.kp + f;
        float cur = ldf(a.state + e);
        if (prev)
          for (uint32_t jj = 0; jj < i; jj++)
            if (__ldg(a.col + beg + jj) == id) {
              const float xj = __ldg(a.val + beg + jj);
              cur += -lr * (mult * (xj * (s[j] - cur * xj)) + 2.f * rv * cur);
            }
        const float gv = mult * (x * (s[j] - cur * x));
        const float step = -lr * (gv + 2.f * rv * cur);
        const float gm = damped ? gamma_scale(c, lr * (hjoint + 2.f * rv)) : 1.f;
        acc_add(a.acc + e, gm * step, bad);
        if (last) acc_add(a.gacc + e, gv, bad);
      }
    }
  }
}

// sgd_lambda_step (:201-248) on validation row vr, in fp64: its per-group terms into `out` [G][k + 1]
template <int KF>
__device__ void lambda_row(const SgdaHwArgs& a, uint64_t vr, double* out, int lane) {
  const uint64_t beg = __ldg(a.v_row_ptr + vr);
  const uint32_t size = (uint32_t)(__ldg(a.v_row_ptr + vr + 1) - beg);
  const double y = __ldg(a.v_target + vr);
  const int k = a.k;
  const int E = k + 1;
  const double lr = a.lr;
  const float* w = a.state + a.off_w;
  const float* v = a.state + a.off_v;
  const float* gw_ = a.grad + a.off_w;
  const float* gv_ = a.grad + a.off_v;
  for (uint32_t i = lane; i < a.G * (uint32_t)E; i += 32) out[i] = 0.0;
  // predict_scaled (:171-199): one theta-step ahead with the stored gradient
  double lin = 0.0, sfd[KF], sqd[KF];
#pragma unroll
  for (int j = 0; j < KF; j++) sfd[j] = sqd[j] = 0.0;
  for (uint32_t i = 0; i < size; i++) {
    const uint32_t id = __ldg(a.v_col + beg + i);
    const double x = __ldg(a.v_val + beg + i);
    const uint32_t g = __ldg(a.group + id);
    if (a.use_w) {
      const double wv = ldf(w + (uint64_t)id * a.ws);
      lin += (wv - lr * (ldf(gw_ + (uint64_t)id * a.ws) + 2 * ldd(a.reg_w + g) * wv)) * x;
    }
#pragma unroll
    for (int j = 0; j < KF; j++) {
      const int f = lane + 32 * j;
      if (f < k) {
        const double vv = ldf(v + (uint64_t)id * a.kp + f);
        const double d = (vv - lr * (ldf(gv_ + (uint64_t)id * a.kp + f) + 2 * ldd(a.reg_v + (uint64_t)g * k + f) * vv)) * x;
        sfd[j] += d;
        sqd[j] += d * d;
      }
    }
  }
  double quad = 0.0;
#pragma unroll
  for (int j = 0; j < KF; j++) quad += sfd[j] * sfd[j] - sqd[j];
  quad = warp_sum_d(quad);
  double p = (a.use_w0 ? (double)ldf(a.state) : 0.0) + lin + 0.5 * quad;
  double gl;
  if (a.task == FMB200_TASK_REGRESSION) {
    p = fmax((double)a.min_target, fmin((double)a.max_target, p));
    gl = 2 * (p - y);
  } else {
    gl = y * ((1.0 / (1.0 + exp(-y * p))) - 1.0);
  }
  __syncwarp();
  // the per-group sums: lane f owns column f of every group, lane 0 the w column
  for (uint32_t i = 0; i < size; i++) {
    const uint32_t id = __ldg(a.v_col + beg + i);
    const double x = __ldg(a.v_val + beg + i);
    const uint32_t g = __ldg(a.group + id);
    if (a.use_w && lane == 0) out[(uint64_t)g * E + k] += x * (double)ldf(w + (uint64_t)id * a.ws);
#pragma unroll
    for (int j = 0; j < KF; j++) {
      const int f = lane + 32 * j;
      if (f < k) {
        const double vv = ldf(v + (uint64_t)id * a.kp + f);
        const double vd = vv - lr * (ldf(gv_ + (uint64_t)id * a.kp + f) + 2 * ldd(a.reg_v + (uint64_t)g * k + f) * vv);
        out[(uint64_t)g * E + f] += sfd[j] * (vv * x) - vd * x * vv * x;
      }
    }
  }
  __syncwarp();
  // reg -= lr * grad_loss * (-2 lr * sum): the term each row adds to reg
  for (uint32_t i = lane; i < a.G * (uint32_t)E; i += 32) out[i] = -(lr * gl * (-2 * lr * out[i]));
}

template <int KF>
__global__ void __launch_bounds__(kSgdaThreads) fm_sgda_hogwild_kernel(const SgdaHwArgs a) {
  const int tid = threadIdx.x, lane = tid & 31;
  const int nwarps = blockDim.x >> 5;
  const int gw = blockIdx.x * nwarps + (tid >> 5), GW = gridDim.x * nwarps;
  const uint64_t gt = (uint64_t)blockIdx.x * blockDim.x + tid, GT = (uint64_t)gridDim.x * blockDim.x;
  GridBarrier bar{a.gbar, a.gbar_base};
  const uint64_t n_win = (a.n_rows + a.W - 1) / a.W;
  const uint32_t E = a.G * (uint32_t)(a.k + 1);
  const uint64_t fk = (uint64_t)a.kp + 1;  // elements of a feature: kp factors, then w
  if (a.moments_window < 0) sgda_moments(a, gw, GW, lane);
  for (uint64_t j = 0; j < n_win; j++) {
    const uint64_t r0 = j * a.W;
    const uint64_t R = a.n_rows - r0 < a.W ? a.n_rows - r0 : a.W;
    const uint32_t stamp = a.stamp0 + (uint32_t)j;
    // ---- theta ----
    long long w0_sum = 0;
    for (uint64_t r = gw; r < R; r += GW) theta_row<KF>(a, r0 + r, stamp, lane, &w0_sum);
    if (a.use_w0 && lane == 0 && w0_sum != 0) red_add_u64(a.acc, (unsigned long long)w0_sum);
    bar.arrive(tid);
    bar.wait(tid);
    // ---- fold ----
    const bool bad = __ldcg(a.acc + a.n_floats) != 0ull;
    if (gt == 0 && (a.use_w0 || bad)) {
      a.state[0] = acc_fold(a.state[0], __ldcg(a.acc), bad);
      a.acc[0] = 0ull;
    }
    for (uint64_t t = gt; t < (uint64_t)a.n * fk; t += GT) {
      const uint32_t i = (uint32_t)(t / fk);
      const int f = (int)(t % fk);
      if (!bad && __ldcg(a.stamp + i) != stamp) continue;
      uint64_t e;
      if (f == a.kp) {
        if (!a.use_w && !bad) continue;
        e = a.off_w + (uint64_t)i * a.ws;
      } else {
        if (f >= a.k) continue;
        e = a.off_v + (uint64_t)i * a.kp + f;
      }
      a.state[e] = acc_fold(a.state[e], __ldcg(a.acc + e), bad);
      a.grad[e] = bad ? __int_as_float(0x7fffffff) : acc_value(__ldcg(a.gacc + e));
      a.acc[e] = 0ull;
      a.gacc[e] = 0ull;
    }
    bar.arrive(tid);
    bar.wait(tid);
    if ((int64_t)j == a.moments_window) sgda_moments(a, gw, GW, lane);
    if (!a.lambda) continue;
    // ---- lambda ----
    for (uint64_t r = gw; r < R; r += GW) lambda_row<KF>(a, (r0 + r) % a.v_rows, a.part + r * E, lane);
    bar.arrive(tid);
    bar.wait(tid);
    // ---- reg ----
    for (uint32_t e = gw; e < E; e += GW) {
      double s = 0.0;
      for (uint64_t r = lane; r < R; r += 32) s += ldd(a.part + r * E + e);
      s = warp_sum_d(s);
      if (lane == 0) {
        const uint32_t g = e / (a.k + 1), f = e % (a.k + 1);
        double* reg = f == (uint32_t)a.k ? a.reg_w + g : a.reg_v + (uint64_t)g * a.k + f;
        const double x = ldd(reg) + s;
        *reg = (0.0 < x) ? x : 0.0;
      }
    }
    bar.arrive(tid);
    bar.wait(tid);
  }
}

}  // namespace

uint64_t sgda_hogwild_window(const fmb200_ctx* c) {
  return c->tune_rows_per_tile > 0 ? (uint64_t)c->tune_rows_per_tile : kSgdaWindowRows;
}

cudaError_t launch_sgda_hogwild(fmb200_ctx* c, const DataSlot& tr, const DataSlot& va, int lambda_steps) {
  if (c->kp / 4 > 32) return cudaErrorInvalidValue;  // num_factor <= 128 in this mode (fmb200_sgda_begin refuses)
  const uint64_t N = tr.n_rows, V = va.n_rows;
  const uint64_t W = sgda_hogwild_window(c);
  const bool lam = lambda_steps && V > 0;
  const uint32_t E = c->sgda_groups * (uint32_t)(c->k + 1);
  cudaError_t e;
  if (lam && (e = grow(c->sgda_part, c->sgda_part_cap, std::min(W, N) * E)) != cudaSuccess) return e;
  SgdaHwArgs a;
  a.row_ptr = tr.row_ptr.get();
  a.col = tr.col.get();
  a.val = tr.val.get();
  a.target = tr.target.get();
  a.n_rows = N;
  a.v_row_ptr = va.row_ptr.get();
  a.v_col = va.col.get();
  a.v_val = va.val.get();
  a.v_target = va.target.get();
  a.v_rows = V;
  a.feat_cnt = tr.feat_cnt.get();
  a.conc_scale = N ? (float)((double)std::min(W, N) / (double)N) : 1.f;
  a.w0_conc = (float)std::min(W, N);
  a.state = c->p32.base;
  a.grad = c->sgda_grad32.get();
  a.gacc = c->sgda_gacc.get();
  a.n_floats = c->p32.n_floats;
  a.off_w = c->p32.off_w;
  a.off_v = c->p32.off_v;
  a.ws = c->p32.ws;
  a.kp = c->kp;
  a.k = c->k;
  a.n = c->n;
  a.reg_w = c->sgda_reg_w.get();
  a.reg_v = c->sgda_reg_v.get();
  a.group = c->sgda_group.get();
  a.G = c->sgda_groups;
  a.part = c->sgda_part.get();
  a.moments = c->sgda_moments.get();
  a.W = W;
  const uint64_t t_star = sgda_last_moments_step(N, V, lam);
  a.moments_window = t_star > 0 ? (int64_t)(t_star / W) : -1;
  a.use_w0 = c->k0;
  a.use_w = c->k1;
  a.task = c->hp.task;
  a.lambda = lam ? 1 : 0;
  a.damp = c->tune_damp >= 0 ? 1 : 0;
  a.lr = (float)c->hp.lr;
  a.min_target = (float)c->hp.min_target;
  a.max_target = (float)c->hp.max_target;
  const uint32_t n_win = (uint32_t)((N + W - 1) / W);
  return with_kf<4>(c->k, [&](auto kf) -> cudaError_t {
    int grid = 0;
    const cudaError_t e_ =
        launch_windows(c, fm_sgda_hogwild_kernel<decltype(kf)::value>, a, kSgdaThreads, n_win, lam ? 4 : 2, &grid);
    if (e_ != cudaSuccess) return e_;
    c->last_cfg = EpochConfig{32, 1, (int)std::min<uint64_t>(W, 0x7fffffff), grid, kSgdaThreads, 0, a.damp, 0};
    return cudaGetLastError();
  });
}

}  // namespace fmb
