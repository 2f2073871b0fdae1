// fm_sgd_window.cu -- the reproducible HOGWILD SGD epoch (fmb200_set_reproducible): windows of a constant number of
// rows, any k <= 128, rows of any length.
//
// Tiles are T consecutive training rows in file order, windows B tiles (W = T * B rows), the first at row 0, the
// last tile and window what is left; with the bias ramp the first kWindowRampTiles windows are one tile each.  T
// and B are library constants (kWindowTileRows, kWindowTiles) or the caller's, never the grid.  One cooperative
// launch walks the windows; each is two phases behind grid barriers:
//   theta  a warp per row (lanes over factors, KF = ceil(k / 32) factors a lane) scores the row from the state as
//          the window found it and takes the reference's SGD step (fm_sgd.h:38-50) for every entry, damped by
//          gamma(c_i, lr (h_joint + reg)) with c_i = count_i * min(N, flight) / N, quantised to 2^-32 and added to
//          the fixed-point accumulator (fm_hogwild_common.cuh: exact in any order).  A feature the row names twice
//          takes two steps, both from the window's state.  The first touch of a feature in the window goes to the
//          window's list (window_touch).  The row's (mult, h_joint) goes to its slot of a per-row buffer.
//   fold   a warp per tile sums the tile's (mult, h_joint) in a fixed order (lane l takes rows l, l + 32, ...; then
//          the shuffle tree) and adds the tile's damped bias step to the window's bias accumulator; the listed
//          features are folded into the fp32 state (window_fold).  The bias itself folds at the start of the next
//          window (each thread folds it into a register) and into the state at the end.
// A step that is not finite or not below the cap sets the divergence flag, and every later fold turns the whole
// state NaN (nan_state).  These pieces and the cooperative launch are fm_window.cuh's; the stamp table and the
// launch are shared with the HOGWILD SGDA epoch.  Which warp takes which row or tile only decides the order in which
// integers are added, and the fp32 arithmetic of a row depends on k and the row alone, so the epoch is the same bits
// on every run, at every grid size, CTAs per SM, threads per CTA and SM count.  It is the fp64 model of the row-lane
// windows with TR = T, grid = B, its budget widened for long rows and wide k; tests/test_sgd_window_gpu.py holds the
// kernel to it (DESIGN.md section 3.3).
//
// Exactness: at most S = min(W * max_row_nnz, nnz) steps land on one element per window (at most B on the bias),
// so a per-step cap of min(2^11, 2^31 / S) keeps every u64 sum below 2^63.
#include "fm_window.cuh"

namespace fmb {

namespace {

constexpr int kWindowMaxThreads = 256;

struct WindowArgs {
  const uint64_t* row_ptr;
  const uint32_t* col;
  const float* val;
  const float* target;
  uint64_t n_rows;
  uint32_t n_tiles, ramp_tiles, TR, B;
  const float* feat_cnt;
  float conc_scale, w0_conc;            // count -> concurrency, and the bias's, of a full window ...
  float ramp_conc_scale, ramp_w0_conc;  // ... and of a ramp window (one tile)
  float* state;                         // packed fp32 state (Params32)
  unsigned long long* acc;              // steps [n_floats], then the divergence flag
  uint64_t n_floats, off_w, off_v;
  int ws, kp, k;
  uint32_t* stamp;  // [n]: the stamp of the last window that touched the feature
  uint32_t stamp0;  // stamp of this launch's window 0
  uint32_t* list;   // [n]: the features the window touched, in no particular order
  // [0, 1] the bias steps of a window, [2, 3] the length of its list, both by window parity; zero when the
  // launch starts
  unsigned long long* aux;
  float2* rows;  // [min(W, N)]: each row's (mult, h_joint), by its position in the window
  int use_w0, use_w, task, damp;
  float lr, reg0, regw, regv, min_target, max_target, step_cap;
  unsigned int* gbar;
  uint32_t gbar_base;
  unsigned long long* prof;  // phase timers (development aid): kWindowProfSlots clock64 sums over the CTAs, or null
};

constexpr int kWindowProfSlots = 4;  // theta, barrier 1, fold, barrier 2

// window j: its first tile and its tiles (the ramp windows are one tile each)
__device__ __forceinline__ void window_tiles(const WindowArgs& a, uint32_t j, uint32_t* t0, uint32_t* nt) {
  if (j < a.ramp_tiles) {
    *t0 = j;
    *nt = 1;
  } else {
    *t0 = a.ramp_tiles + (j - a.ramp_tiles) * a.B;
    *nt = min(a.B, a.n_tiles - *t0);
  }
}

template <int KF>
__device__ void window_row(const WindowArgs& a, uint64_t r, float w0, float conc_scale, uint32_t stamp,
                           unsigned long long* cnt, int lane, float2* pair) {
  const uint64_t beg = __ldg(a.row_ptr + r);
  const uint32_t size = (uint32_t)(__ldg(a.row_ptr + r + 1) - beg);
  const float y = __ldg(a.target + r);
  const int k = a.k;
  const float* w = a.state + a.off_w;
  const float* v = a.state + a.off_v;
  unsigned long long* bad = a.acc + a.n_floats;
  // ---- the score from the window's state: lane l holds entry b + l of each chunk of 32 ----
  float s[KF], q = 0.f, lin = 0.f, xx = 0.f;
#pragma unroll
  for (int j = 0; j < KF; j++) s[j] = 0.f;
  for (uint32_t b = 0; b < size; b += 32) {
    const uint32_t m = min(32u, size - b);
    uint32_t my_id = 0;
    float my_x = 0.f;
    if ((uint32_t)lane < m) {
      my_id = __ldg(a.col + beg + b + lane);
      my_x = __ldg(a.val + beg + b + lane);
      if (a.use_w) lin += __ldcg(w + (uint64_t)my_id * a.ws) * my_x;
      xx += my_x * my_x;
    }
#pragma unroll 4
    for (uint32_t i = 0; i < m; i++) {
      const uint32_t id = __shfl_sync(0xffffffffu, my_id, i);
      const float x = __shfl_sync(0xffffffffu, my_x, i);
#pragma unroll
      for (int j = 0; j < KF; j++) {
        const int f = lane + 32 * j;
        if (f < k) {
          const float vx = __ldcg(v + (uint64_t)id * a.kp + f) * x;
          s[j] += vx;
          q += vx * vx;
        }
      }
    }
  }
  float s2 = 0.f;
#pragma unroll
  for (int j = 0; j < KF; j++) s2 += s[j] * s[j];
  s2 = warp_sum(s2);
  const float sq = warp_sum(q);
  lin = warp_sum(lin);
  xx = warp_sum(xx);
  const float p = w0 + lin + 0.5f * (s2 - sq);
  const LossStep l = loss_step(a.task, a.min_target, a.max_target, p, y);
  const float hrow = (a.use_w ? xx : 0.f) + fmaxf((xx - 2.f) * s2 + sq, 0.f);
  const float hjoint = a.damp ? l.curv * ((a.use_w0 ? 1.f : 0.f) + hrow) : l.curv;
  if (lane == 0) *pair = make_float2(l.mult, hjoint);
  const float lr = a.lr;
  const float nlr_mult = -lr * l.mult, nlr_regv = -lr * a.regv, nlr_regw = -lr * a.regw;
  const float cap = a.step_cap;
  // ---- the steps: lane l takes entry b + l's w step, damping and stamp; the warp its V row ----
  for (uint32_t b = 0; b < size; b += 32) {
    const uint32_t m = min(32u, size - b);
    uint32_t my_id = 0;
    float my_x = 0.f, my_sv = 1.f;
    if ((uint32_t)lane < m) {
      my_id = __ldg(a.col + beg + b + lane);
      my_x = __ldg(a.val + beg + b + lane);
      const float c = __ldg(a.feat_cnt + my_id) * conc_scale;
      const bool damped = a.damp && c > 1.f;
      if (damped) my_sv = gamma_scale(c, lr * (hjoint + a.regv));
      if (a.use_w) {
        const uint64_t e = a.off_w + (uint64_t)my_id * a.ws;
        const float sw = damped ? gamma_scale(c, lr * (hjoint + a.regw)) : 1.f;
        const float wv = __ldcg(a.state + e);
        red_add_u64(a.acc + e, acc_quantise(sw * (nlr_mult * my_x + nlr_regw * wv), bad, cap));
      }
    }
    window_touch(a, stamp, cnt, my_id, (uint32_t)lane < m, lane);
#pragma unroll 4
    for (uint32_t i = 0; i < m; i++) {
      const uint32_t id = __shfl_sync(0xffffffffu, my_id, i);
      const float x = __shfl_sync(0xffffffffu, my_x, i);
      const float sv = __shfl_sync(0xffffffffu, my_sv, i);
      const float x2 = x * x;
#pragma unroll
      for (int j = 0; j < KF; j++) {
        const int f = lane + 32 * j;
        if (f < k) {
          const uint64_t e = a.off_v + (uint64_t)id * a.kp + f;
          const float vv = __ldcg(a.state + e);
          red_add_u64(a.acc + e, acc_quantise(sv * (nlr_mult * (s[j] * x - vv * x2) + nlr_regv * vv), bad, cap));
        }
      }
    }
  }
}

template <int KF>
__global__ void __launch_bounds__(kWindowMaxThreads, KF == 4 ? 3 : 4) fm_sgd_window_kernel(const WindowArgs a) {
  const int tid = threadIdx.x, lane = tid & 31;
  const int nwarps = blockDim.x >> 5;
  const uint64_t gw = (uint64_t)blockIdx.x * nwarps + (tid >> 5), GW = (uint64_t)gridDim.x * nwarps;
  const uint64_t gt = (uint64_t)blockIdx.x * blockDim.x + tid, GT = (uint64_t)gridDim.x * blockDim.x;
  GridBarrier bar{a.gbar, a.gbar_base};
  unsigned long long* flag = a.acc + a.n_floats;
  unsigned long long* accb = a.aux;
  const uint32_t n_win = a.ramp_tiles + (a.n_tiles - a.ramp_tiles + a.B - 1) / a.B;
  float w0 = a.use_w0 ? __ldcg(a.state) : 0.f;
  long long t_prof = clock64();
  unsigned long long s_prof[kWindowProfSlots] = {0ull, 0ull, 0ull, 0ull};
  auto mark = [&](int slot) {  // thread 0 of each CTA: the cycles since the last mark go to `slot`
    if (a.prof && tid == 0) {
      const long long now = clock64();
      s_prof[slot] += (unsigned long long)(now - t_prof);
      t_prof = now;
    }
  };
  for (uint32_t j = 0; j < n_win; j++) {
    uint32_t t0, nt;
    window_tiles(a, j, &t0, &nt);
    const bool ramp = j < a.ramp_tiles;
    const uint64_t r0 = (uint64_t)t0 * a.TR;
    const uint64_t R = min(a.n_rows, r0 + (uint64_t)nt * a.TR) - r0;
    const uint32_t stamp = a.stamp0 + j;
    if (j > 0 && a.use_w0) w0 = acc_fold(w0, __ldcg(accb + ((j - 1) & 1)), false);  // the previous window's steps
    // ---- theta ----
    const float cs = ramp ? a.ramp_conc_scale : a.conc_scale;
    for (uint64_t r = gw; r < R; r += GW)
      window_row<KF>(a, r0 + r, w0, cs, stamp, a.aux + 2 + (j & 1), lane, a.rows + r);
    mark(0);
    bar.arrive(tid);
    bar.wait(tid);
    mark(1);
    // ---- fold: the tiles' bias steps, then the listed features ----
    const bool bad = __ldcg(flag) != 0ull;  // read once: a bias step below may raise it (the end catches that)
    if (a.use_w0) {
      const float w0c = ramp ? a.ramp_w0_conc : a.w0_conc;
      for (uint64_t t = gw; t < nt; t += GW) {
        const uint64_t rb = t * a.TR;
        const uint32_t T = (uint32_t)min((uint64_t)a.TR, R - rb);
        float M = 0.f, H = 0.f;
        for (uint32_t i = lane; i < T; i += 32) {
          const float2 pr = __ldcg(a.rows + rb + i);
          M += pr.x;
          H += pr.y;
        }
        M = warp_sum(M);
        H = warp_sum(H);
        if (lane == 0) {
          M += (float)T * a.reg0 * w0;
          const float gb = gamma_scale(fmaxf(w0c, 1.f), a.lr * (H / (float)T + a.reg0));
          red_add_u64(accb + (j & 1), acc_quantise(-a.lr * gb * M, flag, a.step_cap));
        }
      }
    }
    if (gt == 0) {  // every thread has folded the previous window's bias steps; the next list starts empty
      if (j > 0) accb[(j - 1) & 1] = 0ull;
      a.aux[2 + ((j + 1) & 1)] = 0ull;
    }
    if (bad) {  // a step overflowed: the whole state turns NaN
      nan_state(a, gt, GT);
    } else {
      window_fold(a, __ldcg(a.aux + 2 + (j & 1)), gt, GT);
    }
    mark(2);
    bar.arrive(tid);
    bar.wait(tid);
    mark(3);
  }
  if (a.prof && tid == 0)
    for (int i = 0; i < kWindowProfSlots; i++) atomicAdd(a.prof + i, s_prof[i]);
  // ---- the last window's bias; a flag its bias steps raised turns the state NaN ----
  if (__ldcg(flag) != 0ull) {
    nan_state(a, gt, GT);
  } else if (gt == 0 && a.use_w0) {
    a.state[0] = acc_fold(w0, __ldcg(accb + ((n_win - 1) & 1)), false);
  }
}

}  // namespace

cudaError_t launch_sgd_window(fmb200_ctx* c, DataSlot& d) {
  if (c->kp / 4 > 32) return cudaErrorInvalidValue;  // num_factor <= 128 in this mode
  const uint64_t N = d.n_rows;
  if (N == 0) return cudaSuccess;
  const uint32_t TR = (uint32_t)c->win_tile_rows, B = (uint32_t)c->win_tiles;
  const uint64_t W = (uint64_t)TR * B;
  const uint64_t n_tiles = (N + TR - 1) / TR;
  if (n_tiles > 0xffffffffull) return cudaErrorInvalidValue;
  const uint64_t n_floats = c->p32.n_floats;
  if (n_floats % 4 != 0 || c->p32.off_v % 4 != 0) return cudaErrorInvalidValue;  // the fold takes float4s
  cudaError_t e;
  if ((e = grow(c->win_rows, c->win_rows_cap, std::min(W, N))) != cudaSuccess) return e;
  // The bias ramp of the row-lane epoch: the first epoch after the state was set starts the bias far from its
  // equilibrium, so its first windows are one tile each
  const bool ramp = c->hogwild_fresh && c->k0 && c->tune_damp >= 0 && n_tiles > 8 * kWindowRampTiles;
  c->hogwild_fresh = false;
  const uint64_t flight = std::min(W, N);
  const double q_max = (double)d.max_feat_cnt * (double)flight / (double)N * c->hp.lr *
                       (1.0 + std::max(c->hp.regw, c->hp.regv));
  const bool damp = c->tune_damp == 1 || (c->tune_damp == 0 && q_max > 0.5);
  const double steps = (double)std::max<uint64_t>(std::min<uint64_t>(W * std::max<uint32_t>(d.max_row_nnz, 1), d.nnz), B);
  WindowArgs a;
  a.row_ptr = d.row_ptr.get();
  a.col = d.col.get();
  a.val = d.val.get();
  a.target = d.target.get();
  a.n_rows = N;
  a.n_tiles = (uint32_t)n_tiles;
  a.ramp_tiles = ramp ? (uint32_t)kWindowRampTiles : 0u;
  a.TR = TR;
  a.B = B;
  a.feat_cnt = d.feat_cnt.get();
  a.conc_scale = (float)((double)flight / (double)N);
  a.w0_conc = (float)flight;
  a.ramp_conc_scale = (float)((double)TR / (double)N);
  a.ramp_w0_conc = (float)TR;
  a.state = c->p32.base;
  a.n_floats = n_floats;
  a.off_w = c->p32.off_w;
  a.off_v = c->p32.off_v;
  a.ws = c->p32.ws;
  a.kp = c->kp;
  a.k = c->k;
  a.rows = reinterpret_cast<float2*>(c->win_rows.get());
  a.use_w0 = c->k0;
  a.use_w = c->k1;
  a.task = c->hp.task;
  a.damp = damp ? 1 : 0;
  a.lr = (float)c->hp.lr;
  a.reg0 = (float)c->hp.reg0;
  a.regw = (float)c->hp.regw;
  a.regv = (float)c->hp.regv;
  a.min_target = (float)c->hp.min_target;
  a.max_target = (float)c->hp.max_target;
  a.step_cap = (float)std::min((double)kAccStepMax, 2147483648.0 / steps);
  PhaseTimers prof;  // fmb200_set_tuning variant 132: phase timers, printed per window
  if (c->tune_variant == 132 && (e = prof.start(kWindowProfSlots, c->stream)) != cudaSuccess) return e;
  a.prof = prof.slots.get();
  const uint32_t n_win = a.ramp_tiles + (uint32_t)((n_tiles - a.ramp_tiles + B - 1) / B);
  const int threads = c->tune_threads > 0 ? std::min(c->tune_threads, kWindowMaxThreads) : kWindowMaxThreads;
  return with_kf<4>(c->k, [&](auto kf) -> cudaError_t {
    int grid = 0;
    cudaError_t e_ = launch_windows(c, fm_sgd_window_kernel<decltype(kf)::value>, a, threads, n_win, 2, &grid);
    if (e_ != cudaSuccess) return e_;
    c->last_cfg = EpochConfig{32, decltype(kf)::value, (int)TR, grid, threads, 0, damp ? 1 : 0, 0};
    if (a.prof) {
      static const char* name[kWindowProfSlots] = {"theta", "barrier1", "fold", "barrier2"};
      if ((e_ = prof.print(c->stream, name, (double)n_win * grid, 1, false,
                           "[window phases, cycles per window of CTA thread 0 (%u windows x %d CTAs)]", n_win,
                           grid)) != cudaSuccess)
        return e_;
    }
    return cudaGetLastError();
  });
}

}  // namespace fmb
