// fm_hogwild.cu -- the throughput SGD epoch (FMB200_MODE_HOGWILD), sm_90a.
//
// Replaces the row loop of fm_learn_sgd_element::learn (reference
// src/libfm/src/fm_learn_sgd_element.h:56-67 = fm_model::predict, fm_model.h:105-127,
// + loss multiplier + fm_SGD, fm_sgd.h:33-51) with ONE persistent kernel launch
// per epoch.
//
// Structure (shared with the one-lane-per-row kernel of fm_rowlane.cu, which serves
// k <= 8 with short rows; this kernel serves every other shape)
//  * persistent grid = (#SMs x CTAs/SM); CTAs claim row tiles (rows_per_tile consecutive
//    rows) from a global counter in file order (TileSched), so the rows in flight are one
//    window sliding through the file and the tail of the epoch is balanced.
//  * CSR staging: lane 0 of the last warp is the TMA producer.  Per tile it issues four
//    1-D bulk copies (cp.async.bulk global->shared, mbarrier complete_tx): row offsets,
//    targets, column ids, values; NSTAGE tiles are in flight per CTA, marked L2
//    evict_first (the CSR is streamed once per epoch).  Claims and the row offsets of the
//    next tile are fetched a tile ahead so the producer never stalls on them.
//  * compute: every warp handles U x 32/E rows at a time with the RowGroup mapping
//    (fm_rowgroup.cuh): the gathers of all U row sets are issued before any is
//    consumed (memory-level parallelism), V rows as float4 with ld.global.cg
//    (parameters are mutated by other SMs through L2, so L1 must not serve them),
//    per-factor sums by segmented warp shuffles, write-back as fire-and-forget
//    red.global.add.v4.f32 / red.global.add.f32 (Hogwild: no locks, no CAS).
//  * bias: warp 0 fetches w0 once per tile (its sector is reduced into by every CTA, so
//    loads of it queue at one L2 slice) and publishes it through shared memory + named
//    barrier 1; per-warp partial sums meet in shared memory; one damped reduction per
//    tile goes to the global w0.
//  * concurrency control.  The reference is strictly sequential; Hogwild sums the
//    steps of all examples that are in flight together.  For a parameter block
//    shared by c concurrent examples that sum has gain c*lr*h (h = curvature of
//    the loss w.r.t. the block) and diverges once it exceeds 2 -- immediately for
//    the bias w0 (every example touches it, fm_sgd.h:34-37) and for popular
//    features of skewed data.  Both are handled by the closed form of the
//    reference's own sequential recurrence under a mean-field linearisation:
//    c sequential steps contract the residual by a = 1 - lr*h each, so each of
//    the c concurrent steps is scaled by
//        gamma(c, lr*h) = (1 - a^c) / (c * (1 - a))        (== 1 for c == 1)
//    which reproduces the reference step for cold features / a single row.
//      - w0: every CTA accumulates sum(mult + reg0*w0) and the mean SECANT curvature
//        h_t = mult_t / (p_raw_t - y_t) of a tile (1 where the score is unclamped,
//        < 1 where fm_learn_sgd_element.h:60-61 clamps it; logistic: s(1-s)), with
//        c = rows in flight = min(N, grid * rows_per_tile).
//      - w_i, V_i (template flag DAMP, compiled in when the hottest feature
//        has c*lr > 0.5): c_i = max(1, count_i * W / N) from a per-feature occurrence table
//        built at upload (W = rows being processed concurrently).
//      - every block a row touches contracts the SAME residual, so all of them use
//        the row's JOINT curvature h = h_loss * (1 + sum_i x_i^2 + sum_i |d p/d V_i|^2)
//        (+ the block's own regulariser) as their contraction rate.
//
// Algorithmic HBM traffic per example (roofline numerator, BASELINE.json):
// 2*k*nnz*4 bytes (V rows read + written back).
#include <algorithm>

#include "fm_hogwild_common.cuh"
#include "fm_rowgroup.cuh"

namespace fmb {

template <int G, int S, int R, int RW, int U, bool DAMP>
__global__ void __launch_bounds__(HW_MAX_THREADS, row_class_ctas(R, U))
    fm_sgd_hogwild_kernel(const HogwildArgs a) {
  using RG = RowGroup<G, S, R, RW>;
  constexpr int E = RG::E;
  constexpr int RPW = 32 / E;  // rows per warp per row set
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem);
  float* s_acc = reinterpret_cast<float*>(smem + 64);  // [3][4]: sum grad, sum curvature

  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const int nwarp = blockDim.x >> 5;
  const int rows_per_set = nwarp * RPW;
  const int lig = lane % E;  // lane in group
  const int c = lig % G;
  const int s = lig / G;
  const int sub = lane / E;  // which of the warp's RPW rows
  const int TR = a.tile_rows;

  const uint64_t policy = ring_init(smem, tid);
  uint32_t* s_tile = reinterpret_cast<uint32_t*>(smem + 208);  // [HW_NSTAGE] tile staged per stage
  TileSched sched{a.sched, a.n_tiles, false};
  // producer duties (tile claims, TMA issue, bias reduction) sit on lane 0 of the LAST
  // warp; warp 0 fetches and publishes the bias -- nobody waits on the producer before
  // the end-of-tile barrier
  const int ptid = (int)blockDim.x - 32;
  uint32_t claim_raw = HW_NO_TILE;  // producer: a claim in flight (resolved one tile later)
  if (tid == ptid) {
    for (int i = 0; i < HW_NSTAGE; i++) {
      const uint32_t t = sched.claim();
      s_tile[i] = t;
      if (t != HW_NO_TILE) {
        const uint64_t r0 = (uint64_t)t * TR, r1 = min(r0 + (uint64_t)TR, a.n_rows);
        issue_tile(a, smem, bars, t, i, policy, __ldg(a.row_ptr + r0), __ldg(a.row_ptr + r1));
      }
    }
    claim_raw = sched.fire();
  }
  __syncthreads();

  const float4* V4 = reinterpret_cast<const float4*>(a.v);
  const bool use_w = a.use_w != 0;
  const bool use_w0 = a.use_w0 != 0;
  const float lr = a.lr;
  const float nlr_regv = -lr * a.regv;
  const float nlr_regw = -lr * a.regw;

  int it = 0;
  for (;; ++it) {
    const int stage = it % HW_NSTAGE;
    const uint32_t parity = (uint32_t)(it / HW_NSTAGE) & 1u;
    const uint64_t tile = s_tile[stage];
    if (tile == HW_NO_TILE) break;  // this CTA's claims ran dry
    // producer: fetch the entry range of the tile that will refill this stage now,
    // so the two dependent global loads overlap this tile's compute
    uint32_t nt = HW_NO_TILE;
    uint64_t nt_nb = 0, nt_ne = 0;
    if (tid == ptid) {
      nt = sched.resolve(claim_raw);  // fired a tile ago: long since returned
      claim_raw = sched.fire();       // not looked at before the next tile
      if (nt != HW_NO_TILE) {
        const uint64_t r0 = (uint64_t)nt * TR, r1 = min(r0 + (uint64_t)TR, a.n_rows);
        nt_nb = __ldg(a.row_ptr + r0);
        nt_ne = __ldg(a.row_ptr + r1);
      }
    }
    BiasFetch bias;
    bias.slot = reinterpret_cast<float*>(smem + 192);
    bias.issue(a, use_w0, tid);
    mbar_wait(bars + stage, parity);

    unsigned char* sb = stage_base(smem, a, stage);
    const uint64_t* rp = reinterpret_cast<const uint64_t*>(sb);
    const float* ys = reinterpret_cast<const float*>(sb + (size_t)(TR + 2) * 8);
    const uint32_t* ids = reinterpret_cast<const uint32_t*>(sb + (size_t)(TR + 2) * 8 + (size_t)TR * 4);
    const float* xs = reinterpret_cast<const float*>(ids + a.tile_cap);
    const uint64_t row0 = tile * (uint64_t)TR;
    const int rows_here = (int)min((uint64_t)TR, a.n_rows - row0);
    const uint64_t ab = rp[0] & ~3ull;
    if (a.global_entries) {  // rows longer than the ring can stage: entries straight from global
      ids = a.col + ab;
      xs = a.val + ab;
    }

    float msum = 0.f, hsum = 0.f;
    float w0 = 0.f;
    bool have_w0 = false;
    for (int rbase = warp * RPW; rbase < rows_here; rbase += U * rows_per_set) {
      RG g[U];
      float y[U];
      bool valid[U];
      // ---- phase 1: put the gathers of all U row sets in flight ----
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int r = rbase + u * rows_per_set + sub;
        valid[u] = r < rows_here;
        int beg = 0, end = 0;
        y[u] = 0.f;
        if (valid[u]) {
          beg = (int)(rp[r] - ab);
          end = (int)(rp[r + 1] - ab);
          y[u] = ys[r];
        }
        g[u].gather(V4, a.w, a.gp, a.ws, use_w, ids, xs, beg, end, c, s, lig);
      }
      if (!have_w0) {  // after this tile's first gathers are in flight
        w0 = bias.get(use_w0, tid, it, (int)blockDim.x);
        have_w0 = true;
      }
      // ---- phase 2: score, multiplier, write-back, one row set at a time ----
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (U > 1 && rbase + u * rows_per_set >= rows_here) break;  // warp-uniform
        RG& gu = g[u];
        const float part = gu.template reduce<DAMP>(V4, a.w, a.gp, a.ws, use_w, ids, xs, c, s, lig);
        const LossStep ls = loss_step(a, w0 + part, y[u]);
        const float mult = ls.mult, curv = ls.curv;
        // curvature of the loss along this row's whole parameter set: every block the
        // row touches contracts the SAME residual, so they share one contraction rate
        const float hjoint = DAMP ? curv * ((use_w0 ? 1.f : 0.f) + gu.hrow) : curv;
        if (valid[u] && lig == 0) {
          msum += mult;
          hsum += hjoint;
        }

        // ---- fm_SGD write-back (fm_sgd.h:38-50) as L2 reductions ----
        const float nlr_mult = -lr * mult;
        // factor rows, chunk-parallel: -lr*(mult*(sum_f*x - v*x^2) + regv*v)
        auto update_v = [&](int j, const float4& v) {
          const uint32_t id = ids[j];
          const float x = xs[j];
          const float x2 = x * x;
          float sv = 1.f;
          if (DAMP) {
            const float conc = __ldg(a.feat_cnt + id) * a.conc_scale;  // expected concurrency
            if (conc > 1.f) sv = gamma_scale(conc, lr * (hjoint + a.regv));
          }
          red_add_f4(a.v + ((size_t)id * a.gp + c) * 4,
                     sv * (nlr_mult * (gu.acc.x * x - v.x * x2) + nlr_regv * v.x),
                     sv * (nlr_mult * (gu.acc.y * x - v.y * x2) + nlr_regv * v.y),
                     sv * (nlr_mult * (gu.acc.z * x - v.z * x2) + nlr_regv * v.z),
                     sv * (nlr_mult * (gu.acc.w * x - v.w * x2) + nlr_regv * v.w));
        };
        if (c < a.gp) {
#pragma unroll
          for (int q = 0; q < R; ++q) {
            const int j = gu.beg + s + q * S;
            if (j < gu.end) update_v(j, gu.vc[q]);
          }
          for (int q = R; q < gu.maxit; ++q) {
            const int j = gu.beg + s + q * S;
            if (j < gu.end) update_v(j, ld_cg_f4(V4 + (size_t)ids[j] * a.gp + c));
          }
        }
        // linear weights, entry-parallel: -lr*(mult*x + regw*w)
        auto update_w = [&](int j, float wv) {
          const uint32_t id = ids[j];
          const float x = xs[j];
          float sw = 1.f;
          if (DAMP) {
            const float conc = __ldg(a.feat_cnt + id) * a.conc_scale;
            if (conc > 1.f) sw = gamma_scale(conc, lr * (hjoint + a.regw));
          }
          red_add_f(a.w + (size_t)id * a.ws, sw * (nlr_mult * x + nlr_regw * wv));
        };
        if (use_w) {
#pragma unroll
          for (int t = 0; t < RW; ++t) {
            const int j = gu.beg + lig + t * E;
            if (j < gu.end) update_w(j, gu.wc[t]);
          }
          for (int t = RW; t < gu.maxwit; ++t) {
            const int j = gu.beg + lig + t * E;
            if (j < gu.end) update_w(j, ld_cg_f(a.w + (size_t)ids[j] * a.ws));
          }
        }
      }
    }

    if (!have_w0) w0 = bias.get(use_w0, tid, it, (int)blockDim.x);  // warps without rows still sync
    // ---- bias: one damped reduction into the global w0 per tile ----
    float2* s_part = reinterpret_cast<float2*>(s_acc) + (it & 1) * 8;  // [2 slots][8 warps]
    if (use_w0) bias_partial(s_part, msum, hsum, tid);
    __syncthreads();  // every warp is done with this stage; partials complete
    if (tid == ptid) {
      s_tile[stage] = nt;
      if (nt != HW_NO_TILE) issue_tile(a, smem, bars, nt, stage, policy, nt_nb, nt_ne);
      if (use_w0) {
        float M = 0.f, H = 0.f;
        for (int i = 0; i < nwarp; i++) {
          M += s_part[i].x;
          H += s_part[i].y;
        }
        const float T = (float)rows_here;
        M += T * a.reg0 * w0;  // sum_t (mult_t + reg0*w0)
        const float gsc = gamma_scale(fmaxf(a.w0_conc, 1.f), lr * (H / T + a.reg0));
        red_add_f(a.w0, -lr * gsc * M);
      }
    }
  }
  if (tid == ptid) sched.finish(gridDim.x, claim_raw);
}

// ---------------------------------------------------------------------------
using KernelFn = HogwildKernelFn;

template <int G, int S, int CLS>
KernelFn pick_damp(bool damp) {
  constexpr RowClass k = row_class(CLS, G);
  return damp ? fm_sgd_hogwild_kernel<G, S, k.R, k.RW, k.U, true>
              : fm_sgd_hogwild_kernel<G, S, k.R, k.RW, k.U, false>;
}

template <int G, int S>
KernelFn pick_r(int cls, bool damp) {
  switch (cls) {
    case -1: return pick_damp<G, S, -1>(damp);
    case 0: return pick_damp<G, S, 0>(damp);
    case 1: return pick_damp<G, S, 1>(damp);
    case 2: return pick_damp<G, S, 2>(damp);
    default: return pick_damp<G, S, 3>(damp);
  }
}

void pick_geometry(int kp, uint64_t n_rows, uint64_t nnz, int* G, int* S, int* cls) {
  int gp = kp / 4;
  int g = 1;
  while (g < gp) g <<= 1;
  if (g > 32) g = 32;
  double avg = n_rows ? (double)nnz / (double)n_rows : 1.0;
  int s = 1;
  while (s < avg && s < 8) s <<= 1;
  while (g * s > 32) s >>= 1;
  if (s < 1) s = 1;
  *G = g;
  *S = s;
  // the register-cache class (row_class): slot iterations of an average row
  const int iters = (int)((avg + s - 1) / s);
  *cls = iters <= 1 ? -1 : (iters <= 2 ? 0 : (iters <= 8 ? 1 : ((iters <= 20 || g < 32) ? 2 : 3)));
}

// Hot-feature damping is compiled in when the tuning forces it, or when the hottest feature's
// expected concurrency over the rows in flight (flight_per_sm per SM) makes q = c*lr*(1+reg)
// non-negligible.
static bool want_damp(const fmb200_ctx* c, const DataSlot& d, double flight_per_sm) {
  const double flight_guess = std::min<double>((double)d.n_rows, (double)c->sm_count * flight_per_sm);
  const double q_max = (double)d.max_feat_cnt * flight_guess / (double)d.n_rows * c->hp.lr *
                       (1.0 + std::max(c->hp.regw, c->hp.regv));
  return c->tune_damp == 1 || (c->tune_damp == 0 && q_max > 0.5);
}

// Persistent grid of `fn`: the CTAs that fit on an SM (at most tune_ctas_per_sm) on every SM,
// at most one per tile.  Also sets the kernel's dynamic shared-memory limit to `smem`.
static cudaError_t fit_grid(fmb200_ctx* c, HogwildKernelFn fn, int threads, int smem, uint64_t n_tiles,
                            int* grid) {
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  int occ = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, threads, smem);
  if (e != cudaSuccess) return e;
  if (occ < 1) return cudaErrorInvalidConfiguration;
  const int per_sm = c->tune_ctas_per_sm > 0 ? std::min(c->tune_ctas_per_sm, occ) : occ;
  *grid = (int)std::min<uint64_t>(n_tiles, (uint64_t)c->sm_count * per_sm);
  return cudaSuccess;
}

static HogwildArgs make_args(fmb200_ctx* c, const DataSlot& d, uint64_t n_tiles, int TR,
                             uint32_t tile_cap, uint32_t sbytes) {
  HogwildArgs a;
  a.row_ptr = d.row_ptr.get();
  a.col = d.col.get();
  a.val = d.val.get();
  a.target = d.target.get();
  a.n_rows = d.n_rows;
  a.n_tiles = (uint32_t)n_tiles;
  a.tile_rows = TR;
  a.tile_cap = tile_cap;
  a.stage_bytes = sbytes;
  a.w0 = c->p32.w0();
  a.w = c->p32.w();
  a.v = c->p32.v();
  a.gp = c->kp / 4;
  a.ws = c->p32.ws;
  a.use_w0 = c->k0;
  a.use_w = c->k1;
  a.task = c->hp.task;
  a.lr = (float)c->hp.lr;
  a.reg0 = (float)c->hp.reg0;
  a.regw = (float)c->hp.regw;
  a.regv = (float)c->hp.regv;
  a.min_target = (float)c->hp.min_target;
  a.max_target = (float)c->hp.max_target;
  a.feat_cnt = d.feat_cnt.get();
  a.conc_scale = 1.f;
  a.w0_conc = 1.f;
  a.acc_w0 = a.acc_w = a.acc_v = a.acc_bad = a.acc = nullptr;
  a.state = nullptr;
  a.n_acc = 0;
  a.ramp_tiles = 0;
  a.ramp_conc_scale = a.ramp_w0_conc = 1.f;
  a.gbar = nullptr;
  a.gbar_base = 0;
  a.prof = nullptr;
  a.deal_pos = nullptr;
  a.bias_rows = nullptr;
  a.acc_w0x = nullptr;
  a.sched = c->d_sched.get();
  a.global_entries = 0;
  return a;
}

// The fixed-point accumulator of the reproducible epochs (the row-lane epoch here, the windowed SGD and SGDA
// epochs of fm_window.cuh): one u64 per float of the packed state, then the flag word of acc_add (set when a step
// was not finite or too large for the fixed point).  Allocated zeroed on first use; every launch leaves the steps
// zero behind it.
static unsigned long long* acc_flag(fmb200_ctx* c) { return c->d_acc.get() + c->p32.n_floats; }

cudaError_t acc_ready(fmb200_ctx* c, unsigned long long** steps, unsigned long long** flag) {
  if (!c->d_acc) {
    const uint64_t words = c->p32.n_floats + 1;
    cudaError_t e = alloc(c->d_acc, words);
    if (e == cudaSuccess) e = cudaMemsetAsync(c->d_acc.get(), 0, words * sizeof(unsigned long long), c->stream);
    if (e != cudaSuccess) {
      c->d_acc.reset();
      return e;
    }
  }
  *steps = c->d_acc.get();
  if (flag) *flag = acc_flag(c);
  return cudaSuccess;
}

cudaError_t clear_acc_flag(fmb200_ctx* c) {
  return c->d_acc ? cudaMemsetAsync(acc_flag(c), 0, sizeof(unsigned long long), c->stream) : cudaSuccess;
}

// A launch of the row-lane epoch: its kernel, the entries it stages per tile, the bytes of a stage, and its
// shared memory (a header of hdr_bytes, then the ring)
struct RowlaneShape {
  HogwildKernelFn fn = nullptr;
  uint32_t cap = 0, sbytes = 0;
  int smem = 0;
};
static RowlaneShape rowlane_shape(HogwildKernelFn fn, int TR, uint32_t cap, int hdr_bytes) {
  const uint32_t sbytes = (uint32_t)hw_stage_bytes(TR, cap);
  return RowlaneShape{fn, cap, sbytes, hdr_bytes + HW_NSTAGE * (int)sbytes};
}

// How the one-lane-per-row variant (fm_rowlane.cu, k <= 8, rows of at most 4 entries) runs a data set.
// dealable: the reproducible epoch may run the dealt schedule (fm_deal.cu), whose windows are those of the
// file-order schedule (the same grid).  It is left out where the rows of a warp decide the result (COMBINE's
// fp32 merge of same-feature steps) and for the warp-specialised variant.  Tuning variant 5 forces the
// file-order schedule (133: with phase timers), to compare the two on one build.
struct RowlanePlan {
  int threads = 0, TR = 0, launch_threads = 0, grid = 0;
  bool damp = false, combine = false, ws = false, prof = false, dealable = false;
  RowlaneShape file, dealt;  // the file-order schedule; the dealt one (when dealable)
};

static cudaError_t plan_rowlane(fmb200_ctx* c, const DataSlot& d, RowlanePlan* p, bool* ok) {
  *ok = false;
  const int gp = c->kp / 4;
  if (gp < 1 || gp > 2 || d.max_row_nnz > 4 || c->tune_variant == 1 || d.n_rows == 0) return cudaSuccess;
  int threads = c->tune_threads > 0 ? std::min(c->tune_threads, HW_MAX_THREADS) : 256;
  int tr_idx = 0;
  while ((32 << (tr_idx + 1)) <= threads) tr_idx++;
  p->threads = 32 << tr_idx;  // rows_per_tile == threads: lane t owns row t of the tile
  p->TR = p->threads;
  p->damp = want_damp(c, d, 3.0 * p->TR);
  // in-warp merging of same-feature steps pays once a warp of 32 rows is likely to hold
  // the hottest feature more than once
  p->combine = (double)d.max_feat_cnt * 32.0 / (double)d.n_rows > 0.5;
  // variant 3 = warp-specialised (producer warp + mbarrier hand-offs, no block barrier)
  p->ws = c->tune_variant == 3;
  // variant 132 / 133 = the window kernel with phase timers, printed per window (development aid)
  p->prof = c->tune_variant == 132 || c->tune_variant == 133;
  const uint32_t cap = (d.tile_span[tr_idx] + 3u) & ~3u;
  p->file = rowlane_shape(pick_rowlane_kernel(gp, (int)d.max_row_nnz, p->ws, p->damp, p->combine, p->prof, false),
                          p->TR, cap, p->ws ? HW_WS_HDR_BYTES : HW_HDR_BYTES);
  if (p->file.fn == nullptr) return cudaSuccess;
  p->launch_threads = p->ws ? p->threads + 32 : p->threads;
  const uint64_t n_tiles = (d.n_rows + p->TR - 1) / p->TR;
  cudaError_t e = fit_grid(c, p->file.fn, p->launch_threads, p->file.smem, n_tiles, &p->grid);
  if (e != cudaSuccess) return e;
  *ok = true;
  if (p->ws || p->combine || c->tune_variant == 5 || c->tune_variant == 133) return cudaSuccess;
  // a dealt tile gathers rows from all over its window: stage the longest rows' worth of entries
  p->dealt = rowlane_shape(pick_rowlane_kernel(gp, (int)d.max_row_nnz, false, p->damp, false, p->prof, true), p->TR,
                           std::max<uint32_t>(cap, (uint32_t)p->TR * d.max_row_nnz + 4u), HW_HDR_BYTES);
  int grid_dealt = 0;
  if ((e = fit_grid(c, p->dealt.fn, p->threads, p->dealt.smem, n_tiles, &grid_dealt)) != cudaSuccess) return e;
  p->dealable = grid_dealt == p->grid;
  return cudaSuccess;
}

cudaError_t prepare_rowlane_deal(fmb200_ctx* c, DataSlot& d) {
  if (c->mode != FMB200_MODE_HOGWILD || c->kp == 0) return cudaSuccess;
  RowlanePlan p;
  bool ok = false;
  cudaError_t e = plan_rowlane(c, d, &p, &ok);
  if (e != cudaSuccess || !ok || !p.dealable) return e;
  return build_rowlane_deal(c, d, p.TR, (uint32_t)p.grid);
}

static cudaError_t launch_rowlane(fmb200_ctx* c, DataSlot& d, bool* handled) {
  *handled = false;
  RowlanePlan p;
  bool ok = false;
  cudaError_t e = plan_rowlane(c, d, &p, &ok);
  if (e != cudaSuccess || !ok) return e;
  const int TR = p.TR;
  const int grid = p.grid;
  const uint64_t n_tiles = (d.n_rows + TR - 1) / TR;
  const bool ws = p.ws;
  // First epoch after the state was (re)set: the bias starts far from its equilibrium (w0 = 0 against a
  // target mean of ~3.5 on ratings) and a window of grid*TR rows would all be scored with that bias -- the
  // sequential loop corrects it within its first few hundred rows (fm_sgd.h:34-37: 1 - lr per row).  So
  // the first kRampTiles tiles run on ONE CTA (window = one tile: the bias contracts as in the sequential
  // loop), the rest on the full grid.  Costs ~40 us once; the epoch-0 RMSE gap to the oracle drops by an
  // order of magnitude (DESIGN.md section 3.3).  That epoch runs the file-order schedule.
  constexpr uint64_t kRampTiles = 4;
  const bool ramp = c->hogwild_fresh && c->k0 && c->tune_damp >= 0 && n_tiles > 8 * kRampTiles;
  c->hogwild_fresh = false;
  // A deal pays over repeated epochs on one data set; streaming a fresh data set in for every epoch and
  // dealing each cost more than it saved (DESIGN.md section 3.3).  So a data set uploaded synchronously is
  // dealt by the upload, one uploaded asynchronously from its second epoch on.
  const bool dealt = p.dealable && !ramp && (d.deal.matches(d.upload_gen, TR, (uint32_t)grid) || d.hogwild_epochs > 0);
  d.hogwild_epochs++;
  const RowlaneShape& shape = dealt ? p.dealt : p.file;
  const HogwildKernelFn fn = shape.fn;
  const int smem = shape.smem;
  const int launch_threads = p.launch_threads;
  HogwildArgs a = make_args(c, d, n_tiles, TR, shape.cap, shape.sbytes);
  a.conc_scale = (float)(std::min<double>((double)d.n_rows, (double)grid * TR) / (double)d.n_rows);
  // the warp-specialised kernel reads the bias when a stage is filled: HW_NSTAGE tiles ahead
  a.w0_conc = (float)std::min<double>((double)d.n_rows, (double)grid * TR * (ws ? HW_NSTAGE : 1));
  if (ws) {
    if (ramp) {
      HogwildArgs r = a;
      r.n_rows = kRampTiles * (uint64_t)TR;
      r.n_tiles = (uint32_t)kRampTiles;
      r.conc_scale = (float)((double)TR / (double)d.n_rows);
      r.w0_conc = (float)TR;
      fn<<<1, launch_threads, smem, c->stream>>>(r);
      c->launches++;
      const uint64_t skip = kRampTiles * (uint64_t)TR;  // a multiple of 32: TMA source alignment holds
      a.row_ptr += skip;
      a.target += skip;
      a.n_rows -= skip;
      a.n_tiles = (uint32_t)(n_tiles - kRampTiles);
    }
    fn<<<grid, launch_threads, smem, c->stream>>>(a);
    c->launches++;
  } else {
    // The epoch as a sequence of windows of grid tiles each (the rows the free-running kernel has
    // in flight), in one cooperative launch; each window reads the state the previous one left and
    // its steps are folded in after it: the same result on every run.  A ramp window is one tile.
    const uint64_t n_acc = c->p32.n_floats;
    if (n_acc % 4 != 0) return cudaErrorInvalidValue;  // the fold takes float4s (Params32: blocks of 4 floats)
    unsigned long long* acc = nullptr;
    if ((e = acc_ready(c, &acc, &a.acc_bad)) != cudaSuccess) return e;
    float* base = c->p32.base;
    a.acc_w0 = acc + (a.w0 - base);
    a.acc_w = acc + (a.w - base);
    a.acc_v = acc + (a.v - base);
    a.state = base;
    a.acc = acc;
    a.n_acc = n_acc;
    if (ramp) {
      a.ramp_tiles = (uint32_t)kRampTiles;
      a.ramp_conc_scale = (float)((double)TR / (double)d.n_rows);
      a.ramp_w0_conc = (float)TR;
    }
    if (dealt) {
      if ((e = build_rowlane_deal(c, d, TR, (uint32_t)grid)) != cudaSuccess) return e;
      a.row_ptr = d.deal.row_ptr.get();
      a.col = d.deal.col.get();
      a.val = d.deal.val.get();
      a.target = d.deal.target.get();
      a.deal_pos = d.deal.pos.get();
      // [2] bias steps (zero between launches), then a window's (mult, hjoint) pairs
      const uint64_t words = 2 + (uint64_t)grid * TR;
      if (c->deal_bias_cap < words) {
        if ((e = grow(c->d_deal_bias, c->deal_bias_cap, words)) != cudaSuccess) return e;
        if ((e = cudaMemsetAsync(c->d_deal_bias.get(), 0, 2 * sizeof(unsigned long long), c->stream)) != cudaSuccess)
          return e;
      }
      a.acc_w0x = c->d_deal_bias.get();
      a.bias_rows = reinterpret_cast<float2*>(c->d_deal_bias.get() + 2);
    }
    a.gbar = c->d_gbar.get();
    a.gbar_base = c->gbar_count;
    PhaseTimers prof;
    if (p.prof && (e = prof.start(RL_PROF_SLOTS, c->stream)) != cudaSuccess) return e;
    a.prof = prof.slots.get();
    // cooperative: the grid barriers between windows need every CTA resident; a grid that cannot be
    // fails to launch instead of hanging (grid <= occ * SMs holds by construction)
    void* args[] = {&a};
    e = cudaLaunchCooperativeKernel((const void*)fn, dim3(grid), dim3(launch_threads), args, (size_t)smem,
                                    c->stream);
    if (e != cudaSuccess) return e;
    c->launches++;
    // every CTA arrives once at each grid barrier of the launch (wraps modulo 2^32, as the counter does)
    const uint32_t n_win = rowlane_windows(a.n_tiles, a.ramp_tiles, (uint32_t)grid);
    c->gbar_count += (uint32_t)grid * rowlane_barriers(a.n_tiles, a.ramp_tiles, (uint32_t)grid, dealt);
    if (p.prof) {
      static const char* name[RL_PROF_SLOTS] = {"bias+gather", "score+issue", "bulk_wait", "barrier1", "fold",
                                                "barrier2"};
      if ((e = prof.print(c->stream, name, (double)n_win * grid, 1, false,
                          "[rowlane phases, cycles per window of CTA thread 0 (%u windows x %d CTAs)]", n_win,
                          grid)) != cudaSuccess)
        return e;
    }
  }
  c->last_cfg = EpochConfig{1, (int)std::max<uint32_t>(1, d.max_row_nnz), TR, grid, launch_threads, smem,
                            p.damp ? 1 : 0, dealt ? 1 : 0};
  *handled = true;
  return cudaGetLastError();
}

cudaError_t launch_sgd_hogwild(fmb200_ctx* c, DataSlot& d) {
  if (c->kp / 4 > 32) return cudaErrorInvalidValue;  // num_factor <= 128 in this mode
  if (d.n_rows == 0) return cudaSuccess;
  if (c->win_on) return launch_sgd_window(c, d);
  {
    bool handled = false;
    cudaError_t e = launch_rowlane(c, d, &handled);
    if (e != cudaSuccess || handled) return e;
  }
  int G, S, cls;
  pick_geometry(c->kp, d.n_rows, d.nnz, &G, &S, &cls);
  const RowClass rc = row_class(cls, G);
  const int threads = c->tune_threads > 0 ? std::min(c->tune_threads, HW_MAX_THREADS) : 256;
  const int ctas_target = row_class_ctas(rc.R, rc.U);

  // tile geometry: largest tile (<= 256 rows by default) whose worst-case
  // staged entry count keeps NSTAGE stages within the CTA's share of the SM's smem
  const int budget = (c->max_smem_optin - 1024) / ctas_target;
  int tr_idx = 3;  // 256 rows
  if (c->tune_rows_per_tile > 0) {
    tr_idx = 0;
    while (tr_idx < 4 && (32 << (tr_idx + 1)) <= c->tune_rows_per_tile) tr_idx++;
  }
  auto stage_bytes_for = [&](int idx) {
    return hw_stage_bytes(32 << idx, ((uint64_t)d.tile_span[idx] + 3u) & ~3ull);
  };
  while (tr_idx > 0 && (uint64_t)HW_HDR_BYTES + HW_NSTAGE * stage_bytes_for(tr_idx) > (uint64_t)budget) tr_idx--;
  // Not even 32 rows fit (rows of hundreds of entries: text / dense libsvm data): stage only the
  // row offsets and targets and let the lanes read ids / values from global memory.  The
  // reference trains on any row length; so does this path, at a lower rate.
  const bool global_entries =
      (uint64_t)HW_HDR_BYTES + (uint64_t)HW_NSTAGE * stage_bytes_for(tr_idx) > (uint64_t)c->max_smem_optin;
  if (global_entries) tr_idx = 1;
  const int TR = 32 << tr_idx;
  const uint32_t cap = global_entries ? 0u : (d.tile_span[tr_idx] + 3u) & ~3u;
  const uint32_t sbytes = (uint32_t)hw_stage_bytes(TR, cap);
  const int smem = HW_HDR_BYTES + HW_NSTAGE * (int)sbytes;

  const double rows_per_cta_step = (double)(threads / 32) * (32.0 / (G * S)) * rc.U;
  const bool damp = want_damp(c, d, ctas_target * rows_per_cta_step);

  const KernelFn fn = dispatch_gs(G, S, [&](auto g, auto s) { return pick_r<g, s>(cls, damp); });
  const uint64_t n_tiles = (d.n_rows + TR - 1) / TR;
  int grid = 0;
  cudaError_t e = fit_grid(c, fn, threads, smem, n_tiles, &grid);
  if (e != cudaSuccess) return e;

  HogwildArgs a = make_args(c, d, n_tiles, TR, cap, sbytes);
  a.global_entries = global_entries ? 1 : 0;
  a.conc_scale = (float)(std::min<double>((double)d.n_rows, (double)grid * rows_per_cta_step) /
                         (double)d.n_rows);
  a.w0_conc = (float)std::min<double>((double)d.n_rows, (double)grid * TR);
  fn<<<grid, threads, smem, c->stream>>>(a);
  c->launches++;
  c->last_cfg = EpochConfig{G, S, TR, grid, threads, smem, damp ? 1 : 0};
  return cudaGetLastError();
}

}  // namespace fmb
