// fm_rowlane.cu -- HOGWILD epoch kernel for SHORT ROWS and k <= 8: one lane per row.
//
// Same algorithm, staging and concurrency control as fm_sgd_hogwild_kernel
// (fm_hogwild.cu) -- this is the instruction-lean mapping for the one-hot
// "MovieLens" shape (BASELINE config C2: k=8, 2 nnz/row).  The sub-warp row-group
// kernel spends ~30 warp instructions per example there (segmented shuffles,
// per-lane address arithmetic replicated over 4 lanes per row); the measured
// bound of the shape is the SM's L1TEX/LSU rate for scattered 32-byte sectors,
// so everything else has to get out of the way.
//
// Mapping
//  * lane t of a CTA owns row t of the staged tile (rows_per_tile == blockDim.x);
//    all per-row math (fm_model::predict, reference fm_model.h:105-127; fm_SGD,
//    fm_sgd.h:33-51) happens in that lane's registers: no shuffles for sums.
//  * a factor row of k=8 floats is one 32-byte sector = two float4 (V starts on a 128-byte
//    line, Params32).  Letting every
//    lane fetch its own two halves would cost two sector requests per row and
//    instruction; instead lane PAIRS (2j, 2j+1) co-operate: instruction A fetches
//    the row of lane 2j (even lane low half, odd lane high half), instruction B the
//    row of lane 2j+1, and one 4-float __shfl_xor swaps the halves into place.
//    The warp-specialised variant's write-back mirrors it: after the swap each lane
//    owns half a sector of one row and issues red.global.add.v4.f32 into the state.
//    fm_sgd_rowlane_kernel adds its steps to a fixed-point accumulator of u64 instead:
//    each lane stages its whole quantised row in shared memory and issues one TMA bulk
//    reduction for it (acc_add_row).
//  * GP == 1 (k <= 4): a factor row is a single float4; every lane fetches its own.
#include <algorithm>

#include "fm_hogwild_common.cuh"

namespace fmb {

template <int GP>
struct FactorRow {
  float v[4 * GP];
};

// Adds the steps d[] of this lane's factor row (feature `id`, if `live`) to the fixed-point accumulator as
// ONE bulk reduction (cp.reduce.async.bulk .add.u64, SASS UBLKRED) of the quantised row staged in shared
// memory.  Scalar 64-bit reductions would take 4*GP instructions per row, each sending the L2 one 8-byte
// request per lane, and the L2 charges per request more than per byte (DESIGN.md section 3.3).  Every
// element is quantised by acc_quantise, the expression of acc_add, so the integer sums are the same.
// Each lane owns two slots of s_wb and alternates them over the row's entries; a slot is rewritten only
// once the bulk read of its previous contents is done.  The kernel waits for the writes before the
// window's grid barrier.
// q(f) gives the quantised element f.
template <int GP>
__device__ __forceinline__ unsigned long long* wb_slot(int e, int tid) {  // one array for every caller
  __shared__ __align__(128) unsigned long long s_wb[2][HW_MAX_THREADS][4 * GP];
  return s_wb[e & 1][tid];
}
template <int GP, int Z, typename Q>
__device__ __forceinline__ void acc_add_row_q(unsigned long long* acc_v, uint32_t id, bool live, int e, int tid, Q q) {
  constexpr int K = 4 * GP;
  unsigned long long* slot = wb_slot<GP>(e, tid);
  bulk_wait_read<Z == 1 ? 0 : 1>();  // Z == 1 reuses slot 0 for every row
  if (live) {
#pragma unroll
    for (int f = 0; f < K; f += 2) *reinterpret_cast<ulonglong2*>(slot + f) = make_ulonglong2(q(f), q(f + 1));
    fence_proxy_async_shared();  // the generic-proxy stores above, before the bulk read of the slot
    bulk_red_add_u64(acc_v + (size_t)id * K, slot, K * 8);
  }
  bulk_commit();
}
template <int GP, int Z>
__device__ __forceinline__ void acc_add_row(unsigned long long* acc_v, uint32_t id, bool live,
                                            const float (&d)[4 * GP], int e, int tid, unsigned long long* bad) {
  acc_add_row_q<GP, Z>(acc_v, id, live, e, tid, [&](int f) { return acc_quantise(d[f], bad); });
}

// This lane's factor row of feature gid (none: 0xffffffff, fetches nothing).  GP == 2: lane pairs fetch
// each other's halves so that one instruction covers a whole sector per row (see the file comment).
template <int GP>
__device__ __forceinline__ FactorRow<GP> gather_row(const float4* V4, uint32_t gid, int odd) {
  FactorRow<GP> r;
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if constexpr (GP == 2) {
    const uint32_t pid = __shfl_xor_sync(0xffffffffu, gid, 1);
    const uint32_t idA = odd ? pid : gid;  // row of the even lane
    const uint32_t idB = odd ? gid : pid;  // row of the odd lane
    const float4 la = idA != 0xffffffffu ? ld_cg_f4(V4 + (size_t)idA * 2 + odd) : zero4;
    const float4 lb = idB != 0xffffffffu ? ld_cg_f4(V4 + (size_t)idB * 2 + odd) : zero4;
    const float4 send = odd ? la : lb;
    float4 recv;
    recv.x = __shfl_xor_sync(0xffffffffu, send.x, 1);
    recv.y = __shfl_xor_sync(0xffffffffu, send.y, 1);
    recv.z = __shfl_xor_sync(0xffffffffu, send.z, 1);
    recv.w = __shfl_xor_sync(0xffffffffu, send.w, 1);
    const float4 lo = odd ? recv : la;
    const float4 hi = odd ? lb : recv;
    r.v[0] = lo.x; r.v[1] = lo.y; r.v[2] = lo.z; r.v[3] = lo.w;
    r.v[4] = hi.x; r.v[5] = hi.y; r.v[6] = hi.z; r.v[7] = hi.w;
  } else {
    const float4 l = gid != 0xffffffffu ? ld_cg_f4(V4 + (size_t)gid) : zero4;
    r.v[0] = l.x; r.v[1] = l.y; r.v[2] = l.z; r.v[3] = l.w;
  }
  return r;
}

// One tile, one lane per row: gather, score, multiplier, write-back.  `get_w0` is called
// once the gathers are in flight and returns the tile's bias.  Returns this lane's loss
// multiplier and joint curvature (zero for lanes without a row) for the bias step.
// ACC: the steps go to the fixed-point accumulator (a.acc_*) instead of the state.
// DEALT (with ACC, without COMBINE): rows sharing the key entry's feature merge its gather and its steps.
template <int GP, int Z, bool DAMP, bool COMBINE, bool ACC, bool DEALT, typename W0F>
__device__ __forceinline__ void rowlane_tile(const HogwildArgs& a, const uint64_t* rp,
                                             const float* ys, const uint32_t* ids,
                                             const float* xs, int rows_here, int tid, W0F get_w0,
                                             float& mult_out, float& hjoint_out) {
  constexpr int K = 4 * GP;
  const int lane = tid & 31;
  const int odd = lane & 1;
  const float4* V4 = reinterpret_cast<const float4*>(a.v);
  const bool use_w = a.use_w != 0;
  const bool use_w0 = a.use_w0 != 0;
  const float lr = a.lr;
  const uint64_t ab = rp[0] & ~3ull;
  // ---- this lane's row ----
  const bool valid = tid < rows_here;
  int beg = 0, cnt = 0;
  float y = 0.f;
  if (valid) {
    beg = (int)(rp[tid] - ab);
    cnt = (int)(rp[tid + 1] - ab) - beg;
    y = ys[tid];
  }
  uint32_t id[Z];
  float x[Z], wv[Z];
  FactorRow<GP> vr[Z];
  // ---- gather: all entries in flight at once ----
#pragma unroll
  for (int e = 0; e < Z; ++e) {
    const bool on = e < cnt;
    id[e] = on ? ids[beg + e] : 0u;
    x[e] = on ? xs[beg + e] : 0.f;
  }
  // DEALT: the row's last entry is its key entry.  The deal sorts a window's rows by its id, so the lanes of
  // a warp whose rows share the key form a run; `seg` is the run's first lane, which issues the run's summed
  // steps after the scores.  Every lane gathers the key itself, as in file order: the run's lanes load the
  // same sector, which the warp's load instruction requests from L2 once.
  const int kq = DEALT ? cnt - 1 : -1;  // the key entry (-1: none)
  uint32_t kid = 0xffffffffu;
#pragma unroll
  for (int e = 0; e < Z; ++e)
    if (e == kq) kid = id[e];
  int seg = lane;
  if (DEALT) {
    const uint32_t prev = __shfl_up_sync(0xffffffffu, kid, 1);
    const bool head = lane == 0 || kid == 0xffffffffu || prev != kid;
    seg = 31 - __clz(__ballot_sync(0xffffffffu, head) & (0xffffffffu >> (31 - lane)));
  }
#pragma unroll
  for (int e = 0; e < Z; ++e) {
    // a missing entry (ragged rows) fetches nothing: an unconditional gather of feature 0's sector would add
    // L2 loads on a line the rows that really contain feature 0 are reducing into
    const bool fetch = e < cnt;
    vr[e] = gather_row<GP>(V4, fetch ? id[e] : 0xffffffffu, odd);
    wv[e] = (use_w && fetch) ? ld_cg_f(a.w + (size_t)id[e] * a.ws) : 0.f;
  }

  // ---- fm_model::predict in registers (fm_model.h:105-127) ----
  float sum[K];
#pragma unroll
  for (int f = 0; f < K; ++f) sum[f] = 0.f;
  float sq = 0.f, lin = 0.f, xx = 0.f;
#pragma unroll
  for (int e = 0; e < Z; ++e) {
#pragma unroll
    for (int f = 0; f < K; ++f) {
      const float d = vr[e].v[f] * x[e];
      sum[f] += d;
      sq += d * d;
    }
    lin += wv[e] * x[e];
    xx += x[e] * x[e];
  }
  float s2 = 0.f;
#pragma unroll
  for (int f = 0; f < K; ++f) s2 += sum[f] * sum[f];
  const float w0 = get_w0();
  const float p = w0 + lin + 0.5f * (s2 - sq);

  const LossStep ls = loss_step(a, p, y);
  float mult = ls.mult, curv = ls.curv;
  if (!valid) {
    mult = 0.f;
    curv = 0.f;
  }
  // joint curvature of the row's whole parameter set (see fm_hogwild.cu)
  const float hrow = (use_w ? xx : 0.f) + fmaxf((xx - 2.f) * s2 + sq, 0.f);
  const float hjoint = DAMP ? curv * ((use_w0 ? 1.f : 0.f) + hrow) : curv;

  // ---- fm_SGD write-back (fm_sgd.h:38-50) ----
  struct KeyStep {
    float v[K], w;
  } kd{};  // DEALT: the key entry's steps
  auto make_kd = [](const float (&d)[K], float dw) {
    KeyStep k;
#pragma unroll
    for (int f = 0; f < K; ++f) k.v[f] = d[f];
    k.w = dw;
    return k;
  };
  const float nlr_mult = -lr * mult;
  const float nlr_regv = -lr * a.regv;
  const float nlr_regw = -lr * a.regw;
#pragma unroll
  for (int e = 0; e < Z; ++e) {
    const bool on = e < cnt;
    float sv = 1.f, sw = 1.f;
    if (DAMP) {
      const float conc = on ? __ldg(a.feat_cnt + id[e]) * a.conc_scale : 0.f;
      if (conc > 1.f) {
        sv = gamma_scale(conc, lr * (hjoint + a.regv));
        sw = gamma_scale(conc, lr * (hjoint + a.regw));
      }
    }
    const float x2 = x[e] * x[e];
    float d[K];
#pragma unroll
    for (int f = 0; f < K; ++f)
      d[f] = sv * (nlr_mult * (sum[f] * x[e] - vr[e].v[f] * x2) + nlr_regv * vr[e].v[f]);
    float dw = sw * (nlr_mult * x[e] + nlr_regw * wv[e]);
    bool on_c = on;  // this lane still owns a reduction for entry e
    if (DEALT && e == kq) {  // the key entry's steps are summed over the run below
      kd = make_kd(d, dw);
      on_c = false;
    }
    if (COMBINE) {
      // Skewed data: several rows of a warp hit the same feature.  Sum their steps
      // inside the warp (log-step segmented reduction over the lanes that share the
      // id, after "Voting and Shuffling to Optimize Atomic Operations") and let the
      // lowest lane issue ONE reduction: hot rows serialise at L2, so every merged
      // reduction is time saved for the whole chip.
      const uint32_t key = on ? id[e] : (0x80000000u | (uint32_t)lane);  // inactive: unique
      unsigned peers = __match_any_sync(0xffffffffu, key);
      if (__any_sync(0xffffffffu, __popc(peers) > 1)) {
        const int first = __ffs(peers) - 1;
        int rel = __popc(peers << (31 - lane) << 1);  // peers below this lane
        peers &= (0xfffffffeu << lane);               // peers above this lane
        while (__any_sync(0xffffffffu, peers != 0u)) {
          const int next = __ffs(peers);
          const int src = next ? next - 1 : lane;
#pragma unroll
          for (int f = 0; f < K; ++f) {
            const float t = __shfl_sync(0xffffffffu, d[f], src);
            if (next) d[f] += t;
          }
          const float tw = __shfl_sync(0xffffffffu, dw, src);
          if (next) dw += tw;
          const unsigned done = __ballot_sync(0xffffffffu, rel & 1);
          peers &= ~done;
          rel >>= 1;
        }
        on_c = on && (lane == first);
      }
    }
    if constexpr (ACC) {
      acc_add_row<GP, Z>(a.acc_v, id[e], on_c, d, e, tid, a.acc_bad);
    } else if (GP == 2) {
      // swap halves inside the lane pair so that each reduction covers a full sector
      const uint32_t pid = __shfl_xor_sync(0xffffffffu, id[e], 1);
      const bool pon = __shfl_xor_sync(0xffffffffu, (int)on_c, 1) != 0;
      const uint32_t idA = odd ? pid : id[e];
      const uint32_t idB = odd ? id[e] : pid;
      const bool onA = odd ? pon : on_c;
      const bool onB = odd ? on_c : pon;
      float4 send, keep;
      if (odd) {
        send = make_float4(d[0], d[1], d[2], d[3]);  // my low half goes to the even lane
        keep = make_float4(d[4], d[5], d[6], d[7]);
      } else {
        send = make_float4(d[4], d[5], d[6], d[7]);  // my high half goes to the odd lane
        keep = make_float4(d[0], d[1], d[2], d[3]);
      }
      float4 recv;
      recv.x = __shfl_xor_sync(0xffffffffu, send.x, 1);
      recv.y = __shfl_xor_sync(0xffffffffu, send.y, 1);
      recv.z = __shfl_xor_sync(0xffffffffu, send.z, 1);
      recv.w = __shfl_xor_sync(0xffffffffu, send.w, 1);
      // row A (even lane's): even writes its low half, odd writes the received high half
      const float4 va = odd ? recv : keep;
      // row B (odd lane's): even writes the received low half, odd writes its high half
      const float4 vb = odd ? keep : recv;
      if (onA) red_add_f4(a.v + ((size_t)idA * 2 + odd) * 4, va.x, va.y, va.z, va.w);
      if (onB) red_add_f4(a.v + ((size_t)idB * 2 + odd) * 4, vb.x, vb.y, vb.z, vb.w);
    } else if (on_c) {
      red_add_f4(a.v + (size_t)id[e] * 4, d[0], d[1], d[2], d[3]);
    }
    if (on_c && use_w) {
      if (ACC) acc_add(a.acc_w + (size_t)id[e] * a.ws, dw, a.acc_bad);
      else red_add_f(a.w + (size_t)id[e] * a.ws, dw);
    }
  }
  if constexpr (DEALT) {
    // Quantise as acc_add does, then sum the run's integers (any order gives the same sums): after the
    // segmented suffix sum, lane l holds the sum over [l, end of its run), so the run's first lane holds all
    // of it and issues one bulk reduction and one w reduction.  Slot Z of acc_add_row_q follows the Z
    // entries' alternation.
    const bool has_key = kid != 0xffffffffu;
    unsigned long long q[K + 1];
#pragma unroll
    for (int f = 0; f < K; ++f) q[f] = has_key ? acc_quantise(kd.v[f], a.acc_bad) : 0ull;
    q[K] = (has_key && use_w) ? acc_quantise(kd.w, a.acc_bad) : 0ull;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const bool take = __shfl_down_sync(0xffffffffu, seg, s) == seg && lane + s < 32;
#pragma unroll
      for (int f = 0; f <= K; ++f) {
        const unsigned long long t = __shfl_down_sync(0xffffffffu, q[f], s);
        if (take) q[f] += t;
      }
    }
    const bool issue = has_key && lane == seg;
    acc_add_row_q<GP, Z>(a.acc_v, kid, issue, Z, tid, [&](int f) { return q[f]; });
    if (issue && use_w) red_add_u64(a.acc_w + (size_t)kid * a.ws, q[K]);
  }

  mult_out = mult;
  hjoint_out = valid ? hjoint : 0.f;
}

// The whole epoch in one cooperative launch, as a sequence of windows separated by grid barriers.
// Window j covers tiles [t0_j, t0_j + nt_j): the first a.ramp_tiles windows are one tile each (the
// bias ramp, with its own concurrency a.ramp_*), every later one gridDim.x tiles (the rows the
// free-running kernel has in flight), the last one what is left.  CTA b runs tile t0_j + b of each
// window, if there is one.  A window reads the state and accumulates its steps in a.acc_*; after a
// grid barrier every CTA folds its slice of the accumulator into the state, and after a second one
// the next window starts.  So every row of a window sees the state as the previous window left it,
// whichever CTA runs it and whenever, and the epoch computes the same state on every run.
// Every CTA runs every window's barriers and fold, with or without a tile in it.
// PROF: phase timers (development aid, launch_rowlane: tuning variant 132).  Thread 0 adds the cycles of
// each phase of a window to a shared-memory slot; the sums go to a.prof once, at the end.
constexpr int RL_PROF_OFF = 200;  // RL_PROF_SLOTS u64 in the spare bytes of the HW_HDR_BYTES header

//
// DEALT: the CSR is the dealt copy (fm_deal.cu), no bias ramp.  CTA b runs chunk b of each window's rows in
// key order; the rows' steps and the state they read are those of the file-order schedule, so only the bias
// step needs care: it is formed per file-order tile from its rows' (mult, hjoint) in lane order, the
// expression and summation order of the file-order schedule.  Every row stores its pair at its file-order
// position in a.bias_rows; after barrier 1, CTA b forms the step of file-order tile b from it and reduces
// it into a.acc_w0x[j & 1]; after barrier 2 thread 0 of every CTA folds that into its running w0, with
// the fold's expression, so the bias each window reads is the state's bias of the file-order schedule.
// One thread zeroes the slot again after the next window's barrier 1, and the epoch ends with one more
// grid barrier, behind which CTA 0 writes the bias into the state.
template <int GP, int Z, bool DAMP, bool COMBINE, bool PROF, bool DEALT>
__global__ void __launch_bounds__(HW_MAX_THREADS, 3) fm_sgd_rowlane_kernel(const HogwildArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem);
  float* s_acc = reinterpret_cast<float*>(smem + 64);
  unsigned long long* s_prof = reinterpret_cast<unsigned long long*>(smem + RL_PROF_OFF);

  const int tid = threadIdx.x;
  const int TR = a.tile_rows;  // == blockDim.x
  const uint32_t G = gridDim.x;
  const uint32_t R = a.ramp_tiles;
  const uint32_t n_win = rowlane_windows(a.n_tiles, R, G);
  long long tprof = 0;
  auto prof_mark = [&](int slot) {  // the cycles since the previous mark go to `slot`
    if constexpr (PROF) {
      if (tid == 0) {
        const long long now = clock64();
        s_prof[slot] += (unsigned long long)(now - tprof);
        tprof = now;
      }
    }
  };
  if (PROF && tid < RL_PROF_SLOTS) s_prof[tid] = 0ull;  // ordered before any mark by ring_init's barrier
  // this CTA's tile of window j, or HW_NO_TILE
  auto tile_of = [&](uint32_t j) -> uint32_t {
    const uint32_t t = j < R ? (blockIdx.x == 0 ? j : HW_NO_TILE) : R + (j - R) * G + blockIdx.x;
    return t < a.n_tiles ? t : HW_NO_TILE;
  };

  const uint64_t policy = ring_init(smem, tid);
  // producer duties (TMA issue, bias reduction) sit on lane 0 of the LAST warp; warp 0
  // fetches and publishes the bias -- nobody waits on the producer before the end-of-tile
  // barrier.  The CSR is read-only, so the producer stages this CTA's tiles of the coming
  // windows HW_NSTAGE tiles ahead, across the window barriers.
  const int ptid = (int)blockDim.x - 32;
  uint32_t pj = 0;  // producer: the next window whose tile is not staged yet
  auto next_tile = [&]() -> uint32_t {
    for (; pj < n_win; ++pj)
      if (tile_of(pj) != HW_NO_TILE) return tile_of(pj++);
    return HW_NO_TILE;
  };
  if (tid == ptid) {
    for (int i = 0; i < HW_NSTAGE; i++) {
      const uint32_t t = next_tile();
      if (t != HW_NO_TILE) {
        const uint64_t r0 = (uint64_t)t * TR, r1 = min(r0 + (uint64_t)TR, a.n_rows);
        issue_tile(a, smem, bars, t, i, policy, __ldg(a.row_ptr + r0), __ldg(a.row_ptr + r1));
      }
    }
  }
  __syncthreads();

  const bool use_w0 = a.use_w0 != 0;
  const float lr = a.lr;
  GridBarrier gbar{a.gbar, a.gbar_base};
  // This thread's slice of the fold: the four elements [4q, 4q+4) for every q ≡ q0 (mod fold_stride) below
  // n_acc / 4 (the launcher checks that n_acc is a multiple of 4; the flag word acc[n_acc] lies behind).
  const uint64_t q0 = blockIdx.x * (uint64_t)blockDim.x + tid;
  const uint64_t fold_stride = (uint64_t)G * blockDim.x;
  const uint64_t n_vec = a.n_acc / 4;
  float4* state4 = reinterpret_cast<float4*>(a.state);
  ulonglong2* acc2 = reinterpret_cast<ulonglong2*>(a.acc);  // two u64 steps per 16-byte access
  if (PROF && tid == 0) tprof = clock64();

  // DEALT, thread 0: the bias of the current window, and the previous window's bias step
  float w0_run = (DEALT && use_w0 && tid == 0) ? ld_cg_f(a.w0) : 0.f;
  bool bad = false;  // the accumulator's overflow flag as the latest fold saw it
  int it = 0;  // tiles this CTA has run
  for (uint32_t j = 0; j < n_win; ++j) {
    const uint32_t tile = tile_of(j);
    if (DEALT && use_w0 && tid == 0 && j > 0) w0_run = acc_fold(w0_run, __ldcg(a.acc_w0x + ((j - 1) & 1)), bad);
    if (tile != HW_NO_TILE) {
      const int stage = it % HW_NSTAGE;
      const uint32_t parity = (uint32_t)(it / HW_NSTAGE) & 1u;
      // producer: fetch the entry range of the tile that will refill this stage now,
      // so the two dependent global loads overlap this tile's compute
      uint32_t nt = HW_NO_TILE;
      uint64_t nt_nb = 0, nt_ne = 0;
      if (tid == ptid) {
        nt = next_tile();
        if (nt != HW_NO_TILE) {
          const uint64_t r0 = (uint64_t)nt * TR, r1 = min(r0 + (uint64_t)TR, a.n_rows);
          nt_nb = __ldg(a.row_ptr + r0);
          nt_ne = __ldg(a.row_ptr + r1);
        }
      }
      HogwildArgs w = a;  // the window's concurrency
      if (j < R) {
        w.conc_scale = a.ramp_conc_scale;
        w.w0_conc = a.ramp_w0_conc;
      }
      BiasFetch bias;
      bias.slot = reinterpret_cast<float*>(smem + 192);
      if (DEALT) bias.pending = w0_run;
      else bias.issue(a, use_w0, tid);
      // DEALT: this lane's row's position in file order, for its bias pair
      const uint32_t pos = DEALT && tid < (int)min((uint64_t)TR, a.n_rows - (uint64_t)tile * TR)
                               ? __ldg(a.deal_pos + (uint64_t)tile * TR + tid)
                               : 0xffffffffu;
      mbar_wait(bars + stage, parity);

      unsigned char* sb = stage_base(smem, a, stage);
      const uint64_t* rp = reinterpret_cast<const uint64_t*>(sb);
      const float* ys = reinterpret_cast<const float*>(sb + (size_t)(TR + 2) * 8);
      const uint32_t* ids = reinterpret_cast<const uint32_t*>(sb + (size_t)(TR + 2) * 8 + (size_t)TR * 4);
      const float* xs = reinterpret_cast<const float*>(ids + a.tile_cap);
      const uint64_t row0 = (uint64_t)tile * TR;
      const int rows_here = (int)min((uint64_t)TR, a.n_rows - row0);

      float mult, hj, w0 = 0.f;
      rowlane_tile<GP, Z, DAMP, COMBINE, true, DEALT>(
          w, rp, ys, ids, xs, rows_here, tid,
          [&]() {
            w0 = bias.get(use_w0, tid, it, (int)blockDim.x);
            prof_mark(0);  // bias fetch and gathers: the scores need both
            return w0;
          },
          mult, hj);
      // ---- bias: one damped reduction into the global w0 per tile ----
      float2* s_part = reinterpret_cast<float2*>(s_acc) + (it & 1) * 8;  // [2 slots][8 warps]
      if (DEALT) {
        if (use_w0 && pos != 0xffffffffu) a.bias_rows[pos] = make_float2(mult, hj);
      } else if (use_w0) {
        bias_partial(s_part, mult, hj, tid);
      }
      __syncthreads();
      if (tid == ptid) {
        if (nt != HW_NO_TILE) issue_tile(a, smem, bars, nt, stage, policy, nt_nb, nt_ne);
        if (!DEALT && use_w0) {
          float M = 0.f, H = 0.f;
          for (int i = 0; i < (int)(blockDim.x >> 5); i++) {
            M += s_part[i].x;
            H += s_part[i].y;
          }
          const float T = (float)rows_here;
          M += T * a.reg0 * w0;
          const float gsc = gamma_scale(fmaxf(w.w0_conc, 1.f), lr * (H / T + a.reg0));
          acc_add(a.acc_w0, -lr * gsc * M, a.acc_bad);
        }
      }
      ++it;
    }
    prof_mark(1);  // scores, quantisation, reductions issued, bias partials
    // every step of the window is in the accumulator: the bulk reductions' writes are complete and,
    // through the proxy fence, ordered before the barrier's release like the generic reductions
    bulk_wait_all();
    fence_proxy_async_global();
    gbar.arrive(tid);
    prof_mark(2);
    // Only the fold writes the state, and this slice only this thread's fold: its first state vector can be
    // read while the other CTAs arrive.  acc and state through L2 (ld.global.cg): an L1 line from an
    // earlier window would be stale.
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 < n_vec) s = __ldcg(state4 + q0);
    gbar.wait(tid);
    prof_mark(3);
    // DEALT: the pair of row tid of this CTA's file-order tile (zero without a row, as in the tile)
    float2 pr = make_float2(0.f, 0.f);
    if (DEALT && use_w0 && tile != HW_NO_TILE && tid < (int)min((uint64_t)TR, a.n_rows - (uint64_t)tile * TR))
      pr = __ldcg(a.bias_rows + blockIdx.x * TR + tid);
    // ---- fold: state[i] += acc[i] (fixed point), acc[i] = 0; all NaN once a step overflowed ----
    bad = __ldcg(a.acc + a.n_acc) != 0ull;
    for (uint64_t q = q0; q < n_vec; q += fold_stride) {
      const ulonglong2 lo = __ldcg(acc2 + 2 * q), hi = __ldcg(acc2 + 2 * q + 1);
      if (q != q0) s = __ldcg(state4 + q);
      s.x = acc_fold(s.x, lo.x, bad);
      s.y = acc_fold(s.y, lo.y, bad);
      s.z = acc_fold(s.z, hi.x, bad);
      s.w = acc_fold(s.w, hi.y, bad);
      // elements without a step keep their value, so a whole-vector store rewrites them unchanged; likewise
      // a pair of accumulator words is cleared whole when either holds a step
      if (bad || (lo.x | lo.y | hi.x | hi.y) != 0ull) state4[q] = s;
      if ((lo.x | lo.y) != 0ull) acc2[2 * q] = make_ulonglong2(0ull, 0ull);
      if ((hi.x | hi.y) != 0ull) acc2[2 * q + 1] = make_ulonglong2(0ull, 0ull);
    }
    if (DEALT && use_w0) {
      // the bias step of file-order tile b of this window, formed as the file-order schedule forms it
      if (tile != HW_NO_TILE) {
        float2* s_part = reinterpret_cast<float2*>(s_acc);
        bias_partial(s_part, pr.x, pr.y, tid);
        __syncthreads();
        if (tid == 0) {
          float M = 0.f, H = 0.f;
          for (int i = 0; i < (int)(blockDim.x >> 5); i++) {
            M += s_part[i].x;
            H += s_part[i].y;
          }
          const float T = (float)min((uint64_t)TR, a.n_rows - (uint64_t)tile * TR);
          M += T * a.reg0 * w0_run;
          const float gsc = gamma_scale(fmaxf(a.w0_conc, 1.f), lr * (H / T + a.reg0));
          acc_add(a.acc_w0x + (j & 1), -lr * gsc * M, a.acc_bad);
        }
      }
      // every CTA has folded the previous window's step (before barrier 1): its slot is free again
      if (blockIdx.x == 0 && tid == 0 && j > 0) a.acc_w0x[(j - 1) & 1] = 0ull;
    }
    prof_mark(4);
    if (DEALT || j + 1 < n_win) {  // the next window reads the folded state into a zero accumulator
      gbar.arrive(tid);
      gbar.wait(tid);
    }
    fence_proxy_async_global();  // ... and its bulk reductions add to the fold's zeros
    prof_mark(5);
  }
  if (DEALT) {
    // behind the last barrier: a step that overflowed after the last fold read the flag (the bias step of the
    // last window) turns the state into NaN as the fold would have; CTA 0 writes the bias and frees its slot
    const bool bad_end = __ldcg(a.acc + a.n_acc) != 0ull;
    if (bad_end && !bad)
      for (uint64_t q = q0; q < n_vec; q += fold_stride) state4[q] = make_float4(NAN, NAN, NAN, NAN);
    if (use_w0 && blockIdx.x == 0 && tid == 0) {
      *a.w0 = acc_fold(w0_run, __ldcg(a.acc_w0x + ((n_win - 1) & 1)), bad_end);
      a.acc_w0x[(n_win - 1) & 1] = 0ull;
    }
  }
  if constexpr (PROF) {
    __syncthreads();
    if (tid < RL_PROF_SLOTS) atomicAdd(a.prof + tid, s_prof[tid]);
  }
}

// ---------------------------------------------------------------------------
// Warp-specialised variant: the CTA has one extra PRODUCER warp (tile claims, TMA issue,
// bias fetch and bias reduction) and the consumer warps never meet in a block barrier:
//   full[s]  : producer -> consumers, mbarrier (1 arrival + TMA transaction bytes);
//              the tile id and the bias for the tile ride along in shared memory
//   empty[s] : consumers -> producer, mbarrier (one arrival per consumer warp, issued
//              after the warp has stored its partial bias sums for the tile)
// A warp that finishes its 32 rows early starts the next staged tile at once; the
// per-tile __syncthreads of the kernel above (top stall in its ncu capture) is gone.
// The bias is read when a stage is FILLED, i.e. HW_NSTAGE tiles ahead of its use; the
// launcher widens the bias' concurrency window accordingly.  Shared-memory header: HW_WS_HDR_BYTES.

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

template <int GP, int Z, bool DAMP, bool COMBINE>
__global__ void __launch_bounds__(HW_MAX_THREADS + 32, 3) fm_sgd_rowlane_ws_kernel(const HogwildArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty = reinterpret_cast<uint64_t*>(smem + 64);
  uint32_t* s_tile = reinterpret_cast<uint32_t*>(smem + 128);
  float* s_w0 = reinterpret_cast<float*>(smem + 160);
  float2* s_part = reinterpret_cast<float2*>(smem + 192);

  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int TR = a.tile_rows;       // == number of consumer threads
  const int n_cwarps = TR >> 5;
  const bool use_w0 = a.use_w0 != 0;
  auto stage_ptr = [&](int stage) { return smem + HW_WS_HDR_BYTES + (size_t)stage * a.stage_bytes; };

  if (tid == 0) {
    for (int i = 0; i < HW_NSTAGE; i++) {
      mbar_init(full + i, 1);
      mbar_init(empty + i, (uint32_t)n_cwarps);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (tid >= TR) {
    // ===================== producer warp (one lane) =====================
    if (lane != 0) return;
    TileSched sched{a.sched, a.n_tiles, false};
    const uint64_t policy = policy_evict_first();
    auto fill = [&](int stage, uint32_t t) {
      s_tile[stage] = t;
      if (t == HW_NO_TILE) {
        mbar_arrive(full + stage);  // wakes the consumers; they see NO_TILE and leave
        return;
      }
      s_w0[stage] = use_w0 ? ld_cg_f(a.w0) : 0.f;
      const uint64_t r0 = (uint64_t)t * TR, r1 = min(r0 + (uint64_t)TR, a.n_rows);
      // the arrival on full[stage] releases the tile id and the bias
      issue_tile(a, smem, full, t, stage, policy, __ldg(a.row_ptr + r0), __ldg(a.row_ptr + r1), HW_WS_HDR_BYTES);
    };
    for (int i = 0; i < HW_NSTAGE; i++) fill(i, sched.claim());
    for (int it = 0;; ++it) {
      const int stage = it % HW_NSTAGE;
      const uint32_t t = s_tile[stage];
      if (t == HW_NO_TILE) break;  // the consumers left at this stage without arriving
      mbar_wait(empty + stage, (uint32_t)(it / HW_NSTAGE) & 1u);
      if (use_w0) {
        float M = 0.f, H = 0.f;
        for (int i = 0; i < n_cwarps; i++) {
          const float2 p = s_part[stage * 8 + i];
          M += p.x;
          H += p.y;
        }
        const uint64_t row0 = (uint64_t)t * TR;
        const float T = (float)min((uint64_t)TR, a.n_rows - row0);
        M += T * a.reg0 * s_w0[stage];
        const float gsc = gamma_scale(fmaxf(a.w0_conc, 1.f), a.lr * (H / T + a.reg0));
        red_add_f(a.w0, -a.lr * gsc * M);
      }
      fill(stage, sched.claim());
    }
    sched.finish(gridDim.x, 0u);
    return;
  }

  // ========================= consumer warps =========================
  for (int it = 0;; ++it) {
    const int stage = it % HW_NSTAGE;
    mbar_wait(full + stage, (uint32_t)(it / HW_NSTAGE) & 1u);
    const uint32_t tile = s_tile[stage];
    if (tile == HW_NO_TILE) break;
    unsigned char* sb = stage_ptr(stage);
    const uint64_t* rp = reinterpret_cast<const uint64_t*>(sb);
    const float* ys = reinterpret_cast<const float*>(sb + (size_t)(TR + 2) * 8);
    const uint32_t* ids = reinterpret_cast<const uint32_t*>(sb + (size_t)(TR + 2) * 8 + (size_t)TR * 4);
    const float* xs = reinterpret_cast<const float*>(ids + a.tile_cap);
    const uint64_t row0 = (uint64_t)tile * TR;
    const int rows_here = (int)min((uint64_t)TR, a.n_rows - row0);
    const float w0 = s_w0[stage];
    float mult, hj;
    rowlane_tile<GP, Z, DAMP, COMBINE, false, false>(a, rp, ys, ids, xs, rows_here, tid, [&]() { return w0; }, mult,
                                                     hj);
    if (use_w0) bias_partial(s_part + stage * 8, mult, hj, tid);
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + stage);  // release: partials + "done reading the stage"
  }
}

// f(std::integral_constant<decltype(V), V>{}) for the V of Vs equal to v; nullptr if there is none
template <auto... Vs, class T, class F>
static HogwildKernelFn dispatch(T v, F f) {
  HogwildKernelFn fn = nullptr;
  (void)((v == Vs && (fn = f(std::integral_constant<decltype(Vs), Vs>{}), true)) || ...);
  return fn;
}

HogwildKernelFn pick_rowlane_kernel(int gp, int max_row_nnz, bool ws, bool damp, bool combine, bool prof, bool dealt) {
  const int z = max_row_nnz <= 1 ? 1 : (max_row_nnz <= 2 ? 2 : (max_row_nnz <= 4 ? 4 : 0));
  return dispatch<1, 2>(gp, [&](auto GP) {
    return dispatch<1, 2, 4>(z, [&](auto Z) {
      return dispatch<false, true>(damp, [&](auto D) {
        return dispatch<false, true>(combine, [&](auto C) {
          if (ws) return fm_sgd_rowlane_ws_kernel<GP, Z, D, C>;
          return dispatch<false, true>(prof, [&](auto P) {
            return dispatch<false, true>(dealt, [&](auto DL) -> HogwildKernelFn {
              // the dealt schedule never merges in fp32 (COMBINE): that merge depends on which rows share a warp
              if constexpr (DL && C) return nullptr;
              else return fm_sgd_rowlane_kernel<GP, Z, D, C, P, DL>;
            });
          });
        });
      });
    });
  });
}

}  // namespace fmb
