// fm_hogwild_common.cuh -- the tile protocol shared by the three HOGWILD epoch kernels
// (fm_hogwild.cu: sub-warp row groups, any k / row length; fm_rowlane.cu: one lane per row
// for short rows with k <= 8, block-synchronous and warp-specialised): launch arguments,
// the staging ring's stage layout, set-up and TMA producer, the loss multiplier, the
// per-warp bias partials and the mean-field step scale.  See fm_hogwild.cu for the design
// notes.
#pragma once
#include "fm_device.cuh"
#include "fmb200_internal.h"

namespace fmb {

constexpr int HW_NSTAGE = 3;
constexpr int HW_MAX_THREADS = 256;
constexpr uint32_t HW_NO_TILE = 0xffffffffu;
constexpr int HW_HDR_BYTES = 256;  // mbarriers [0,64) + per-warp bias partials [64,192): [2 slots][8 warps] float2
// header of the warp-specialised kernel: full[3] @0, empty[3] @64, tile[3] @128, w0[3] @160,
// per-warp bias partials @192: [3 stages][8 warps] float2
constexpr int HW_WS_HDR_BYTES = 512;

// One stage of the ring: [row offsets (TR+2)·u64 | targets TR·f32 | ids cap·u32 | values cap·f32],
// padded to 16 bytes.  TR is a multiple of 32 and cap of 4, so every part starts 16-byte aligned as
// the bulk copies need.  cap == 0 stages only the row offsets and targets.
// T is the width of the arithmetic: uint32_t for the bulk-copy byte counts, uint64_t for the launchers.
template <typename T>
__host__ __device__ inline T hw_rp_bytes(int TR) { return (T)(TR + 2) * 8; }
template <typename T>
__host__ __device__ inline T hw_y_bytes(int TR) { return (T)TR * 4; }
// 64-bit: the launcher sizes the stage of a tile of very long rows, whose cap exceeds 32 bits
__host__ __device__ inline uint64_t hw_stage_bytes(int TR, uint64_t cap) {
  return (hw_rp_bytes<uint64_t>(TR) + hw_y_bytes<uint64_t>(TR) + 2 * cap * 4 + 15) & ~15ull;
}

struct HogwildArgs {
  const uint64_t* row_ptr;
  const uint32_t* col;
  const float* val;
  const float* target;
  uint64_t n_rows;
  uint32_t n_tiles;
  int tile_rows;       // TR (multiple of 32)
  uint32_t tile_cap;   // max staged entries per tile (multiple of 4)
  uint32_t stage_bytes;
  float* w0;
  float* w;
  float* v;
  int gp;  // float4 chunks per V row (kp / 4)
  int ws;  // stride of w in floats
  int use_w0, use_w, task;
  float lr, reg0, regw, regv, min_target, max_target;
  const float* feat_cnt;  // occurrences of each feature in this data set (DAMP)
  float conc_scale;       // rows processed concurrently / n_rows: count -> concurrency
  float w0_conc;          // rows in flight w.r.t. the bias (tile granularity)
  unsigned int* sched;    // [0] next unclaimed tile, [1] CTAs that ran dry (both 0 between launches)
  int global_entries;     // rows too long for the staging ring: ids / values are read from global
                          // memory, only row offsets and targets are staged (tile_cap == 0)
  // fm_sgd_rowlane_kernel: the steps of a window accumulate here as fixed point (acc_add), element i
  // beside element i of the packed state, and are folded into the state after the window
  unsigned long long *acc_w0, *acc_w, *acc_v;
  unsigned long long* acc_bad;  // set when a step was not finite or too large for the fixed point
  float* state;                 // the packed state [n_acc] ...
  unsigned long long* acc;      // ... and its accumulator [n_acc + 1]; acc[n_acc] is acc_bad
  uint64_t n_acc;
  // fm_sgd_rowlane_kernel: the first ramp_tiles windows are one tile each, with these concurrencies
  uint32_t ramp_tiles;
  float ramp_conc_scale, ramp_w0_conc;
  // fm_sgd_rowlane_kernel: the grid barriers' arrival counter and its value when the launch starts (GridBarrier)
  unsigned int* gbar;
  uint32_t gbar_base;
  unsigned long long* prof;  // phase timers (development aid): RL_PROF_SLOTS clock64 sums over the CTAs, or null
  // fm_sgd_rowlane_kernel<DEALT>: the CSR arrays above hold the dealt copy (fm_deal.cu); deal_pos[i] is
  // dealt row i's position inside its window in file order, bias_rows [gridDim.x * tile_rows] takes every
  // row's (mult, hjoint) at that position, and acc_w0x [2] the bias step of a window, by window parity
  const uint32_t* deal_pos;
  float2* bias_rows;
  unsigned long long* acc_w0x;
};

// Windows of the row-lane epoch over n_tiles tiles: `ramp` windows of one tile, then windows of G tiles
// (the grid), the last one what is left
__host__ __device__ inline uint32_t rowlane_windows(uint32_t n_tiles, uint32_t ramp, uint32_t G) {
  return ramp + (n_tiles - ramp + G - 1) / G;
}
// The row-lane epoch separates its windows by 2 * windows - 1 grid barriers (none behind the last fold);
// the dealt schedule also publishes the last window's bias step by one
__host__ __device__ inline uint32_t rowlane_barriers(uint32_t n_tiles, uint32_t ramp, uint32_t G, bool dealt) {
  return 2u * rowlane_windows(n_tiles, ramp, G) - (dealt ? 0u : 1u);
}

// Split-phase grid barrier of a cooperative launch (every CTA resident).  Each CTA adds 1 to a counter
// with release semantics when it arrives, and its thread 0 polls the counter with acquire loads until
// all gridDim.x CTAs have arrived; bar.sync on both sides extends both orderings to the whole CTA.
// The counter only grows: barrier k of a launch is complete at base + (k+1)·gridDim.x, compared modulo
// 2^32, so it is never reset and the host passes each launch the value its predecessors left.
// Work placed between arrive() and wait() overlaps the other CTAs' arrival.
struct GridBarrier {
  unsigned int* count;
  uint32_t target;  // the counter's value once the latest barrier arrived at is complete
  __device__ __forceinline__ void arrive(int tid) {
    __syncthreads();
    if (tid == 0) red_release_add_u32(count, 1u);
    target += gridDim.x;
  }
  __device__ __forceinline__ void wait(int tid) {
    if (tid == 0)
      while ((int32_t)(ld_acquire_u32(count) - target) < 0) {
      }
    __syncthreads();
  }
};

// Fixed point of the accumulated steps: integer sums do not depend on the order in which the
// reductions arrive, so an epoch built from such windows computes the same state on every run.
// Resolution 2^-32; the int64 range holds sums up to 2^31.  A step that is not finite or not below
// kAccStepMax (a diverging run) is not added but raises *bad, and the fold then turns the whole state
// into NaN, as the free-running fp32 reductions would have spread it: with at most 2^20 rows per
// window the sums stay below 2^31.
constexpr float kAccScale = 0x1p32f;
constexpr float kAccStepMax = 0x1p11f;

__device__ __forceinline__ void acc_add(unsigned long long* p, float d, unsigned long long* bad) {
  if (fabsf(d) < kAccStepMax) red_add_u64(p, (unsigned long long)__float2ll_rn(d * kAccScale));
  else atomicOr(bad, 1ull);  // also NaN: the comparison is false
}
// the value acc_add adds, for a caller that adds it in bulk: a step it would not add is 0.  A caller whose
// windows add more steps to one element may pass a smaller cap.
__device__ __forceinline__ unsigned long long acc_quantise(float d, unsigned long long* bad, float cap = kAccStepMax) {
  if (fabsf(d) < cap) return (unsigned long long)__float2ll_rn(d * kAccScale);
  atomicOr(bad, 1ull);  // also NaN: the comparison is false
  return 0ull;
}

// the fold of one accumulated element into the state: NaN once a step overflowed
__device__ __forceinline__ float acc_fold(float x, unsigned long long u, bool bad) {
  if (bad) return __int_as_float(0x7fffffff);
  return u != 0ull ? x + (float)((double)(long long)u * (1.0 / (double)kAccScale)) : x;
}

// stage `stage` of the ring, which follows a shared-memory header of `hdr` bytes
__device__ __forceinline__ unsigned char* stage_base(unsigned char* smem, const HogwildArgs& a,
                                                     int stage, int hdr = HW_HDR_BYTES) {
  return smem + hdr + (size_t)stage * a.stage_bytes;
}

// TMA producer: stage one tile whose entry range [nb, ne) is already known into stage `stage` of
// the ring behind a header of `hdr` bytes, completing on bars[stage].  The barrier's arrival
// releases the producer's earlier shared stores.
__device__ __forceinline__ void issue_tile(const HogwildArgs& a, unsigned char* smem, uint64_t* bars,
                                           uint32_t tile, int stage, uint64_t policy, uint64_t nb,
                                           uint64_t ne, int hdr = HW_HDR_BYTES) {
  const int TR = a.tile_rows;
  const uint64_t r0 = (uint64_t)tile * TR;
  const uint64_t ab = nb & ~3ull;
  const uint64_t ae = (ne + 3ull) & ~3ull;
  const uint32_t ebytes = a.global_entries ? 0u : (uint32_t)(ae - ab) * 4u;
  const uint32_t rp_bytes = hw_rp_bytes<uint32_t>(TR);
  const uint32_t y_bytes = hw_y_bytes<uint32_t>(TR);
  unsigned char* sb = stage_base(smem, a, stage, hdr);
  uint64_t* bar = bars + stage;
  mbar_arrive_expect_tx(bar, rp_bytes + y_bytes + 2u * ebytes);
  bulk_g2s_hint(sb, a.row_ptr + r0, rp_bytes, bar, policy);
  bulk_g2s_hint(sb + rp_bytes, a.target + r0, y_bytes, bar, policy);
  if (ebytes) {
    unsigned char* cb = sb + rp_bytes + y_bytes;
    bulk_g2s_hint(cb, a.col + ab, ebytes, bar, policy);
    bulk_g2s_hint(cb + (size_t)a.tile_cap * 4u, a.val + ab, ebytes, bar, policy);
  }
}

// Set-up of the block-synchronous kernels (one mbarrier per stage, HW_HDR_BYTES header): thread 0
// initialises the barriers and the producer, lane 0 of the last warp, takes the evict-first
// policy, which this returns.
__device__ __forceinline__ uint64_t ring_init(unsigned char* smem, int tid) {
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem);
  uint64_t policy = 0;
  if (tid == 0) {
    for (int i = 0; i < HW_NSTAGE; i++) mbar_init(bars + i, 1);
    fence_mbar_init();
  }
  if (tid == (int)blockDim.x - 32) policy = policy_evict_first();
  __syncthreads();
  return policy;
}

// fm_learn_sgd_element.h:58-65: the loss multiplier of score p against target y, and the secant
// curvature of the loss w.r.t. the raw score (1 where the clamp is inactive; logistic: s(1-s))
struct LossStep {
  float mult, curv;
};
__device__ __forceinline__ LossStep loss_step(int task, float min_target, float max_target, float p, float y) {
  LossStep l;
  if (task == FMB200_TASK_REGRESSION) {
    const float pc = fmaxf(min_target, fminf(max_target, p));
    l.mult = pc - y;
    const float den = p - y;
    l.curv = (pc == p) ? 1.f : (fabsf(den) > 1e-12f ? fminf(fmaxf(l.mult / den, 0.f), 1.f) : 0.f);
  } else {  // y in {-1,+1}
    const float sg = 1.f / (1.f + __expf(-y * p));
    l.mult = -y * (1.f - sg);
    l.curv = sg * (1.f - sg);
  }
  return l;
}
__device__ __forceinline__ LossStep loss_step(const HogwildArgs& a, float p, float y) {
  return loss_step(a.task, a.min_target, a.max_target, p, y);
}

// gamma(c, u) = (1 - (1-u)^c) / (c*u): scale of each of c concurrent steps whose
// sequential execution would contract the residual by (1-u) per step
__device__ __forceinline__ float gamma_scale(float c, float u) {
  if (c <= 1.f || u <= 0.f) return 1.f;
  const float q = c * u;
  if (q < 1e-3f) return 1.f;
  const float a = fmaxf(1.f - u, 0.f);
  const float ac = a > 0.f ? __expf(c * __logf(a)) : 0.f;
  return fminf(1.f, (1.f - ac) / q);
}

// the bias partials of a warp: lane 0 stores the warp's sums of (mult, hjoint) at part[warp]
__device__ __forceinline__ void bias_partial(float2* part, float mult, float hjoint, int tid) {
  mult = warp_sum(mult);
  hjoint = warp_sum(hjoint);
  if ((tid & 31) == 0) part[tid >> 5] = make_float2(mult, hjoint);
}

// The bias sector is reduced into by every CTA once per tile; loads of it queue behind
// those reductions at its single L2 slice.  So ONE lane per CTA fetches it per tile
// (issued at the top of the tile, consumed after the gathers are in flight) and hands
// it to the other warps through shared memory + named barrier 1.
struct BiasFetch {
  float* slot;   // [2] floats in the smem header, indexed by tile parity
  float pending; // lane 0 of warp 0: the in-flight value
  __device__ __forceinline__ void issue(const HogwildArgs& a, bool use_w0, int tid) {
    pending = 0.f;
    if (use_w0 && tid == 0) pending = ld_cg_f(a.w0);  // warp 0 fetches the bias
  }
  // returns the tile's bias in every thread of the CTA
  __device__ __forceinline__ float get(bool use_w0, int tid, int it, int nthreads) {
    if (!use_w0) return 0.f;
    float* s = slot + (it & 1);
    if (tid < 32) {
      const float v = __shfl_sync(0xffffffffu, pending, 0);
      if (tid == 0) *s = v;
      __threadfence_block();
      named_bar_arrive(1, nthreads);
      return v;
    }
    named_bar_sync(1, nthreads);
    return *s;
  }
};

// Dynamic tile scheduler: CTAs claim row tiles from a global counter in file order, so
// the tail of the epoch is balanced (a static round-robin leaves 1/9 of the CTAs a whole
// tile short on C2) and the rows in flight stay one contiguous window.  Used by thread 0
// only.  The last CTA to run dry resets the two words for the next launch.
struct TileSched {
  unsigned int* w;
  uint32_t n_tiles;
  bool dry;
  __device__ __forceinline__ uint32_t claim() {
    if (dry) return HW_NO_TILE;
    const uint32_t t = atomicAdd(w, 1u);
    if (t >= n_tiles) {
      dry = true;
      return HW_NO_TILE;
    }
    return t;
  }
  // split claim: fire() only issues the atomic (its latency must not stall the producer
  // thread, which also processes rows); resolve() interprets the value a tile later
  __device__ __forceinline__ uint32_t fire() { return dry ? HW_NO_TILE : atomicAdd(w, 1u); }
  __device__ __forceinline__ uint32_t resolve(uint32_t raw) {
    if (raw >= n_tiles) {
      dry = true;
      return HW_NO_TILE;
    }
    return raw;
  }
  // `last_raw`: the claim still in flight.  Its value must have RETURNED (the counter
  // increment performed) before this CTA reports itself dry, or the reset below could be
  // overtaken by it and the next launch would start at tile 1.
  __device__ __forceinline__ void finish(unsigned int n_ctas, uint32_t last_raw) {
    unsigned int inc = (last_raw == 0x7fffffffu) ? 2u : 1u;  // data dependence on the return value
    __threadfence();
    if (atomicAdd(w + 1, inc) == n_ctas - 1) {
      w[0] = 0u;
      w[1] = 0u;
    }
  }
};

using HogwildKernelFn = void (*)(const HogwildArgs);

// fm_rowlane.cu: kernel for (float4 chunks per row gp in {1,2}, rows of at most max_row_nnz <= 4
// entries), nullptr for any other shape.  The window kernel: a cooperative launch whose grid size is
// the window size; prof: the instantiation with phase timers; dealt: the schedule over the dealt CSR
// (no COMBINE, no bias ramp).  ws: the warp-specialised variant instead (no phase timers, no dealt
// schedule): blockDim = rows_per_tile + 32, smem header HW_WS_HDR_BYTES.
HogwildKernelFn pick_rowlane_kernel(int gp, int max_row_nnz, bool ws, bool damp, bool combine, bool prof, bool dealt);
// the window kernel's phase timers: cycles of CTA thread 0 per window, summed over the CTAs
constexpr int RL_PROF_SLOTS = 6;  // bias+gather, score+issue, bulk wait, barrier 1, fold, barrier 2

}  // namespace fmb
