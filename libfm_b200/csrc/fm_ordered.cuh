// fm_ordered.cuh -- FMB200_MODE_ORDERED: the sequentially CONSISTENT epoch.
//
// Reference semantics (src/libfm/src/fm_learn_sgd_element.h:56-67): example t reads every
// parameter as examples 0..t-1 left it.  This kernel keeps exactly that read/write ORDER
// for w0, w and V and changes only the association of three floating-point sums, so its
// result is deterministic and differs from the reference by rounding only (fp64 state;
// ~1e-13 relative on the parameters, far inside the 1e-5 RMSE gate of BASELINE.json).  It
// is NOT bit-exact: that is FMB200_MODE_INORDER (fm_inorder.cu).
//
// What makes the reference's loop serial, and how each part is handled here:
//   (1) w / V rows: example t depends on the LAST earlier example that names one of its
//       features.  Every upload precomputes, per entry, the distance to that previous
//       entry (`link`) and, per row, the distance to the nearest earlier row sharing a
//       feature (`rowdep`) -- pure index work (fm_ordered.cu).  Consecutive rows with no
//       dependency among them form a RUN (found on the fly from rowdep with two ballots):
//       their gathers, scores and fm_SGD write-backs (fm_sgd.h:38-50) run in parallel.
//   (2) the bias: w0 is read and rewritten by every example (fm_model.h:107-109,
//       fm_sgd.h:34-37), but only through  p_t = w0_t + R_t,  R_t = sum_i w_i x_i +
//       1/2 sum_f (sum_f^2 - sumsq_f)  independent of w0.  For regression the step
//       w0' = w0 - lr((clamp(w0+R_t) - y_t) + reg0 w0) is AFFINE in w0 once the example's
//       clamp state (inside / at min / at max) is fixed.  Every example's thread guesses its
//       state from the bias at the start of the run and publishes (a_t, b_t); warp 0 walks
//       w <- fma(a_t, w, b_t), cut into 8 segments composed in parallel (ord_bias_chain);
//       the examples' threads check their guess against the bias they actually read, and
//       the chain is re-walked behind the first contradicted one -- a consistent assignment
//       IS the sequential answer (induction over t).  Classification (logistic multiplier)
//       walks the chain serially from shared memory.
//   (3) memory: one CTA owns the epoch (there is ONE chain).  Compute warps walk the runs of
//       tile T; tile T-1's final records are written back to global memory and tile T+1's
//       records fetched (cp.async, L2 -> shared, 16 B) into a 3-deep ring by a helper warp
//       beside the runs where the thread budget allows (k <= 32), else by the compute warps
//       before them (ordered_epoch: one driver, two configurations); the CSR
//       of tile T+2 arrives by TMA bulk copies (cp.async.bulk + mbarrier).  A record fetched
//       that early is stale if its feature is written by tile T or T+1 itself; exactly those
//       entries (known from `link`) skip the fetch and read the record FORWARDED in shared
//       memory: every fm_SGD result lands in the writer's own ring slot.
//
// Thread mapping: GL lanes per example, each owning KF <= 8 CONSECUTIVE factors (k <= 8: one
// lane per example, no cross-lane reduction at all), at most min(ORD_SMAX, 1024 / GL) examples
// per run.  ZF > 0 kernels (k in {2,4,8}, rows of <= ZF entries) keep a row's records in
// registers from the score to the update; the one-hot two-field shape has its own formulas.
//
// The mode is bound by LATENCY: with one warp per scheduler every dependent instruction costs
// 4-8 cycles, and a run is score -> chain -> check + update with three barriers.  What the
// round-2 measurements say about each structure tried is in DESIGN.md section 3.2.
//
// This header is also compiled for the host (tests/simt/: FMB_SIMT_HOST) and run thread
// for thread against the sequential oracle.
#pragma once
#include <stdint.h>
#ifndef FMB_SIMT_HOST
#include "fm_device.cuh"
#endif

namespace fmb {

// phase timing (development aid): one thread per role adds the cycles since its previous mark to a slot
#ifdef FMB_SIMT_HOST
#define ORD_PROF(cond, slot)
#else
#define ORD_PROF(cond, slot)                                                                 \
  if (a.prof != nullptr && (cond)) {                                                         \
    const long long now_ = clock64();                                                        \
    reinterpret_cast<unsigned long long*>(smem + ORD_PROF_OFF)[slot] += (unsigned long long)(now_ - tprof); \
    tprof = now_;                                                                            \
  }
#endif

constexpr uint32_t ORD_NONE = 0xffffffffu;
constexpr int ORD_SMAX = 128;  // examples per run: ORD_EL per lane in the bias scan
constexpr int ORD_EL = ORD_SMAX / 32;
constexpr int ORD_NBUF = 3;    // ring depth (CSR stages and record buffers)
// [0,24) mbarriers | [32,40) run lengths | [40,48) first contradicted clamp guess, by iteration parity |
// [64, +2048) sAB: per example (a_t, b_t) of its bias step w -> a_t w + b_t   (classification: sR scores | sM
// multipliers) | [2112, +1032) sW: [0, 8) the bias at the start of each chain segment, [ORD_SMAX] the bias after the run
// | [3200, +2048) sPre: per example the affine map from its segment's start to the bias it reads
// | [5248, +256) spare | [5504, +128) phase timers (development aid)
constexpr int ORD_HDR_BYTES = 5632;
constexpr int ORD_PROF_OFF = 5504;
constexpr int ORD_SW_OFF = 64 + 2 * ORD_SMAX * 8;  // sW[0..8): the bias at the start of each segment; sW[ORD_SMAX]: after the run
constexpr int ORD_SPRE_OFF = 3200;
constexpr int ORD_SEGS = 8;  // segments of the bias chain (lanes of warp 0 composing in parallel)
constexpr int ORD_MAX_THREADS = 1024;

struct OrderedArgs {
  const uint64_t* row_ptr;
  const uint32_t* col;
  const float* val;
  const float* target;
  const uint32_t* link;    // [nnz]: e - (previous entry with the same feature), ORD_NONE if none
  const uint32_t* rowdep;  // [n_rows]: r - (nearest earlier row sharing a feature); 0 = the row
                           // names a feature twice; ORD_NONE if none
  const uint32_t* shape;   // one word: bit 0 = every value is 1, bit 1 = every row has exactly max_row_nnz entries
  uint64_t n_rows;
  uint32_t n_tiles;
  int tile_rows;      // TR
  uint32_t tile_cap;  // TE: entries staged per tile incl. alignment slack (multiple of 4)
  double* w0;
  double* w;  // 16-byte aligned
  double* v;  // 16-byte aligned, attribute-major [n][k]
  int k;
  int kw;  // doubles copied per V row: k (k even) or k+1 (k odd: 16-byte window around the row)
  int rs;  // record stride in doubles = kw + 2 (the aligned pair holding w[id])
  int use_w0, use_w;
  double lr, reg0, regw, regv, min_target, max_target;
  uint32_t csr_bytes;  // one CSR stage
  uint32_t rec_bytes;  // one record buffer = tile_cap * rs * 8
  unsigned long long* prof;  // phase timing (development aid): 16 clock64 accumulators, or null
  int debug;           // timing experiments only (results become wrong): 1 = no write-back to global,
                       // 2 = no bias scan (multiplier 0), 4 = no fm_SGD phase, 8 = no score phase
};

// ---- shared-memory layout (host and device agree through these) -------------------------
// every staged array is a whole number of 16-byte units (TMA bulk copies) starting on one
__host__ __device__ inline uint32_t ord_rp_bytes(int TR) { return ((uint32_t)(TR + 2) * 8u + 15u) & ~15u; }
__host__ __device__ inline uint32_t ord_row_bytes(int TR) { return ((uint32_t)(TR + 4) * 4u + 15u) & ~15u; }
__host__ __device__ inline uint32_t ord_csr_bytes(int TR, uint32_t TE) {
  // rp | target | rowdep | col | val | link | src | superseded (1 byte per entry, TE is a multiple of 4)
  return ord_rp_bytes(TR) + 2u * ord_row_bytes(TR) + 4u * TE * 4u + ((TE + 15u) & ~15u);
}
__host__ __device__ inline size_t ord_smem_bytes(int TR, uint32_t TE, int rs) {
  return (size_t)ORD_HDR_BYTES + (size_t)ORD_NBUF * ord_csr_bytes(TR, TE) +
         (size_t)ORD_NBUF * TE * (size_t)rs * 8u;
}

struct OrdStage {  // views into one CSR stage
  const uint64_t* rp;     // rp[i] = row_ptr[r0 + i]
  const float* tg;        // tg[i] = target[r0 + i]
  const uint32_t* rd;     // rd[i] = rowdep[r0 + i]
  const uint32_t* col;    // index j = e - (E0 & ~3)
  const float* val;
  const uint32_t* link;
  uint32_t* src;          // byte offset (from the smem base) of the record each entry reads
  unsigned char* sup;     // 1 = a later entry of the SAME tile rewrites this feature (no write-back)
};

__device__ __forceinline__ OrdStage ord_stage(const OrderedArgs& a, unsigned char* smem, uint32_t tile) {
  unsigned char* b = smem + ORD_HDR_BYTES + (size_t)(tile % ORD_NBUF) * a.csr_bytes;
  const uint64_t r0 = (uint64_t)tile * a.tile_rows;
  const uint32_t rpb = ord_rp_bytes(a.tile_rows), rwb = ord_row_bytes(a.tile_rows);
  OrdStage s;
  s.rp = reinterpret_cast<const uint64_t*>(b) + (r0 & 1);
  s.tg = reinterpret_cast<const float*>(b + rpb) + (r0 & 3);
  s.rd = reinterpret_cast<const uint32_t*>(b + rpb + rwb) + (r0 & 3);
  unsigned char* e = b + rpb + 2 * rwb;
  s.col = reinterpret_cast<const uint32_t*>(e);
  s.val = reinterpret_cast<const float*>(e + (size_t)a.tile_cap * 4);
  s.link = reinterpret_cast<const uint32_t*>(e + (size_t)a.tile_cap * 8);
  s.src = reinterpret_cast<uint32_t*>(e + (size_t)a.tile_cap * 12);
  s.sup = e + (size_t)a.tile_cap * 16;
  return s;
}

__device__ __forceinline__ uint32_t ord_rec_base(const OrderedArgs& a, uint32_t tile) {
  return (uint32_t)ORD_HDR_BYTES + (uint32_t)ORD_NBUF * a.csr_bytes + (tile % ORD_NBUF) * a.rec_bytes;
}

// TMA producer (one thread): stage the CSR of `tile`, whose entry range [nb, ne) is known.
__device__ __forceinline__ void ord_issue_csr(const OrderedArgs& a, unsigned char* smem, uint64_t* bars,
                                              uint32_t tile, uint64_t nb, uint64_t ne, uint64_t policy) {
  unsigned char* b = smem + ORD_HDR_BYTES + (size_t)(tile % ORD_NBUF) * a.csr_bytes;
  const uint64_t r0 = (uint64_t)tile * a.tile_rows;
  const uint32_t rpb = ord_rp_bytes(a.tile_rows), rwb = ord_row_bytes(a.tile_rows);
  const uint64_t ab = nb & ~3ull, ae = (ne + 3ull) & ~3ull;
  const uint32_t eb = (uint32_t)(ae - ab) * 4u;
  uint64_t* bar = bars + (tile % ORD_NBUF);
  mbar_arrive_expect_tx(bar, rpb + 2u * rwb + 3u * eb);
  bulk_g2s_hint(b, a.row_ptr + (r0 & ~1ull), rpb, bar, policy);
  bulk_g2s_hint(b + rpb, a.target + (r0 & ~3ull), rwb, bar, policy);
  bulk_g2s_hint(b + rpb + rwb, a.rowdep + (r0 & ~3ull), rwb, bar, policy);
  if (eb) {
    unsigned char* e = b + rpb + 2 * rwb;
    bulk_g2s_hint(e, a.col + ab, eb, bar, policy);
    bulk_g2s_hint(e + (size_t)a.tile_cap * 4, a.val + ab, eb, bar, policy);
    bulk_g2s_hint(e + (size_t)a.tile_cap * 8, a.link + ab, eb, bar, policy);
  }
}

// Decide, for every entry of tile `tile`, where its record will be read from, and start the
// fetch of the records that come from HBM/L2.  Runs while tile-1 is being processed, i.e.
// after the barrier that closed tile-2: anything tile-2 or earlier wrote is visible to the
// fetch; a feature last written by tile-1 or by this tile is forwarded from the writer's
// ring slot instead (the fetched copy would be stale).
template <int KC>  // KC > 0: kw == KC at compile time (the fetch unrolls); 0: runtime
__device__ __forceinline__ void ord_prep(const OrderedArgs& a, unsigned char* smem, uint32_t tile, int tid,
                                         int nthreads) {
  const OrdStage s = ord_stage(a, smem, tile);
  const uint64_t r0 = (uint64_t)tile * a.tile_rows;
  const uint32_t nrows = (uint32_t)min((uint64_t)a.tile_rows, a.n_rows - r0);
  const uint64_t E0 = s.rp[0], E1 = s.rp[nrows];
  const uint64_t ab = E0 & ~3ull;
  const uint32_t j0 = (uint32_t)(E0 - ab), j1 = (uint32_t)(E1 - ab);
  uint64_t E0p = E0, abp = ab;  // first entry of the previous tile (forwarding window)
  if (tile > 0) {
    const OrdStage sp = ord_stage(a, smem, tile - 1);
    E0p = sp.rp[0];
    abp = E0p & ~3ull;
  }
  const uint32_t rec = ord_rec_base(a, tile), recp = ord_rec_base(a, tile + ORD_NBUF - 1);
  const uint32_t recb = (uint32_t)a.rs * 8u;
  const int k = a.k, kw = a.kw;
  // (s.sup[] is all zero here: zeroed at kernel start and re-zeroed by the write-back that read it)
  // Four entries per thread at a time: their link / id loads are issued together, then the decisions, then
  // the fetches -- one dependent load chain per batch instead of one per entry.
  constexpr int PU = 4;
  for (uint32_t jbase = j0 + tid; jbase < j1; jbase += PU * nthreads) {
    uint32_t L[PU], id[PU];
    bool in[PU];
#pragma unroll
    for (int u = 0; u < PU; u++) {
      const uint32_t j = jbase + u * nthreads;
      in[u] = j < j1;
      L[u] = in[u] ? s.link[j] : ORD_NONE;
      id[u] = in[u] ? s.col[j] : 0u;
    }
#pragma unroll
    for (int u = 0; u < PU; u++) {
      if (!in[u]) continue;
      const uint32_t j = jbase + u * nthreads;
      const uint64_t e = ab + j;
      uint32_t src = rec + j * recb;
      if (L[u] != ORD_NONE && (uint64_t)L[u] <= e - E0p) {  // previous writer is inside the window
        if (L[u] <= j - j0) {  // this tile: that entry's value never needs to reach global memory
          src = rec + (j - L[u]) * recb;
          s.sup[j - L[u]] = 1;
        } else src = recp + (uint32_t)((e - L[u]) - abp) * recb;                 // the previous tile
      } else {
        unsigned char* dst = smem + src;
        if (KC > 0) {
          const double* gv = a.v + (size_t)id[u] * KC;
#pragma unroll
          for (int c = 0; c < KC; c += 2) cp_async_16(dst + c * 8, gv + c);
          if (a.use_w) cp_async_16(dst + KC * 8, a.w + (id[u] & ~1u));
        } else {
          const uint32_t vo = (k & 1) ? (id[u] & 1u) : 0u;
          const double* gv = a.v + (size_t)id[u] * k - vo;
          for (int c = 0; c < kw; c += 2) cp_async_16(dst + c * 8, gv + c);
          if (a.use_w) cp_async_16(dst + kw * 8, a.w + (id[u] & ~1u));
        }
      }
      s.src[j] = src;
    }
  }
}

__device__ __forceinline__ double ord_shfl(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }
__device__ __forceinline__ double ord_shfl_up(double v, int d) { return __shfl_up_sync(0xffffffffu, v, d); }
__device__ __forceinline__ double ord_shfl_xor(double v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }

// clamp state of a score: 0 inside, 1 at min_target, 2 at max_target.  Same selection as
// fmin(max, p) then fmax(min, .) (fm_learn_sgd_element.h:60-61): NaN or too large -> max,
// then anything below min -> min.
__device__ __forceinline__ int ord_state(double p, double lo, double hi, bool inverted) {
  const bool h = !(p <= hi), l = p < lo;
  return h ? (inverted ? 1 : 2) : (l ? 1 : 0);  // selects, no branches: this sits on the scan's critical path
}

// length of the run starting at tile-relative row t0 (executed by one whole warp): rows are
// added while they depend on no row of the run (rd[r] = distance to the nearest earlier row
// sharing a feature; 0 = the row names a feature twice and must run alone)
__device__ __forceinline__ int ord_detect(const OrdStage& s, int t0, int nrows, int smax, int lane) {
  int P = smax;
#pragma unroll
  for (int q = ORD_EL - 1; q >= 0; q--) {
    const int t = 32 * q + lane, r = t0 + t;
    bool stop = (t >= smax) || (r >= nrows);
    if (!stop && t > 0) stop = s.rd[r] <= (uint32_t)t;
    const unsigned m = __ballot_sync(0xffffffffu, stop);
    if (m) P = 32 * q + __ffs(m) - 1;
  }
  if (P < 1) P = 1;
  if (s.rd[t0] == 0u) P = 1;
  return P;
}

template <int KF>
__device__ __forceinline__ void ord_load(const double* p, double (&v)[KF], int nvalid, bool vec) {
  if (KF >= 2 && vec) {
#pragma unroll
    for (int q = 0; q < KF; q += 2) {
      double2 t = make_double2(0.0, 0.0);
      if (q < nvalid) t = *reinterpret_cast<const double2*>(p + q);
      v[q] = t.x;
      v[q + 1] = t.y;
    }
  } else {
#pragma unroll
    for (int q = 0; q < KF; q++) v[q] = (q < nvalid) ? p[q] : 0.0;
  }
}
template <int KF>
__device__ __forceinline__ void ord_store(double* p, const double (&v)[KF], int nvalid, bool vec) {
  if (KF >= 2 && vec) {
#pragma unroll
    for (int q = 0; q < KF; q += 2)
      if (q < nvalid) *reinterpret_cast<double2*>(p + q) = make_double2(v[q], v[q + 1]);
  } else {
#pragma unroll
    for (int q = 0; q < KF; q++)
      if (q < nvalid) p[q] = v[q];
  }
}

// The bias chain of one run, regression.  The step  w0' = w0 - lr((clamp(w0 + R_t) - y_t) + reg0 w0)
// (fm_learn_sgd_element.h:58-62, fm_sgd.h:34-37) is affine in w0 once the example's clamp state (inside / at
// min / at max) is fixed: w0' = a_t w0 + b_t.  Every example's own thread GUESSES its state from the bias at
// the start of the run and publishes (a_t, b_t); warp 0 then walks  w <- fma(a_t, w, b_t)  -- one dependent
// DFMA per example, cut into segments that are composed in parallel (ord_bias_chain); the
// Kogge-Stone scan over shuffles this replaces spent 270 dependent instructions per run.  The examples' threads then check their guess against the bias they
// actually read, in parallel; the first contradicted one corrects its pair and the chain is walked again from
// there (a consistent assignment IS the sequential answer, by induction over t; every pass finalises at least
// one more example).
struct OrdBias {
  double lr, lo, hi, a_mid, a_out;
  bool inverted;
};
__device__ __forceinline__ double2 ord_bias_pair(const OrdBias& c, int st, double R, double y) {
  return make_double2(st == 0 ? c.a_mid : c.a_out, -c.lr * ((st == 0 ? R : (st == 1 ? c.lo : c.hi)) - y));
}
// The chain of one run, walked by warp 0.  The run is cut into up to ORD_SEGS segments of `1 << sh` examples;
// lane s composes the affine maps of segment s (two independent DFMA chains: 8 cycles per example, all segments
// at once) and leaves in sPre[t] the map from the segment's start to the bias example t reads; the bias is then
// threaded through the segment totals (one DFMA per segment) into sW[s].  Example t reads
//   fma(sPre[t].x, sW[t >> sh], sPre[t].y).
// Critical path ~ 8 (P / 8 + 8) cycles instead of 8 P.
// A re-walk behind a contradicted guess (from > 0, rare) is serial: sPre[t] = (0, bias) for t >= from.
template <int SEG>
__device__ __forceinline__ void ord_bias_compose(const double2* sAB, double2* sPre, int t0, double& A, double& B) {
  // the segment's pairs first (independent loads), then the two dependent chains, the stores trailing.
  // No bounds: slots behind the run hold the identity (1, 0) and sPre has room for every slot.
  double2 ab[SEG];
#pragma unroll
  for (int e = 0; e < SEG; e++) ab[e] = sAB[t0 + e];
#pragma unroll
  for (int e = 0; e < SEG; e++) {
    sPre[t0 + e] = make_double2(A, B);
    B = fma(ab[e].x, B, ab[e].y);  // w -> ab.x (A w + B) + ab.y
    A = ab[e].x * A;
  }
}
// Executed by the whole of warp 0.  sh = log2(segment length): 2 (P <= 32), 3 (P <= 64), 4.
__device__ __forceinline__ void ord_bias_chain(const double2* sAB, double2* sPre, double* sW, int from, int P, int sh,
                                               double w0, int lane) {
  if (from == 0) {
    double A = 1.0, B = 0.0;  // lanes without a segment keep the identity
    if (lane < ORD_SEGS) {
      const int t0 = lane << sh;
      if (sh == 2) ord_bias_compose<4>(sAB, sPre, t0, A, B);
      else if (sh == 3) ord_bias_compose<8>(sAB, sPre, t0, A, B);
      else ord_bias_compose<16>(sAB, sPre, t0, A, B);
    }
    // Inclusive scan of the 8 segment totals over the first 8 lanes (3 Kogge-Stone steps: maps compose as
    // (A2,B2) o (A1,B1) = (A2 A1, A2 B1 + B2)), then lane s applies "everything before segment s" to the run's
    // starting bias.  28 instructions where threading the bias through 8 fetched totals took ~60; this warp's
    // instruction count IS the run's critical path.
#pragma unroll
    for (int o = 1; o < ORD_SEGS; o <<= 1) {
      const double Ap = __shfl_up_sync(0xffffffffu, A, o), Bp = __shfl_up_sync(0xffffffffu, B, o);
      if (lane >= o) {  // (lanes >= ORD_SEGS carry the identity through and are never read)
        B = fma(A, Bp, B);
        A = A * Ap;
      }
    }
    // exclusive prefix = the inclusive one of the lane below
    double Ae = __shfl_up_sync(0xffffffffu, A, 1), Be = __shfl_up_sync(0xffffffffu, B, 1);
    if (lane == 0) {
      Ae = 1.0;
      Be = 0.0;
    }
    if (lane < ORD_SEGS) sW[lane] = fma(Ae, w0, Be);
    const double w = fma(A, w0, B);  // lane ORD_SEGS - 1: the bias after the run
    if (lane == ORD_SEGS - 1) sW[ORD_SMAX] = w;
  } else if (lane == 0) {
    double w = fma(sPre[from - 1].x, sW[(from - 1) >> sh], sPre[from - 1].y);  // the bias example from-1 read ...
    w = fma(sAB[from - 1].x, w, sAB[from - 1].y);                             // ... and left (its pair is corrected)
    for (int t = from; t < P; t++) {
      const double2 ab = sAB[t];
      sPre[t] = make_double2(0.0, w);
      w = fma(ab.x, w, ab.y);
    }
    sW[ORD_SMAX] = w;
  }
}

// barrier over one role's threads: the whole CTA (0), or a named barrier over the role (WS)
template <bool WS>
__device__ __forceinline__ void ord_group_sync(int id, int nthreads) {
  if (WS) named_bar_sync(id, nthreads);
  else __syncthreads();
}

struct OrdConsts {
  int k, kw;
  bool k0, k1;
  double lr, reg0, regw, regv, lo, hi;
  bool inverted;
  OrdBias bias;
  uint32_t recb;
};
__device__ __forceinline__ OrdConsts ord_consts(const OrderedArgs& a) {
  OrdConsts c;
  c.k = a.k;
  c.kw = a.kw;
  c.k0 = a.use_w0 != 0;
  c.k1 = a.use_w != 0;
  c.lr = a.lr;
  c.reg0 = a.reg0;
  c.regw = a.regw;
  c.regv = a.regv;
  c.lo = a.min_target;
  c.hi = a.max_target;
  c.inverted = c.hi < c.lo;
  c.bias.lr = c.lr;
  c.bias.lo = c.lo;
  c.bias.hi = c.hi;
  c.bias.a_mid = 1.0 - c.lr * (1.0 + c.reg0);
  c.bias.a_out = 1.0 - c.lr * c.reg0;
  c.bias.inverted = c.inverted;
  c.recb = (uint32_t)a.rs * 8u;
  return c;
}

// ZF > 0 selects the register-resident fast path: one lane per example (GL == 1), k == KF even, every
// row of the data set at most ZF entries.  The rows' records are loaded once with 16-byte accesses, kept
// in registers across the bias scan and written back to the ring from there -- no per-entry loop, no
// second read.  Rows that name a feature twice (singleton runs) take the general path.
//
// All runs of tile T, executed by the `nthreads` compute threads (tid in [0, nthreads)); sP[0] holds the
// length of the tile's first run.  Every thread carries the bias w0 (the clamp guesses start from it).
template <int GL, int KF, int TASK, int ZF, bool WS>
__device__ __forceinline__ void ord_tile_runs(const OrderedArgs& a, unsigned char* smem, const OrdConsts& cc,
                                              uint32_t T, int tid, int nthreads, double& w0, uint32_t& it,
                                              bool onehot) {
  const int lane = tid & 31, warp = tid >> 5;
  // the one-hot two-field shape (ratings data: every row is exactly user:1 item:1): with x = 1 and two
  // entries a, b the score is  w_a + w_b + sum_f v_af v_bf  (1/2 ((a+b)^2 - a^2 - b^2) = ab) and the
  // gradient of v_af is mult v_bf  (sum_f - v_af = v_bf)  -- 10 fp64 operations per example instead of 64 for
  // the score, 52 instead of ~100 for the update; fp64 instruction issue is what phase A of a run spends its
  // time on
  const bool oh = (ZF == 2) && onehot;
  const int gl = tid % GL;   // lane inside the example's group
  const int grp = tid / GL;  // example slot inside a run
  const int smax = min(ORD_SMAX, nthreads / GL);
  int* sP = reinterpret_cast<int*>(smem + 32);  // [2]: run lengths, double-buffered by run parity
  int* sBad = reinterpret_cast<int*>(smem + 40);  // [2]: first contradicted guess, by pass parity
  double* sR = reinterpret_cast<double*>(smem + 64);
  double* sM = sR + ORD_SMAX;
  double2* sAB = reinterpret_cast<double2*>(smem + 64);
  double* sW = reinterpret_cast<double*>(smem + ORD_SW_OFF);
  double2* sPre = reinterpret_cast<double2*>(smem + ORD_SPRE_OFF);
  const int dwarp = nthreads > 32 ? 1 : 0;  // the warp that searches the next run
  const int k = cc.k, kw = cc.kw;
  const bool k0 = cc.k0, k1 = cc.k1;
  const double lr = cc.lr, reg0 = cc.reg0, regw = cc.regw, regv = cc.regv, lo = cc.lo, hi = cc.hi;
  const bool inverted = cc.inverted;
  const OrdBias& bias = cc.bias;
  const uint32_t recb = cc.recb;
  const int f0 = gl * KF;                       // this lane's first factor
  const int nf = max(0, min(KF, k - f0));       // ... and how many of its KF slots are real
  const bool vec = ((k & 1) == 0) && (KF % 2 == 0);  // 16-byte aligned factor slices
  const OrdStage s = ord_stage(a, smem, T);
  const uint64_t r0 = (uint64_t)T * a.tile_rows;
  const int nrows = (int)min((uint64_t)a.tile_rows, a.n_rows - r0);
  const uint64_t ab = s.rp[0] & ~3ull;
  const uint32_t j00 = (uint32_t)(s.rp[0] - ab);  // tile-relative index of the tile's first entry (even for width 2)
  const uint32_t rec = ord_rec_base(a, T);

  int t0 = 0;
  int pi = 0;  // parity of the run inside the tile
  long long tprof = 0;
  ORD_PROF(tid == 0, 15);  // (resets the mark; slot 15 collects what lies between tiles)
  while (t0 < nrows) {
    const int P = sP[pi];
    // ---- scores of the run's examples: fm_model.h:105-127 with R_t = p_t - w0 ----------
    const bool act = grp < P;
    const int r = t0 + grp;
    uint32_t jb = 0, je = 0;
    bool rowdup = false;
    double sum[KF];  // (zeroed by the paths that use it: the one-hot path does not)
    double Rloc = 0.0;
    if (act && !oh) {
      jb = (uint32_t)(s.rp[r] - ab);
      je = (uint32_t)(s.rp[r + 1] - ab);
      rowdup = s.rd[r] == 0u;
    }
    constexpr int ZR = ZF > 0 ? ZF : 1;
    double fv[ZR][KF], fw[ZR], fx[ZR];  // fast path: the row's records, weights and values
    uint32_t fid[ZR];
    const bool fast = (ZF > 0) && (s.rd[t0] != 0u);  // uniform: a row naming a feature twice runs alone
    if (act && oh && !fast) {  // (that row takes the general path: it wants its offsets)
      jb = (uint32_t)(s.rp[r] - ab);
      je = (uint32_t)(s.rp[r + 1] - ab);
      rowdup = s.rd[r] == 0u;
    }
    if (fast && oh) {
      if (act) {  // fixed width: no offsets to read
        jb = j00 + 2u * (uint32_t)r;
        je = jb + 2u;
      }
      if (act && !(a.debug & 8)) {
        const uint2 so = *reinterpret_cast<const uint2*>(s.src + jb);
        const uint2 ids = *reinterpret_cast<const uint2*>(s.col + jb);
        fid[0] = ids.x;
        fid[1] = ids.y;
        const double* ra = reinterpret_cast<const double*>(smem + so.x);
        const double* rb = reinterpret_cast<const double*>(smem + so.y);
#pragma unroll
        for (int q = 0; q < KF; q += 2) {
          const double2 ta = *reinterpret_cast<const double2*>(ra + q), tb = *reinterpret_cast<const double2*>(rb + q);
          fv[0][q] = ta.x;
          fv[0][q + 1] = ta.y;
          fv[1][q] = tb.x;
          fv[1][q + 1] = tb.y;
        }
        fw[0] = k1 ? ra[kw + (ids.x & 1u)] : 0.0;
        fw[1] = k1 ? rb[kw + (ids.y & 1u)] : 0.0;
        double r0 = fw[0], r1 = fw[1];  // two accumulators: half the dependent chain
#pragma unroll
        for (int q = 0; q < KF; q += 2) {
          r0 = fma(fv[0][q], fv[1][q], r0);
          r1 = fma(fv[0][q + 1], fv[1][q + 1], r1);
        }
        Rloc = r0 + r1;
      }
    } else if (fast) {
#pragma unroll
      for (int q = 0; q < KF; q++) sum[q] = 0.0;
      if (act && !(a.debug & 8)) {
        const uint32_t cnt = je - jb;
#pragma unroll
        for (int e = 0; e < ZR; e++) {
          // slots beyond the row's length hold zeros and touch nothing: an empty row's jb may lie past the
          // tile's last entry, where src[] was never written (a misaligned shared-memory address on the device)
          fid[e] = 0u;
          fx[e] = 0.0;
          fw[e] = 0.0;
#pragma unroll
          for (int q = 0; q < KF; q++) fv[e][q] = 0.0;
          if ((uint32_t)e < cnt) {
            const uint32_t j = jb + e;
            const double* rp_ = reinterpret_cast<const double*>(smem + s.src[j]);
            fid[e] = s.col[j];
            fx[e] = (double)s.val[j];
#pragma unroll
            for (int q = 0; q < KF; q += 2) {
              const double2 t2 = *reinterpret_cast<const double2*>(rp_ + q);
              fv[e][q] = t2.x;
              fv[e][q + 1] = t2.y;
            }
            if (k1) fw[e] = rp_[kw + (fid[e] & 1u)];
          }
        }
        double ssq[KF];
#pragma unroll
        for (int q = 0; q < KF; q++) ssq[q] = 0.0;
#pragma unroll
        for (int e = 0; e < ZR; e++) {
#pragma unroll
          for (int q = 0; q < KF; q++) {
            const double d = fv[e][q] * fx[e];
            sum[q] += d;
            ssq[q] += d * d;
          }
          Rloc += fw[e] * fx[e];
        }
#pragma unroll
        for (int q = 0; q < KF; q++) Rloc += 0.5 * (sum[q] * sum[q] - ssq[q]);
      }
    } else {
#pragma unroll
      for (int q = 0; q < KF; q++) sum[q] = 0.0;
    }
    if (!fast && act && !(a.debug & 8)) {
      double ssq[KF];
#pragma unroll
      for (int q = 0; q < KF; q++) ssq[q] = 0.0;
      for (uint32_t j = jb; j < je; j++) {
        uint32_t jj = j;
        if (rowdup)  // a feature named twice: both entries score with the value before the row
          while (s.link[jj] != ORD_NONE && s.link[jj] <= jj - jb) jj -= s.link[jj];
        const double* rp_ = reinterpret_cast<const double*>(smem + s.src[jj]);
        const uint32_t id = s.col[j];
        const double x = (double)s.val[j];
        const uint32_t vo = (k & 1) ? (id & 1u) : 0u;
        double vv[KF];
        ord_load<KF>(rp_ + vo + f0, vv, nf, vec);
#pragma unroll
        for (int q = 0; q < KF; q++) {
          const double d = vv[q] * x;  // slots beyond k hold 0
          sum[q] += d;
          ssq[q] += d * d;
        }
        if (k1 && (int)((j - jb) % GL) == gl) Rloc += rp_[kw + (id & 1u)] * x;
      }
#pragma unroll
      for (int q = 0; q < KF; q++) Rloc += 0.5 * (sum[q] * sum[q] - ssq[q]);
    }
#pragma unroll
    for (int o = GL / 2; o > 0; o >>= 1) Rloc += ord_shfl_xor(Rloc, o);

    const int t0n = t0 + P;

    // ---- fm_SGD (fm_sgd.h:38-50) for the lane's example with multiplier `mult`: result into the own ring slot
    auto sgd_update = [&](double mult) {
      if (fast && oh) {
        if (act && !(a.debug & 4)) {
          double* oa = reinterpret_cast<double*>(smem + rec + jb * recb);
          double* ob = oa + a.rs;
          // fm_sgd.h:44-48 with x = 1: grad of v_af = sum_f - v_af = v_bf
          if (regv == 0.0) {  // (uniform) no regularisation: one FMA per factor, v - (lr mult) v_other
            const double lm = -lr * mult;
#pragma unroll
            for (int q = 0; q < KF; q += 2) {
              const double a0 = fv[0][q], a1 = fv[0][q + 1], b0 = fv[1][q], b1 = fv[1][q + 1];
              *reinterpret_cast<double2*>(oa + q) = make_double2(fma(lm, b0, a0), fma(lm, b1, a1));
              *reinterpret_cast<double2*>(ob + q) = make_double2(fma(lm, a0, b0), fma(lm, a1, b1));
            }
          } else {
#pragma unroll
            for (int q = 0; q < KF; q += 2) {
              const double a0 = fv[0][q], a1 = fv[0][q + 1], b0 = fv[1][q], b1 = fv[1][q + 1];
              *reinterpret_cast<double2*>(oa + q) =
                  make_double2(fma(-lr, fma(regv, a0, mult * b0), a0), fma(-lr, fma(regv, a1, mult * b1), a1));
              *reinterpret_cast<double2*>(ob + q) =
                  make_double2(fma(-lr, fma(regv, b0, mult * a0), b0), fma(-lr, fma(regv, b1, mult * a1), b1));
            }
          }
          if (k1) {
            oa[kw + (fid[0] & 1u)] = fma(-lr, fma(regw, fw[0], mult), fw[0]);
            ob[kw + (fid[1] & 1u)] = fma(-lr, fma(regw, fw[1], mult), fw[1]);
          }
        }
      } else if (fast) {
        if (act && !(a.debug & 4)) {
          const uint32_t cnt = je - jb;
#pragma unroll
          for (int e = 0; e < ZR; e++) {
            if ((uint32_t)e < cnt) {
              double* own = reinterpret_cast<double*>(smem + rec + (jb + e) * recb);
              const double x = fx[e], x2 = x * x;
#pragma unroll
              for (int q = 0; q < KF; q += 2) {
                double c0 = fv[e][q], c1 = fv[e][q + 1];
                c0 -= lr * (mult * (sum[q] * x - c0 * x2) + regv * c0);
                c1 -= lr * (mult * (sum[q + 1] * x - c1 * x2) + regv * c1);
                *reinterpret_cast<double2*>(own + q) = make_double2(c0, c1);
              }
              if (k1) {
                double cw = fw[e];
                cw -= lr * (mult * x + regw * cw);
                own[kw + (fid[e] & 1u)] = cw;
              }
            }
          }
        }
      } else if (act && !(a.debug & 4)) {
        for (uint32_t j = jb; j < je; j++) {
          uint32_t jj = j;
          bool dupj = false;
          if (rowdup) {
            dupj = s.link[j] != ORD_NONE && s.link[j] <= j - jb;
            if (!dupj)
              while (s.link[jj] != ORD_NONE && s.link[jj] <= jj - jb) jj -= s.link[jj];
          }
          // a repeated feature continues from the row's previous write (fm_sgd.h:46 reads v again)
          const uint32_t so = dupj ? rec + (j - s.link[j]) * recb : s.src[jj];
          const double* rp_ = reinterpret_cast<const double*>(smem + so);
          double* own = reinterpret_cast<double*>(smem + rec + j * recb);
          const uint32_t id = s.col[j];
          const double x = (double)s.val[j];
          const uint32_t vo = (k & 1) ? (id & 1u) : 0u;
          double c[KF];
          ord_load<KF>(rp_ + vo + f0, c, nf, vec);
#pragma unroll
          for (int q = 0; q < KF; q++) {
            const double grad = sum[q] * x - c[q] * x * x;
            c[q] -= lr * (mult * grad + regv * c[q]);
          }
          ord_store<KF>(own + vo + f0, c, nf, vec);
          const bool mine = rowdup ? (gl == 0) : ((int)((j - jb) % GL) == gl);
          if (k1 && mine) {
            double cw = rp_[kw + (id & 1u)];
            cw -= lr * (mult * x + regw * cw);
            own[kw + (id & 1u)] = cw;
          }
        }
      }
    };

    if (k0 && TASK == 0) {
      // ---- regression: the bias chain (see ord_bias_chain) ----------------------------------------------
      constexpr bool SPEC = ZF > 0;  // (a ZF kernel's general-path runs are single rows: never redone)
      const int sh = P <= 32 ? 2 : (P <= 64 ? 3 : 4);  // segment length 4 / 8 / 16: at most ORD_SEGS segments
      const double y = act ? (double)s.tg[r] : 0.0;
      int st = ord_state(w0 + Rloc, lo, hi, inverted);  // guess: the bias at the start of the run
      // (slots behind the run hold the identity: the chain composes whole segments without bounds)
      // (sAB starts as all identity; a slot is dirtied only by its own thread group, which writes it every run)
      if (gl == 0 && grp < ORD_SMAX) sAB[grp] = act ? ord_bias_pair(bias, st, Rloc, y) : make_double2(1.0, 0.0);
      ORD_PROF(tid == 0, 0);  // phase A: scores
      ord_group_sync<WS>(1, nthreads);
      ORD_PROF(tid == 0, 1);  // ... waiting for the other warps' scores
      int from = 0;  // examples below `from` are final
      for (;;) {
        if (warp == 0) {
          if (a.debug & 2) {
            for (int t = lane; t < P; t += 32) sPre[t] = make_double2(0.0, 0.0);
            if (lane == 0) sW[ORD_SMAX] = 0.0;
          } else {
            ord_bias_chain(sAB, sPre, sW, from, P, sh, w0, lane);
          }
        }
        ORD_PROF(tid == 0, 2);  // the chain
        if (from == 0 && warp == dwarp) {  // the next run's length: warp 1 searches while thread 0 walks the chain
          const int Pn = (t0n < nrows) ? ord_detect(s, t0n, nrows, smax, lane) : 1;
          if (lane == 0) sP[pi ^ 1] = Pn;
        }
        ord_group_sync<WS>(1, nthreads);
        ORD_PROF(tid == 0, 3);  // barrier behind the chain
        // the next pass' flag word: its last readers (after the previous pass' closing barrier) are past the
        // barrier above, its next writers come after the barrier below
        if (tid == 0) sBad[(it + 1) & 1] = 0x7fffffff;
        double mult = 0.0;
        bool pending = false;
        if (act && grp >= from) {
          const double2 pre = sPre[grp];
          const double wt = fma(pre.x, sW[grp >> sh], pre.y);
          const double p = wt + Rloc;
          const int ns = (a.debug & 2) ? st : ord_state(p, lo, hi, inverted);
          if (ns != st) {  // the guess is contradicted: correct the pair; everything behind it is walked again
            st = ns;
            if (gl == 0) {
              sAB[grp] = ord_bias_pair(bias, ns, Rloc, y);
              atomicMin(&sBad[it & 1], grp);
            }
          }
          // fm_learn_sgd_element.h:58-62: mult = -(y - clamp(p)).  wt is final for the first contradicted
          // example and everything before it, so is their multiplier; later examples are checked again.
          mult = (a.debug & 2) ? 0.0 : (ns == 0 ? p : (ns == 1 ? lo : hi)) - y;
          // The register-resident path updates right away: its inputs stay in registers, so an example that
          // turns out to lie behind a contradicted guess simply writes its slots again in the next pass.  The
          // general path fetched its records INTO the slots it writes: it updates only once wt is known final.
          if (SPEC) sgd_update(mult);
          else pending = true;
        }
        ORD_PROF(tid == 0, 4);  // check + fm_SGD
        ord_group_sync<WS>(1, nthreads);  // ring slots, sAB corrections, the flag, the next run length
        ORD_PROF(tid == 0, 5);  // closing barrier
        const int bad = sBad[it & 1];
        it++;
        if (!SPEC && pending && grp <= bad) sgd_update(mult);
        if (bad >= P) break;
        from = bad + 1;  // (example `bad` read the right bias: its own result is final, its pair is corrected)
      }
      if (!SPEC) ord_group_sync<WS>(1, nthreads);  // the general path's ring slots are final
      w0 = sW[ORD_SMAX];  // every thread: the next run's guess
    } else if (k0) {
      // ---- classification: the chain walked serially by warp 0 (fm_learn_sgd_element.h:63-64) ----
      if (act && gl == 0) sR[grp] = Rloc;
      ord_group_sync<WS>(1, nthreads);
      if (warp == 0) {
        double wc = w0;
        for (int t = 0; t < P; t++) {
          const double y = (double)s.tg[t0 + t];
          const double p = wc + sR[t];
          const double m = (a.debug & 2) ? 0.0 : -y * (1.0 - 1.0 / (1.0 + exp(-y * p)));
          if (lane == (t & 31)) sM[t] = m;
          wc -= lr * (m + reg0 * wc);
        }
        if (lane == 0) sW[ORD_SMAX] = wc;
      }
      if (warp == dwarp) {
        const int Pn = (t0n < nrows) ? ord_detect(s, t0n, nrows, smax, lane) : 1;
        if (lane == 0) sP[pi ^ 1] = Pn;
      }
      ord_group_sync<WS>(1, nthreads);
      sgd_update(act ? sM[grp] : 0.0);
      ord_group_sync<WS>(1, nthreads);
      w0 = sW[ORD_SMAX];
    } else {
      double mult = 0.0;
      if (act) {
        const double y = (double)s.tg[r];
        if (TASK == 0) {
          const int st = ord_state(Rloc, lo, hi, inverted);
          mult = (st == 0 ? Rloc : (st == 1 ? lo : hi)) - y;
        } else {
          mult = -y * (1.0 - 1.0 / (1.0 + exp(-y * Rloc)));
        }
      }
      if (warp == 0) {  // the other parity: a slower warp may still be reading this run's length
        const int Pn = (t0n < nrows) ? ord_detect(s, t0n, nrows, smax, lane) : 1;
        if (lane == 0) sP[pi ^ 1] = Pn;
      }
      sgd_update(mult);
      ord_group_sync<WS>(1, nthreads);  // the run's ring slots (and the next length) are final before the next run reads them
    }
    t0 = t0n;
    pi ^= 1;
  }
}

// Write-back of tile T by `nthreads` threads (tid in [0, nthreads)): the tile's FINAL records go to global
// memory in one pass.  Per-update stores made every run's barrier wait behind them (r02 ncu); an entry
// whose feature is rewritten later in this tile (sup) never needs to leave the SM.  Also re-zeroes sup[].
template <bool WS, int KC>
__device__ __forceinline__ void ord_writeback(const OrderedArgs& a, unsigned char* smem, const OrdConsts& cc,
                                              uint32_t T, int tid, int nthreads) {
  const int k = cc.k, kw = cc.kw;
  const bool k1 = cc.k1;
  const uint32_t recb = cc.recb;
  const OrdStage s = ord_stage(a, smem, T);
  const uint64_t r0 = (uint64_t)T * a.tile_rows;
  const int nrows = (int)min((uint64_t)a.tile_rows, a.n_rows - r0);
  const uint64_t ab = s.rp[0] & ~3ull;
  const uint32_t rec = ord_rec_base(a, T);
  // ---- write-back: the tile's FINAL records go to global memory in one pass.  Per-update stores
  // made every run's barrier wait for their acknowledgement (r02 ncu: half of all stall samples on
  // the barriers, 5 200 cycles per run); an entry whose feature is rewritten later in this tile
  // (sup) never needs to leave the SM.  The next tile's fetches are issued behind the barrier of
  // ord_prep, i.e. after these stores.
  if (!(a.debug & 1)) {
    const uint32_t j0 = (uint32_t)(s.rp[0] - ab), j1 = (uint32_t)(s.rp[nrows] - ab);
    if ((k & 1) == 0) {
      // One entry per thread, four entries in flight: flags and ids first, then the records, then the stores.
      // (An earlier form spread the 16-byte pieces of a record over consecutive lanes -- fuller sectors per
      // store instruction, but ~60 instructions per piece of index arithmetic on warps that run one per
      // scheduler: the r02 v8 capture had the write-back at 8 500 cycles per 256-row tile.)
      constexpr int WU = 4;
      for (uint32_t jb_ = j0 + tid; jb_ < j1; jb_ += WU * nthreads) {
        bool go[WU];
        uint32_t idu[WU];
#pragma unroll
        for (int u = 0; u < WU; u++) {
          const uint32_t j = jb_ + u * nthreads;
          go[u] = j < j1 && !s.sup[j];
          idu[u] = go[u] ? s.col[j] : 0u;
        }
#pragma unroll
        for (int u = 0; u < WU; u++) {
          if (!go[u]) continue;
          const uint32_t j = jb_ + u * nthreads;
          const double* own = reinterpret_cast<const double*>(smem + rec + j * recb);
          double* gv = a.v + (size_t)idu[u] * k;
          if (KC > 0) {
            double2 t[KC / 2 > 0 ? KC / 2 : 1];
#pragma unroll
            for (int c = 0; c < KC / 2; c++) t[c] = *reinterpret_cast<const double2*>(own + 2 * c);
            const double wv = own[KC + (idu[u] & 1u)];
#pragma unroll
            for (int c = 0; c < KC / 2; c++) *reinterpret_cast<double2*>(gv + 2 * c) = t[c];
            if (k1) a.w[idu[u]] = wv;
          } else {
            for (int c = 0; c < kw; c += 2)
              *reinterpret_cast<double2*>(gv + c) = *reinterpret_cast<const double2*>(own + c);
            if (k1) a.w[idu[u]] = own[kw + (idu[u] & 1u)];
          }
        }
      }
      ord_group_sync<WS>(2, nthreads);  // every piece of a record has read its flag
      for (uint32_t jz = j0 + tid; jz < j1; jz += nthreads) s.sup[jz] = 0;
    } else {
      for (uint32_t j = j0 + tid; j < j1; j += nthreads) {
        const unsigned char sup = s.sup[j];
        s.sup[j] = 0;
        if (sup) continue;
        const double* own = reinterpret_cast<const double*>(smem + rec + j * recb);
        const uint32_t id = s.col[j];
        const uint32_t vo = id & 1u;
        double* gv = a.v + (size_t)id * k;
        for (int q = 0; q < k; q++) gv[q] = own[vo + q];
        if (k1) a.w[id] = own[kw + (id & 1u)];
      }
    }
  } else {
    const uint32_t j0 = (uint32_t)(s.rp[0] - ab), j1 = (uint32_t)(s.rp[nrows] - ab);
    for (uint32_t j = j0 + tid; j < j1; j += nthreads) s.sup[j] = 0;
  }
}

// ---- the epoch driver --------------------------------------------------------------------------------
// Threads [0, ncompute) are the compute threads: they walk the runs of tile T.  Threads [ncompute, ncompute +
// nparked) leave after the set-up (warp w runs on scheduler w % 4: they choose which compute warps the helpers
// share a scheduler with; measured to matter little, see fm_ordered.cu).  The rest, if any, are helpers.
// The helper steps of tile T: write tile T-1's final records back to global memory, stage the CSR of tile T+2
// (TMA into the stage tile T-1 held, which that write-back has just read), fetch tile T+1's records.
//   - With helpers, they run these steps while the compute threads walk tile T.  The write-back and the fetch
//     issue are LSU work a single SM issues at about one 16-byte request per cycle and neither is on the
//     dependency chain; done by the compute threads they take a share of the stall samples.  One CTA barrier
//     per tile joins the two roles.
//   - Without helpers (k > 32, where the compute threads fill the CTA), the compute threads run the same
//     steps themselves before the runs of tile T and leave tile T+1's fetches in flight during those runs.
// Either way the fetch of tile T+1 is issued behind tile T-1's write-back (a barrier over the threads of the
// helper steps in between), so what it may miss is what tiles T and T+1 write -- exactly the entries ord_prep
// forwards from the ring.
// HELPERS says at compile time whether there are helpers: one kernel that chose the configuration at run time
// ran the C2-shaped epoch 5% slower (H100 80GB HBM3, 400 W).  Without helpers every barrier is a CTA barrier;
// with them the compute threads (1) and the helpers (2) meet at named barriers.
template <int GL, int KF, int TASK, int ZF, bool HELPERS>
__device__ __forceinline__ void ordered_epoch(const OrderedArgs& a, unsigned char* smem, int ncompute,
                                              int nparked) {
  constexpr int KC = ZF > 0 ? KF : 0;  // the fast kernels run with k == KF (even): fetch and write-back unroll
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nthreads = blockDim.x;
  const int hstart = ncompute + nparked;
  // the threads of the helper steps: the helpers, or all compute threads (htid < 0: not one of them)
  const int nhelp = HELPERS ? nthreads - hstart : ncompute, htid = HELPERS ? tid - hstart : tid;
  const int nlive = nthreads - nparked, ltid = tid >= hstart ? tid - nparked : tid;
  const int smax = min(ORD_SMAX, ncompute / GL);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem);
  int* sP = reinterpret_cast<int*>(smem + 32);

  if (tid == 0) {
    for (int i = 0; i < ORD_NBUF; i++) mbar_init(bars + i, 1);
    fence_mbar_init();
    reinterpret_cast<int*>(smem + 40)[0] = 0x7fffffff;
    reinterpret_cast<int*>(smem + 40)[1] = 0x7fffffff;
  }
  if (tid < 16) reinterpret_cast<unsigned long long*>(smem + ORD_PROF_OFF)[tid] = 0ull;
  for (int g = tid; g < ORD_SMAX; g += nthreads) reinterpret_cast<double2*>(smem + 64)[g] = make_double2(1.0, 0.0);
  for (uint32_t t = 0; t < (uint32_t)ORD_NBUF; t++) {
    unsigned char* sup = ord_stage(a, smem, t).sup;
    for (uint32_t j = tid; j < a.tile_cap; j += nthreads) sup[j] = 0;
  }
  __syncthreads();

  const OrdConsts cc = ord_consts(a);
  double w0 = cc.k0 ? *a.w0 : 0.0;  // every thread follows the bias (the clamp guesses start from it)
  uint32_t it = 0;                   // passes of the bias chain so far (parity selects the flag word)
  const bool onehot = (ZF == 2) && ((*a.shape & 3u) == 3u);
  const uint32_t NT = a.n_tiles;
  const int TR = a.tile_rows;

  // producer state (htid 0): entry range of the next tile to stage, fetched a tile ahead
  uint64_t policy = 0, nb = 0, ne = 0;
  if (htid == 0) {
    policy = policy_evict_first();
    for (uint32_t t = 0; t < 2 && t < NT; t++) {
      const uint64_t r0 = (uint64_t)t * TR, r1 = min(r0 + TR, a.n_rows);
      ord_issue_csr(a, smem, bars, t, a.row_ptr[r0], a.row_ptr[r1], policy);
    }
    if (2 < NT) {
      const uint64_t r0 = 2ull * TR, r1 = min(r0 + TR, a.n_rows);
      nb = a.row_ptr[r0];
      ne = a.row_ptr[r1];
    }
  }
  if (tid >= ncompute && tid < hstart) return;  // parked (barriers below count the threads still running)
  mbar_wait(bars + 0, 0);
  ord_prep<KC>(a, smem, 0, ltid, nlive);  // the first tile's records: everybody fetches
  cp_async_commit();
  if (HELPERS) {  // (without helpers, the wait of tile 0 below covers these fetches)
    cp_async_wait_0();
    __syncthreads();
  }

  long long tprof = 0;
  const bool cprof = HELPERS && tid == 0, hprof = HELPERS && htid == 0;  // the driver's phase timers: with helpers only
  ORD_PROF(cprof || hprof, 15);
  for (uint32_t T = 0; T < NT; T++) {
    if (htid >= 0) {
      if (T > 0) {
        ord_writeback<HELPERS, KC>(a, smem, cc, T - 1, htid, nhelp);
        ord_group_sync<HELPERS>(2, nhelp);  // the stores are issued (and sup[] is clear) before anything below
      }
      ORD_PROF(hprof, 8);  // write-back
      if (htid == 0 && T + 2 < NT) {  // stage (T+2)%3 held tile T-1, whose write-back just read it
        ord_issue_csr(a, smem, bars, T + 2, nb, ne, policy);
        if (T + 3 < NT) {
          const uint64_t r0 = (uint64_t)(T + 3) * TR, r1 = min(r0 + TR, a.n_rows);
          nb = a.row_ptr[r0];
          ne = a.row_ptr[r1];
        }
      }
      if (T + 1 < NT) {
        mbar_wait(bars + (T + 1) % ORD_NBUF, ((T + 1) / ORD_NBUF) & 1);
        ORD_PROF(hprof, 9);  // CSR issue + wait
        ord_prep<KC>(a, smem, T + 1, htid, nhelp);
      }
      ORD_PROF(hprof, 10);  // fetch issue
      cp_async_commit();
      if (HELPERS) cp_async_wait_0();  // tile T+1's records have landed
      else cp_async_wait_1();     // this thread's fetches for tile T have landed, tile T+1's stay in flight
      ORD_PROF(hprof, 11);  // fetch landing
    }
    if (tid < ncompute) {
      // (complete since a tile ago; acquires the TMA's writes.  Without helpers every thread waited before ord_prep)
      if (HELPERS) mbar_wait(bars + T % ORD_NBUF, (T / ORD_NBUF) & 1);
      if (warp == 0) {  // length of the tile's first run (reads the CSR stage only)
        const OrdStage s = ord_stage(a, smem, T);
        const int nrows = (int)min((uint64_t)TR, a.n_rows - (uint64_t)T * TR);
        const int P0 = ord_detect(s, 0, nrows, smax, lane);
        if (lane == 0) sP[0] = P0;
      }
      ord_group_sync<HELPERS>(1, ncompute);  // the first run length (without helpers: also everyone's fetches, src[])
      ORD_PROF(cprof, 6);  // tile prologue (CSR acquire, first run length)
      ord_tile_runs<GL, KF, TASK, ZF, HELPERS>(a, smem, cc, T, tid, ncompute, w0, it, onehot);
      ORD_PROF(cprof, 15);
    }
    if (HELPERS) {  // (without helpers, the runs' last barrier and the one behind the next write-back do this)
      __syncthreads();  // tile T's slots are final, tile T+1's records have landed, tile T-1 is written back
      ORD_PROF(cprof, 7);   // compute side: waiting for the helpers
      ORD_PROF(hprof, 12);  // helper side: waiting for the compute warps
    }
  }
  if (NT > 0) ord_writeback<false, KC>(a, smem, cc, NT - 1, ltid, nlive);  // every thread still running
  if (tid == 0 && cc.k0) *a.w0 = w0;
  if (a.prof != nullptr && tid < 16) a.prof[tid] = reinterpret_cast<unsigned long long*>(smem + ORD_PROF_OFF)[tid];
}

// The two configurations.  Without helpers every thread of the CTA is a compute thread.
template <int GL, int KF, int TASK, int ZF = 0>
__device__ __forceinline__ void ordered_epoch_body(const OrderedArgs& a, unsigned char* smem) {
  ordered_epoch<GL, KF, TASK, ZF, false>(a, smem, blockDim.x, 0);
}
template <int GL, int KF, int TASK, int ZF = 0>
__device__ __forceinline__ void ordered_epoch_body_ws(const OrderedArgs& a, unsigned char* smem, int ncompute,
                                                      int nparked) {
  ordered_epoch<GL, KF, TASK, ZF, true>(a, smem, ncompute, nparked);
}

}  // namespace fmb
