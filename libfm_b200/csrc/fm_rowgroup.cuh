// fm_rowgroup.cuh -- the sub-warp "row group" used by the fp32 kernels.
//
// One training example (one CSR row) is handled by E = G*S lanes of a warp:
//   G lanes span one factor row V[id,:] as G float4 chunks (kp = 4*gp floats,
//     gp <= G; lanes with c >= gp idle when kp/4 is not a power of two),
//   S "slots" walk the row's non-zeros S at a time.
// A warp therefore processes 32/E examples at once (k=64, 39 nnz/row: G=16, S=2,
// one example per warp, two factor rows = four 128-byte lines per LDG.128).
//
// Two access patterns live side by side because the SM pays a floor per memory
// instruction no matter how few sectors it touches:
//   * factor rows V[id,:]  -- chunk-parallel: lane (s,c) owns chunk c of the entries
//     s, s+S, ...; the first R chunks stay in registers for the write-back.
//   * linear weights w[id] -- ENTRY-parallel: lane l of the group owns the entries
//     l, l+E, ...: one warp-wide load / reduction covers E entries instead of one
//     instruction per entry with a single active lane.
// The work is split in phases so a caller can put several rows' gathers in flight
// before consuming any of them:
//   gather()  issues the loads (first R factor chunks and first RW weights per lane),
//   reduce()  restates fm_model::predict (reference src/fm_core/fm_model.h:105-127)
//             in fp32 with the O(k*nnz) trick: per-lane partial sums, segmented
//             __shfl_xor reductions over the slot bits (per-factor sums) and then
//             over the whole group (scalar score).
#pragma once
#include "fm_device.cuh"

namespace fmb {

template <int G, int S, int R, int RW>
struct RowGroup {
  static constexpr int E = G * S;
  static_assert(E <= 32 && (E & (E - 1)) == 0, "group must be a power-of-two slice of a warp");

  float4 acc;     // per-factor sums s_f for this lane's 4 factors (complete after reduce())
  float4 vc[R];   // cached factor chunks of the entries s, s+S, ... (zero when inactive)
  float wc[RW];   // cached linear weights of the entries lig, lig+E, ... (entry-parallel)
  int beg, end;   // this row's entries: [beg, end) in the id / value arrays
  int maxit;      // warp-uniform trip count of the chunk loop
  int maxwit;     // warp-uniform trip count of the entry-parallel loop
  float hrow;     // (WANT_H) curvature of the score w.r.t. all of this row's w/V blocks

  template <typename IdPtr, typename ValPtr>
  __device__ __forceinline__ void gather(const float4* __restrict__ V4,
                                         const float* __restrict__ w, int gp, int ws,
                                         bool use_w, IdPtr ids, ValPtr xs, int beg_, int end_,
                                         int c, int s, int lig) {
    beg = beg_;
    end = end_;
    const bool chunk_on = c < gp;
#pragma unroll
    for (int it = 0; it < R; ++it) {
      const int j = beg + s + it * S;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (j < end && chunk_on) v = ld_cg_f4(V4 + (size_t)ids[j] * gp + c);
      vc[it] = v;
    }
#pragma unroll
    for (int t = 0; t < RW; ++t) {
      const int j = beg + lig + t * E;
      wc[t] = (use_w && j < end) ? ld_cg_f(w + (size_t)ids[j] * ws) : 0.f;
    }
  }

  // Returns the score WITHOUT the bias term, replicated in all E lanes.
  // WANT_H additionally fills hrow = sum_i |d score / d (w_i, V_i)|^2, evaluated with
  // the one-hot identity  A*k1 + (A-2)*sum_f s_f^2 + sum_f sum_i (v_if x_i)^2,
  // A = sum_i x_i^2  (exact for x in {0,1}, a damping heuristic otherwise).
  template <bool WANT_H, typename IdPtr, typename ValPtr>
  __device__ __forceinline__ float reduce(const float4* __restrict__ V4,
                                          const float* __restrict__ w, int gp, int ws,
                                          bool use_w, IdPtr ids, ValPtr xs, int c, int s,
                                          int lig) {
    acc = make_float4(0.f, 0.f, 0.f, 0.f);
    float sq = 0.f, lin = 0.f, xx = 0.f;
    const int cnt = end - beg;
    maxit = __reduce_max_sync(0xffffffffu, (cnt + S - 1) / S);
    maxwit = __reduce_max_sync(0xffffffffu, (cnt + E - 1) / E);
    // ---- factor rows, chunk-parallel ----
#pragma unroll
    for (int it = 0; it < R; ++it) {
      const int j = beg + s + it * S;
      accumulate(vc[it], j < end ? xs[j] : 0.f, sq);
    }
    const bool chunk_on = c < gp;
    for (int it = R; it < maxit; ++it) {
      const int j = beg + s + it * S;
      if (j < end) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (chunk_on) v = ld_cg_f4(V4 + (size_t)ids[j] * gp + c);
        accumulate(v, xs[j], sq);
      }
    }
    // ---- linear weights, entry-parallel ----
#pragma unroll
    for (int t = 0; t < RW; ++t) {
      const int j = beg + lig + t * E;
      if (j < end) {
        const float x = xs[j];
        lin += wc[t] * x;
        if (WANT_H) xx += x * x;
      }
    }
    for (int t = RW; t < maxwit; ++t) {
      const int j = beg + lig + t * E;
      if (j < end) {
        const float x = xs[j];
        if (use_w) lin += ld_cg_f(w + (size_t)ids[j] * ws) * x;
        if (WANT_H) xx += x * x;
      }
    }
    // per-factor sums: reduce over the slot bits (lane strides G, 2G, ... < E)
#pragma unroll
    for (int o = G; o < E; o <<= 1) {
      acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o);
      acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
      acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o);
      acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
    }
    // 0.5*(sum_f^2 - sumsq_f): the square term once per chunk (slot 0), the
    // rest from every lane; then reduce the scalar over the whole group
    float part = lin - 0.5f * sq;
    float s2 = 0.f;
    if (s == 0) {
      s2 = acc.x * acc.x + acc.y * acc.y + acc.z * acc.z + acc.w * acc.w;
      part += 0.5f * s2;
    }
#pragma unroll
    for (int o = 1; o < E; o <<= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (WANT_H) {
#pragma unroll
      for (int o = 1; o < E; o <<= 1) {
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
        sq += __shfl_xor_sync(0xffffffffu, sq, o);
        xx += __shfl_xor_sync(0xffffffffu, xx, o);
      }
      hrow = (use_w ? xx : 0.f) + fmaxf((xx - 2.f) * s2 + sq, 0.f);
    }
    return part;
  }

  // gather + reduce in one go (scoring kernels)
  template <typename IdPtr, typename ValPtr>
  __device__ __forceinline__ float score(const float4* __restrict__ V4,
                                         const float* __restrict__ w, int gp, int ws,
                                         bool use_w, IdPtr ids, ValPtr xs, int beg_, int end_,
                                         int c, int s, int lig) {
    gather(V4, w, gp, ws, use_w, ids, xs, beg_, end_, c, s, lig);
    return reduce<false>(V4, w, gp, ws, use_w, ids, xs, c, s, lig);
  }

  __device__ __forceinline__ void accumulate(const float4& v, float x, float& sq) {
    const float dx = v.x * x, dy = v.y * x, dz = v.z * x, dw = v.w * x;
    acc.x += dx;
    acc.y += dy;
    acc.z += dz;
    acc.w += dw;
    sq += dx * dx + dy * dy + dz * dz + dw * dw;
  }
};

}  // namespace fmb
