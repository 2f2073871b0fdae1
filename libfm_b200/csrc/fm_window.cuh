// fm_window.cuh -- the pieces of the windowed HOGWILD epochs (fm_sgd_window.cu: reproducible SGD,
// fm_sgda_hogwild.cu: SGDA).  Each epoch is one cooperative launch over windows of rows (launch_windows, both
// epochs); a window's theta-phase adds its steps to the fixed-point accumulator (fm_hogwild_common.cuh) and stamps
// the features it touches in the one stamp table of fmb200_ctx::window (fmb200_internal.h: WindowBook, both epochs).
// The SGD epoch also appends each first touch to the window's list (window_touch) and, behind a grid barrier, folds
// the listed features into the fp32 state (window_fold), or, once a step overflowed, turns the whole state NaN
// (nan_state).  The SGDA epoch scans its stamps instead (fm_sgda_hogwild.cu says why).
//
// The kernels' argument structs hold these members under these names: state, acc (steps [n_floats], then the
// divergence flag), n_floats, off_w, off_v, ws, kp, use_w, stamp, stamp0, list, aux, gbar, gbar_base (launch_windows
// needs acc, stamp, stamp0, list, aux, gbar and gbar_base).
#pragma once
#include <algorithm>

#include "fm_device.cuh"
#include "fm_hogwild_common.cuh"
#include "fmb200_internal.h"

namespace fmb {

// A window's first touches: lane l holds feature `id` of a chunk of entries (`valid`: lane l has one).  A feature
// whose stamp is not yet the window's takes it and goes to the list, one reservation of *cnt per warp.
template <class A>
__device__ __forceinline__ void window_touch(const A& a, uint32_t stamp, unsigned long long* cnt, uint32_t id,
                                             bool valid, int lane) {
  const bool first = valid && __ldcg(a.stamp + id) != stamp && atomicExch(a.stamp + id, stamp) != stamp;
  const unsigned fm = __ballot_sync(0xffffffffu, first);
  if (fm) {
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(cnt, (unsigned long long)__popc(fm));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (first) a.list[base + __popc(fm & ((1u << lane) - 1u))] = id;
  }
}

// The fold of the n_listed features on the list, thread gt of GT: each feature's float4s of V (its padding has no
// steps and stays as it is), then its w: state += the accumulated steps, the steps back to zero.
template <class A>
__device__ __forceinline__ void window_fold(const A& a, uint64_t n_listed, uint64_t gt, uint64_t GT) {
  const uint32_t gp = (uint32_t)a.kp / 4, F = gp + 1;  // fold items of a feature
  const uint64_t n_items = n_listed * F;
  for (uint64_t t = gt; t < n_items; t += GT) {
    const uint32_t i = __ldcg(a.list + t / F);
    const uint32_t c = (uint32_t)(t % F);
    if (c < gp) {
      const uint64_t e = a.off_v + (uint64_t)i * a.kp + 4 * c;
      float4 x = __ldcg(reinterpret_cast<const float4*>(a.state + e));
      ulonglong2* ap = reinterpret_cast<ulonglong2*>(a.acc + e);
      const ulonglong2 u0 = __ldcg(ap), u1 = __ldcg(ap + 1);
      x.x = acc_fold(x.x, u0.x, false);
      x.y = acc_fold(x.y, u0.y, false);
      x.z = acc_fold(x.z, u1.x, false);
      x.w = acc_fold(x.w, u1.y, false);
      *reinterpret_cast<float4*>(a.state + e) = x;
      ap[0] = make_ulonglong2(0ull, 0ull);
      ap[1] = make_ulonglong2(0ull, 0ull);
    } else if (a.use_w) {
      const uint64_t e = a.off_w + (uint64_t)i * a.ws;
      a.state[e] = acc_fold(__ldcg(a.state + e), __ldcg(a.acc + e), false);
      a.acc[e] = 0ull;
    }
  }
}

// After a divergence: every element of the state NaN, its accumulated steps cleared (the flag stays)
template <class A>
__device__ __forceinline__ void nan_state(const A& a, uint64_t gt, uint64_t GT) {
  for (uint64_t e = gt; e < a.n_floats; e += GT) {
    a.state[e] = __int_as_float(0x7fffffff);
    a.acc[e] = 0ull;
  }
}

// One cooperative launch of a windowed epoch kernel fn(a): `threads` threads a CTA, as many CTAs on every SM as
// fit (fmb200_set_tuning's ctas_per_sm may take fewer), so the grid barriers find every CTA resident.  Fills in
// a's accumulator, stamps, list, count words and grid barrier, and moves the barrier count on by `barriers` per
// window and the stamp counter by the n_win windows.  *grid := the grid.
template <class A>
cudaError_t launch_windows(fmb200_ctx* c, void (*fn)(A), A& a, int threads, uint32_t n_win, uint32_t barriers,
                           int* grid) {
  WindowBook& w = c->window;
  cudaError_t e = acc_ready(c, &a.acc, nullptr);
  if (e != cudaSuccess) return e;
  if (!w.stamp) {
    const uint64_t n1 = std::max<uint32_t>(c->n, 1);
    if ((e = alloc(w.aux, 4)) != cudaSuccess || (e = alloc(w.list, n1)) != cudaSuccess ||
        (e = alloc(w.stamp, n1)) != cudaSuccess ||
        (e = cudaMemsetAsync(w.stamp.get(), 0, n1 * sizeof(uint32_t), c->stream)) != cudaSuccess) {
      w.stamp.reset();
      return e;
    }
  }
  if ((e = cudaMemsetAsync(w.aux.get(), 0, 4 * sizeof(unsigned long long), c->stream)) != cudaSuccess) return e;
  a.stamp = w.stamp.get();
  a.stamp0 = w.next;
  a.list = w.list.get();
  a.aux = w.aux.get();
  a.gbar = c->d_gbar.get();
  a.gbar_base = c->gbar_count;
  int occ = 0;
  if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, threads, 0)) != cudaSuccess) return e;
  if (occ < 1) return cudaErrorInvalidConfiguration;
  const int per_sm = c->tune_ctas_per_sm > 0 ? std::min(c->tune_ctas_per_sm, occ) : occ;
  *grid = c->sm_count * per_sm;
  void* args[] = {&a};
  if ((e = cudaLaunchCooperativeKernel((const void*)fn, dim3(*grid), dim3(threads), args, 0, c->stream)) != cudaSuccess)
    return e;
  c->launches++;
  c->gbar_count += (uint32_t)*grid * barriers * n_win;
  w.next += n_win;
  return cudaSuccess;
}

}  // namespace fmb
