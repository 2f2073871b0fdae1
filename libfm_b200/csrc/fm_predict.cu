// fm_predict.cu -- fp32 scoring / metric pass and small state kernels.
//
// fm_predict32_kernel replaces fm_learn::evaluate_regression / _classification
// (reference src/libfm/src/fm_learn.h:113-153) and fm_learn_sgd::predict
// (fm_learn_sgd.h:76-90) for the fp32 (HOGWILD) state: the same RowGroup score
// as the training kernel, metric sums accumulated in fp64 per block, per-block
// partials written in a fixed order (the host adds them in block order, so the
// result is a deterministic function of the launch geometry).
#include <algorithm>

#include "fm_rowgroup.cuh"
#include "fmb200_internal.h"

namespace fmb {

struct PredictArgs {
  const uint64_t* row_ptr;
  const uint32_t* col;
  const float* val;
  const float* target;
  uint64_t n_rows;
  const float* w0;
  const float* w;
  const float* v;
  int gp, ws, use_w0, use_w, task, transform;
  float min_target, max_target;
  double* out_pred;
  double* partials;
};

template <int G, int S, int R, int RW>
__global__ void __launch_bounds__(256) fm_predict32_kernel(const PredictArgs a) {
  using RG = RowGroup<G, S, R, RW>;
  constexpr int E = RG::E;
  constexpr int RPW = 32 / E;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nwarp = blockDim.x >> 5;
  const int lig = lane % E, c = lig % G, s = lig / G, sub = lane / E;
  const float4* V4 = reinterpret_cast<const float4*>(a.v);
  const float w0 = a.use_w0 ? *a.w0 : 0.f;
  double sq = 0, ab = 0, ok = 0;

  // contiguous chunk of rows per block, walked RPW rows per warp at a time
  const uint64_t per_block = (a.n_rows + gridDim.x - 1) / gridDim.x;
  const uint64_t b0 = (uint64_t)blockIdx.x * per_block;
  const uint64_t b1 = min(a.n_rows, b0 + per_block);
  for (uint64_t rbase = b0 + (uint64_t)warp * RPW; rbase < b1; rbase += (uint64_t)nwarp * RPW) {
    const uint64_t r = rbase + sub;
    const bool valid = r < b1;
    uint64_t beg = 0, end = 0;
    float y = 0.f;
    if (valid) {
      beg = __ldg(a.row_ptr + r);
      end = __ldg(a.row_ptr + r + 1);
      y = __ldg(a.target + r);
    }
    RG g;
    const float part = g.score(V4, a.w, a.gp, a.ws, a.use_w != 0, a.col + beg, a.val + beg, 0,
                               (int)(end - beg), c, s, lig);
    float p = w0 + part;
    if (valid && lig == 0) {
      if (a.task == FMB200_TASK_REGRESSION) {
        const float pc = fmaxf(a.min_target, fminf(a.max_target, p));
        const double err = (double)pc - (double)y;
        sq += err * err;
        ab += fabs(err);
        if (a.transform) p = pc;
      } else {
        if (((p >= 0.f) && (y >= 0.f)) || ((p < 0.f) && (y < 0.f))) ok += 1;
        if (a.transform) p = 1.f / (1.f + expf(-p));
      }
      if (a.out_pred != nullptr) a.out_pred[r] = (double)p;
    }
  }
  if (a.partials != nullptr) {
    sq = warp_sum_d(sq);
    ab = warp_sum_d(ab);
    ok = warp_sum_d(ok);
    __shared__ double s_part[8][3];
    if (lane == 0) {
      s_part[warp][0] = sq;
      s_part[warp][1] = ab;
      s_part[warp][2] = ok;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double x0 = 0, x1 = 0, x2 = 0;
      for (int i = 0; i < nwarp; i++) {
        x0 += s_part[i][0];
        x1 += s_part[i][1];
        x2 += s_part[i][2];
      }
      a.partials[3 * blockIdx.x + 0] = x0;
      a.partials[3 * blockIdx.x + 1] = x1;
      a.partials[3 * blockIdx.x + 2] = x2;
    }
  }
}

using PredictFn = void (*)(const PredictArgs);

// the (R, RW) of the training kernel's register-cache classes 0..2 (row_class): all of a row's
// gathers are in flight before the first is consumed
template <int G, int S>
static PredictFn pick_predict_r(int cls) {
  constexpr RowClass c0 = row_class(0, G), c1 = row_class(1, G), c2 = row_class(2, G);
  switch (cls) {
    case 0: return fm_predict32_kernel<G, S, c0.R, c0.RW>;
    case 1: return fm_predict32_kernel<G, S, c1.R, c1.RW>;
    default: return fm_predict32_kernel<G, S, c2.R, c2.RW>;
  }
}

cudaError_t launch_predict32(fmb200_ctx* c, const DataSlot& d, int transform, double* out_pred,
                             double* partials, int n_blocks) {
  if (c->kp / 4 > 32) return cudaErrorInvalidValue;
  int G, S, cls;
  pick_geometry(c->kp, d.n_rows, d.nnz, &G, &S, &cls);
  cls = std::clamp(cls, 0, 2);  // the training kernel's classes -1 and 3 are not instantiated here
  const PredictFn fn = dispatch_gs(G, S, [cls](auto g, auto s) { return pick_predict_r<g, s>(cls); });
  PredictArgs a;
  a.row_ptr = d.row_ptr.get();
  a.col = d.col.get();
  a.val = d.val.get();
  a.target = d.target.get();
  a.n_rows = d.n_rows;
  a.w0 = c->p32.w0();
  a.w = c->p32.w();
  a.v = c->p32.v();
  a.gp = c->kp / 4;
  a.ws = c->p32.ws;
  a.use_w0 = c->k0;
  a.use_w = c->k1;
  a.task = c->hp.task;
  a.transform = transform;
  a.min_target = (float)c->hp.min_target;
  a.max_target = (float)c->hp.max_target;
  a.out_pred = out_pred;
  a.partials = partials;
  fn<<<n_blocks, 256, 0, c->stream>>>(a);
  c->launches++;
  return cudaGetLastError();
}

// ---- state conversion --------------------------------------------------------
__global__ void p64_to_p32_kernel(Params64 s, Params32 d, uint32_t n, int k, int kp) {
  const uint64_t total = (uint64_t)n * kp;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total;
       i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t row = i / kp;
    const int f = (int)(i % kp);
    d.v()[i] = f < k ? (float)s.v()[row * k + f] : 0.f;
  }
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n;
       i += (uint64_t)gridDim.x * blockDim.x)
    d.w()[i * d.ws] = (float)s.w()[i];
  if (blockIdx.x == 0 && threadIdx.x == 0) d.w0()[0] = (float)s.w0()[0];
}

__global__ void p32_to_p64_kernel(Params32 s, Params64 d, uint32_t n, int k, int kp) {
  const uint64_t total = (uint64_t)n * k;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total;
       i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t row = i / k;
    const int f = (int)(i % k);
    d.v()[i] = (double)s.v()[row * kp + f];
  }
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n;
       i += (uint64_t)gridDim.x * blockDim.x)
    d.w()[i] = (double)s.w()[i * s.ws];
  if (blockIdx.x == 0 && threadIdx.x == 0) d.w0()[0] = (double)s.w0()[0];
}

__global__ void scale_kernel(float* p, uint64_t n, float f) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n;
       i += (uint64_t)gridDim.x * blockDim.x)
    p[i] *= f;
}

// occurrence histogram of the column ids + the largest id seen (ids >= n are
// counted nowhere: the caller rejects the data set when max id >= n).
// SMEM_BINS > 0: the table fits in shared memory (n <= SMEM_BINS): per-CTA private
// histogram, flushed once -- a few thousand counters under 2M increments would
// otherwise serialise at L2.
template <int SMEM_BINS>
__global__ void hist_kernel(const uint32_t* __restrict__ col, uint64_t nnz, uint32_t n,
                            unsigned int* cnt, unsigned int* out_max) {
  __shared__ unsigned int s_cnt[SMEM_BINS > 0 ? SMEM_BINS : 1];
  if (SMEM_BINS > 0) {
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) s_cnt[i] = 0u;
    __syncthreads();
  }
  unsigned int m = 0;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < nnz;
       i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t id = col[i];
    m = max(m, id);
    if (id < n) {
      if (SMEM_BINS > 0) atomicAdd(s_cnt + id, 1u);
      else atomicAdd(cnt + id, 1u);
    }
  }
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out_max, m);
  if (SMEM_BINS > 0) {
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
      const unsigned int v = s_cnt[i];
      if (v) atomicAdd(cnt + i, v);
    }
  }
}

// in place: uint32 counts -> float counts, and the maximum
__global__ void cnt_to_float_kernel(unsigned int* cnt, uint32_t n, unsigned int* out_max) {
  unsigned int m = 0;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n;
       i += (uint64_t)gridDim.x * blockDim.x) {
    const unsigned int v = cnt[i];
    m = max(m, v);
    reinterpret_cast<float*>(cnt)[i] = (float)v;
  }
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0) atomicMax(out_max, m);
}

// Structural check of the row offsets + the numbers the epoch launcher needs.
// out[0] = error bits (1: row_ptr[0] != 0, 2: not monotone, 4: row_ptr[n] != nnz, 8: row too long)
// out[1] = longest row; out[2..6] = worst 4-aligned entry span of any 32<<i row tile
__global__ void csr_inspect_kernel(const uint64_t* __restrict__ rp, uint64_t n_rows, uint64_t nnz,
                                   unsigned int* out) {
  unsigned int err = 0, longest = 0;
  unsigned int span[5] = {0, 0, 0, 0, 0};
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_rows;
       r += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t a = rp[r], b = rp[r + 1];
    if (b < a) err |= 2u;
    else if (b - a > 0xffffffffull) err |= 8u;
    else longest = max(longest, (unsigned int)(b - a));
    if ((r & 31) == 0) {
#pragma unroll
      for (int i = 0; i < 5; i++) {
        const uint64_t TR = 32ull << i;
        if ((r & (TR - 1)) == 0) {
          const uint64_t r1 = min(r + TR, n_rows);
          const uint64_t ab = a & ~3ull, ae = (rp[r1] + 3ull) & ~3ull;
          const uint64_t sp = ae >= ab ? ae - ab : 0;
          span[i] = max(span[i], sp > 0xffffffffull ? 0xffffffffu : (unsigned int)sp);
        }
      }
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    if (rp[0] != 0) err |= 1u;
    if (rp[n_rows] != nnz) err |= 4u;
  }
  if (err) atomicOr(out + 0, err);
  longest = __reduce_max_sync(0xffffffffu, longest);
  if ((threadIdx.x & 31) == 0 && longest) atomicMax(out + 1, longest);
#pragma unroll
  for (int i = 0; i < 5; i++) {
    const unsigned int m = __reduce_max_sync(0xffffffffu, span[i]);
    if ((threadIdx.x & 31) == 0 && m) atomicMax(out + 2 + i, m);
  }
}

cudaError_t launch_p64_to_p32(fmb200_ctx* c) {
  p64_to_p32_kernel<<<grid_for(c, (uint64_t)c->n * (c->kp + 1)), 256, 0, c->stream>>>(c->p64, c->p32,
                                                                               c->n, c->k, c->kp);
  c->launches++;
  return cudaGetLastError();
}

cudaError_t launch_p32_to_p64(fmb200_ctx* c) {
  p32_to_p64_kernel<<<grid_for(c, (uint64_t)c->n * (c->k + 1)), 256, 0, c->stream>>>(c->p32, c->p64,
                                                                              c->n, c->k, c->kp);
  c->launches++;
  return cudaGetLastError();
}

cudaError_t launch_scale_p32(fmb200_ctx* c, float factor) {
  scale_kernel<<<grid_for(c, c->p32.n_floats), 256, 0, c->stream>>>(c->p32.base, c->p32.n_floats,
                                                                   factor);
  c->launches++;
  return cudaGetLastError();
}

cudaError_t launch_csr_inspect(fmb200_ctx* c, cudaStream_t st, const uint64_t* rp, uint64_t n_rows, uint64_t nnz,
                               unsigned int* out8) {
  csr_inspect_kernel<<<grid_for(c, n_rows ? n_rows : 1), 256, 0, st>>>(rp, n_rows, nnz, out8);
  c->launches++;
  return cudaGetLastError();
}

cudaError_t launch_feature_counts(fmb200_ctx* c, cudaStream_t st, const uint32_t* col, uint64_t nnz, float* cnt,
                                  unsigned int* out_max_id, unsigned int* out_max) {
  unsigned int* u = reinterpret_cast<unsigned int*>(cnt);
  cudaError_t e = cudaMemsetAsync(u, 0, sizeof(unsigned int) * (size_t)c->n, st);
  if (e != cudaSuccess) return e;
  if (nnz > 0) {
    constexpr int BINS = 12288;  // 48 KB of static shared memory
    if (c->n <= (uint32_t)BINS) {
      const int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((nnz + 16383) / 16384, (uint64_t)c->sm_count));
      hist_kernel<BINS><<<grid, 1024, 0, st>>>(col, nnz, c->n, u, out_max_id);
    } else {
      hist_kernel<0><<<grid_for(c, nnz), 256, 0, st>>>(col, nnz, c->n, u, out_max_id);
    }
    c->launches++;
  }
  if (c->n > 0) {
    cnt_to_float_kernel<<<grid_for(c, c->n), 256, 0, st>>>(u, c->n, out_max);
    c->launches++;
  }
  return cudaGetLastError();
}

}  // namespace fmb
