// fm_peer.cu -- parameter averaging over NVLink peer memory (the per-epoch exchange of
// the row-sharded multi-GPU path, SURVEY.md section 8e), without NCCL.
//
// The packed fp32 state of C2 is 0.6 MB: an NCCL all-reduce of that size is pure
// latency (~50 us measured next to an ~80 us epoch).  Every rank instead maps the
// peers' state buffers (CUDA IPC across processes, plain peer access inside one
// process) and ONE kernel per rank does a one-shot all-reduce:
//
//   1. signal: write this epoch's sequence number into slot [self] of every peer's
//      flag block (st.release.sys over NVLink),
//   2. wait until the own flag block shows the sequence number for all ranks
//      (ld.acquire.sys) -- every peer's epoch kernel has then finished (stream order
//      on the peer) and its state buffer `cur` is final,
//   3. read all G `cur` buffers (peer loads travel NVLink) in rank order -- the same
//      order on every rank, so all replicas end bit-identical -- and write the mean
//      into the LOCAL `next` buffer.
//
// The context then swaps cur/next.  Double buffering removes the second barrier: a
// slow peer may still read our old `cur` while we already train into `next`; the old
// buffer is only overwritten by the NEXT averaging kernel, after that kernel's
// barrier has proven that every peer finished this one.
#include <algorithm>

#include "fmb200_internal.h"

namespace fmb {

__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

struct PeerArgs {
  unsigned int* flags[FMB200_MAX_PEERS];  // flag block of every rank (mapped)
  const float4* cur[FMB200_MAX_PEERS];    // current state buffer of every rank (mapped)
  float4* next_local;
  int world, rank;
  unsigned int seq;
  uint64_t n_vec;  // float4 elements
  float inv_world;
};

__global__ void __launch_bounds__(256) fm_peer_mean_kernel(const PeerArgs a) {
  if (blockIdx.x == 0 && threadIdx.x < a.world) st_release_sys(a.flags[threadIdx.x] + COMM_SEQ_WORD + a.rank, a.seq);
  if (threadIdx.x < a.world) {
    const unsigned int* mine = a.flags[a.rank] + COMM_SEQ_WORD + threadIdx.x;
    while ((int)(ld_acquire_sys(mine) - a.seq) < 0) {
    }
  }
  __syncthreads();
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < a.n_vec;
       i += (uint64_t)gridDim.x * blockDim.x) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int q0 = 0; q0 < a.world; q0 += 8) {  // 8 independent peer loads at a time, summed in rank order
      float4 v[8];
#pragma unroll
      for (int u = 0; u < 8; u++)
        v[u] = (q0 + u < a.world) ? __ldcv(a.cur[q0 + u] + i) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < 8; u++) {
        if (q0 + u < a.world) {
          s.x += v[u].x;
          s.y += v[u].y;
          s.z += v[u].z;
          s.w += v[u].w;
        }
      }
    }
    s.x *= a.inv_world;
    s.y *= a.inv_world;
    s.z *= a.inv_world;
    s.w *= a.inv_world;
    a.next_local[i] = s;
  }
}

// ---------------------------------------------------------------------------------------
// Mean-field combine.  Averaging G replicas that each saw N/G rows advances the model by
// about one G-th of an epoch (scripts/study_shard_combine.py: test RMSE after epoch 1 at
// G = 8 is 0.86 against 0.67 for one sequential stream).  The exchange therefore forms
//     theta = theta0 + gamma_i * sum_g (theta_g - theta0)
// per parameter, with gamma_i the factor that makes G summed shard-steps of relative size
// s_i equal to G such steps taken one after the other on a quadratic,
//     gamma_i = (1 - (1 - s_i)^G) / (G s_i),   1 - s_i = exp(-u_i),   u_i = lr (h_i + reg) c_i,
// c_i = the feature's mean occurrence count per shard, h_i = 1 for w0 / w, the mean squared
// factor-row norm of theta0 for V -- the closed form the HOGWILD kernels use inside one GPU
// (fm_hogwild_common.cuh: gamma_scale), applied across GPUs.  A parameter its shard-epoch has
// already converged (the bias, hot features: s -> 1) is averaged, one that was barely touched
// (s -> 0) is summed.
//
// Same one-shot structure as fm_peer_mean_kernel.  Additional state behind the two state
// buffers of the comm block: `base` = theta0 (rewritten here with the new theta), `cnt` = this
// rank's per-feature counts (peers read them), `part` = per-block partial sums of |V|^2 of the
// theta this kernel writes (fixed-order reduction: every rank derives the SAME h for the next
// exchange, so the replicas stay bit-identical).
struct MeanFieldArgs {
  PeerArgs p;
  float4* base_local;              // theta0 in, theta out
  const float* cnt[FMB200_MAX_PEERS];
  float* cntm;                     // local: the features' mean count per shard (fm_peer_counts_mean_kernel)
  const float* part_in;            // [n_part] partial sums of |V|^2 of theta0
  float* part_out;                 // [gridDim.x]
  int n_part;
  uint64_t off_w, off_v;           // in floats
  int ws, kp;
  uint32_t n;
  float lr, regw, regv, reg0;
};

__device__ __forceinline__ float mf_gamma(float u, float G) {
  // (1 - exp(-G u)) / (G (1 - exp(-u))); -> 1 as u -> 0, -> 1/G as u -> inf
  if (!(u > 1e-6f)) return 1.f;
  const float a = -expm1f(-G * u), b = -expm1f(-u);
  return a / (G * b);
}

// header of both mean-field kernels: the leading barrier, h_V from the previous exchange's partials
// (fixed order: identical in every block of every rank), the bias' gamma.  Returns (hv, g0).
__device__ __forceinline__ void mf_barrier(const PeerArgs& p) {
  if (blockIdx.x == 0 && threadIdx.x < p.world) st_release_sys(p.flags[threadIdx.x] + COMM_SEQ_WORD + p.rank, p.seq);
  if (threadIdx.x < p.world) {
    const unsigned int* mine = p.flags[p.rank] + COMM_SEQ_WORD + threadIdx.x;
    while ((int)(ld_acquire_sys(mine) - p.seq) < 0) {
    }
  }
  __syncthreads();
}

// First kernel of a mean-field exchange: the cross-GPU barrier, then every feature's mean count per shard into a
// LOCAL table.  The combine kernels read that table; fetching the G counts per state element from the peers
// again (16 peer loads per k = 8 factor row at G = 8, as many as the state itself) made the C2 exchange 65 us at
// N = 8 (r02 8-GPU run).
__global__ void __launch_bounds__(256) fm_peer_counts_mean_kernel(const MeanFieldArgs a) {
  const PeerArgs& p = a.p;
  mf_barrier(p);
  const float G = (float)p.world;
  if (blockIdx.x == 0) {  // rows per shard (the peers' row-count words of this parity), averaged in rank order
    __shared__ unsigned int s_rows[FMB200_MAX_PEERS];
    if ((int)threadIdx.x < p.world)
      s_rows[threadIdx.x] =
          __ldcv(p.flags[threadIdx.x] + COMM_ROWS_WORD + COMM_ROWS_PARITY_STRIDE * (p.seq & 1u) + threadIdx.x);
    __syncthreads();
    if (threadIdx.x == 0) {
      float rows = 0.f;
      for (int q = 0; q < p.world; q++) rows += (float)s_rows[q];
      p.flags[p.rank][COMM_MEAN_ROWS_WORD + (p.seq & 1u)] = __float_as_uint(rows / G);
    }
  }
  for (uint64_t f = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; f < a.n; f += (uint64_t)gridDim.x * blockDim.x) {
    float c = 0.f;
    for (int q0 = 0; q0 < p.world; q0 += 8) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; u++) v[u] = (q0 + u < p.world) ? __ldcv(a.cnt[q0 + u] + f) : 0.f;
#pragma unroll
      for (int u = 0; u < 8; u++) c += v[u];  // (rank order; absent ranks add an exact 0)
    }
    a.cntm[f] = c / G;
  }
}

// (the barrier has been passed by fm_peer_counts_mean_kernel, in front of this kernel in the stream)
__device__ __forceinline__ void mf_prologue(const MeanFieldArgs& a, float* s_red, float* hv_out, float* g0_out) {
  const PeerArgs& p = a.p;
  const float G = (float)p.world;
  float acc = 0.f;
  for (int i = threadIdx.x; i < a.n_part; i += 256) acc += a.part_in[i];
  s_red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
    __syncthreads();
  }
  *hv_out = a.n ? s_red[0] / (float)a.n : 0.f;
  __syncthreads();
  // mean rows per shard: left in the LOCAL header by fm_peer_counts_mean_kernel (a loop over the peers' words
  // here was 8 NVLink round trips, one after the other, in every block's prologue at G = 8)
  const float rows = __uint_as_float(__ldcv(p.flags[p.rank] + COMM_MEAN_ROWS_WORD + (p.seq & 1u)));
  *g0_out = mf_gamma(a.lr * (1.f + a.reg0) * rows, G);
}

// the combined value of float4 element i (the same arithmetic, in the same order, in both kernels)
__device__ __forceinline__ float4 mf_combine(const MeanFieldArgs& a, uint64_t i, float hv, float g0, float* sq) {
  const PeerArgs& p = a.p;
  const float G = (float)p.world;
  const float4 b4 = a.base_local[i];
  float b[4] = {b4.x, b4.y, b4.z, b4.w};
  float d[4] = {0.f, 0.f, 0.f, 0.f};
  // the replicas' elements in batches of 8 INDEPENDENT peer loads (a loop over a runtime world size issues
  // one NVLink round trip after the other: 8 x ~2 us per element at G = 8), summed in rank order
  for (int q0 = 0; q0 < p.world; q0 += 8) {
    float4 v[8];
#pragma unroll
    for (int u = 0; u < 8; u++)
      v[u] = (q0 + u < p.world) ? __ldcv(p.cur[q0 + u] + i) : b4;  // never from a stale L1 line
#pragma unroll
    for (int u = 0; u < 8; u++) {
      if (q0 + u < p.world) {
        d[0] += v[u].x - b[0];
        d[1] += v[u].y - b[1];
        d[2] += v[u].z - b[2];
        d[3] += v[u].w - b[3];
      }
    }
  }
  const uint64_t e0 = i * 4;
  float g[4];
  if (e0 < a.off_w) {  // the bias, then padding up to w: zero in every replica, and zero it stays
    g[0] = e0 == 0 ? g0 : 0.f;
    g[1] = g[2] = g[3] = 0.f;
  } else if (e0 < a.off_v) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const uint64_t rel = e0 + j - a.off_w;
      const uint64_t f = rel / a.ws;
      g[j] = 0.f;
      if (rel % a.ws == 0 && f < a.n) g[j] = mf_gamma(a.lr * (1.f + a.regw) * a.cntm[f], G);
    }
  } else {
    const uint64_t f = (e0 - a.off_v) / a.kp;  // kp is a multiple of 4: one row per float4
    float gv = 0.f;
    if (f < a.n) gv = mf_gamma(a.lr * (hv + a.regv) * a.cntm[f], G);
    g[0] = g[1] = g[2] = g[3] = gv;
  }
  float4 o;
  o.x = b[0] + g[0] * d[0];
  o.y = b[1] + g[1] * d[1];
  o.z = b[2] + g[2] * d[2];
  o.w = b[3] + g[3] * d[3];
  if (e0 >= a.off_v) *sq += o.x * o.x + o.y * o.y + o.z * o.z + o.w * o.w;
  return o;
}

__device__ __forceinline__ float mf_block_sum(float v, float* s_red) {
  s_red[threadIdx.x] = v;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
    __syncthreads();
  }
  return s_red[0];
}

// one-shot: every rank reads all G replicas whole and keeps the combination (small state: one barrier,
// G x state bytes over NVLink per rank)
__global__ void __launch_bounds__(256) fm_peer_meanfield_kernel(const MeanFieldArgs a) {
  const PeerArgs& p = a.p;
  __shared__ float s_red[256];
  float hv, g0;
  mf_prologue(a, s_red, &hv, &g0);
  float sq = 0.f;  // |V|^2 of what this thread writes
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < p.n_vec;
       i += (uint64_t)gridDim.x * blockDim.x) {
    const float4 o = mf_combine(a, i, hv, g0, &sq);
    p.next_local[i] = o;
    a.base_local[i] = o;
  }
  const float tot = mf_block_sum(sq, s_red);
  if (threadIdx.x == 0) a.part_out[blockIdx.x] = tot;
}

// sliced (reduce-scatter + all-gather in one kernel): rank r combines only slice r of the state -- reading
// that slice from all G replicas -- and PUSHES the result into every rank's `next` and theta0 buffers
// (st over NVLink), the |V|^2 partials of its slice into every rank's partial table.  2 (G-1)/G x state
// bytes over NVLink per rank instead of (G-1) x; the C5-sized state (516 MB, G = 8) moves 0.9 GB per rank
// instead of 3.6 GB.  The pushes must have landed everywhere before any rank trains on: the launcher puts
// fm_peer_barrier_kernel behind this kernel (stream order = this kernel's stores are performed).
struct MeanFieldPush {
  float4* next[FMB200_MAX_PEERS];
  float4* base[FMB200_MAX_PEERS];
  float* part[FMB200_MAX_PEERS];
};
__global__ void __launch_bounds__(256) fm_peer_meanfield_sliced_kernel(const MeanFieldArgs a, const MeanFieldPush t) {
  const PeerArgs& p = a.p;
  __shared__ float s_red[256];
  float hv, g0;
  mf_prologue(a, s_red, &hv, &g0);
  const uint64_t per = (p.n_vec + (uint64_t)p.world - 1) / (uint64_t)p.world;
  const uint64_t lo = min(p.n_vec, per * (uint64_t)p.rank), hi = min(p.n_vec, lo + per);
  float sq = 0.f;
  for (uint64_t i = lo + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < hi;
       i += (uint64_t)gridDim.x * blockDim.x) {
    const float4 o = mf_combine(a, i, hv, g0, &sq);
    for (int q = 0; q < p.world; q++) {
      t.next[q][i] = o;
      t.base[q][i] = o;
    }
  }
  const float tot = mf_block_sum(sq, s_red);
  if ((int)threadIdx.x < p.world) t.part[threadIdx.x][(size_t)p.rank * gridDim.x + blockIdx.x] = tot;
}

// theta0 := the current state, its |V|^2 partials, this rank's counts and row count into the
// comm block (before the FIRST epoch after an attach / set_params)
__global__ void __launch_bounds__(256) fm_peer_capture_kernel(const float4* cur, float4* base, uint64_t n_vec,
                                                              uint64_t off_v4, float* part_out) {
  __shared__ float s_red[256];
  float sq = 0.f;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_vec;
       i += (uint64_t)gridDim.x * blockDim.x) {
    const float4 v = cur[i];
    base[i] = v;
    if (i >= off_v4) sq += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  s_red[threadIdx.x] = sq;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) part_out[blockIdx.x] = s_red[0];
}

__global__ void fm_peer_counts_kernel(const float* __restrict__ src, float* __restrict__ dst, uint32_t n,
                                      unsigned int* rows_word, unsigned int rows) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    dst[i] = src[i];
  if (blockIdx.x == 0 && threadIdx.x == 0) *rows_word = rows;
}

// Cross-GPU barrier on the stream (no data): same signal / wait through the peers' flag
// blocks, on its own flag row and sequence so it never interferes with the averaging.
__global__ void fm_peer_barrier_kernel(const PeerArgs a) {
  if (threadIdx.x < a.world) {
    st_release_sys(a.flags[threadIdx.x] + COMM_BAR_WORD + a.rank, a.seq);
    const unsigned int* mine = a.flags[a.rank] + COMM_BAR_WORD + threadIdx.x;
    while ((int)(ld_acquire_sys(mine) - a.seq) < 0) {
    }
  }
}

// Load every kernel of the exchange NOW (called when peers are attached).  With CUDA's lazy module loading
// the first launch of a kernel may have to synchronise the context; if that happens while an exchange kernel
// of this process is already spinning on a peer's flag -- and the peer's kernel is the one still to be
// launched -- the process deadlocks (seen with two contexts in one process: sliced combine running, the
// barrier kernel behind it never launched before).
cudaError_t peer_preload_kernels() {
  cudaFuncAttributes fa;
  cudaError_t e;
  if ((e = cudaFuncGetAttributes(&fa, fm_peer_mean_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&fa, fm_peer_meanfield_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&fa, fm_peer_meanfield_sliced_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&fa, fm_peer_counts_mean_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&fa, fm_peer_capture_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&fa, fm_peer_counts_kernel)) != cudaSuccess) return e;
  return cudaFuncGetAttributes(&fa, fm_peer_barrier_kernel);
}

cudaError_t launch_peer_barrier(fmb200_ctx* c) {
  PeerArgs a;
  for (int q = 0; q < c->peer_world; q++) a.flags[q] = CommLayout::words(c->peer_base[q]);
  a.world = c->peer_world;
  a.rank = c->peer_rank;
  a.seq = ++c->peer_bar_seq;
  fm_peer_barrier_kernel<<<1, 32, 0, c->stream>>>(a);
  c->launches++;
  return cudaGetLastError();
}

static int peer_grid(const fmb200_ctx* c, uint64_t n_vec) {
  return (int)std::max<uint64_t>(1, std::min<uint64_t>((n_vec + 255) / 256, (uint64_t)c->sm_count * 2));
}

// called in front of a HOGWILD epoch when peers are attached: theta0 and the shard's counts
cudaError_t peer_before_epoch(fmb200_ctx* c, const DataSlot& d) {
  if (c->peer_world <= 1) return cudaSuccess;
  const CommLayout& L = c->comm;
  unsigned char* self = c->comm_base.get();
  const uint64_t n_vec = (c->p32.n_floats + 3) / 4;
  if (!c->peer_base_valid) {
    const int grid = peer_grid(c, n_vec);
    fm_peer_capture_kernel<<<grid, 256, 0, c->stream>>>(reinterpret_cast<const float4*>(c->p32.base),
                                                        reinterpret_cast<float4*>(L.theta0(self)), n_vec,
                                                        c->p32.off_v / 4, L.partials(self, c->peer_part_cur));
    c->peer_n_part = grid;
    c->peer_base_valid = true;
    c->launches++;
  }
  // the shard's counts for the exchange behind this epoch, into the table of that exchange's parity -- unless
  // that table already holds this very upload (every upload of a context has its own generation number)
  const unsigned parity = (c->peer_seq + 1u) & 1u;
  if (c->n > 0 && d.feat_cnt != nullptr && c->peer_cnt_stamp[parity] != d.upload_gen) {
    const int grid = (int)std::max<uint32_t>(1, std::min<uint32_t>((c->n + 255) / 256, 64));
    fm_peer_counts_kernel<<<grid, 256, 0, c->stream>>>(d.feat_cnt.get(), L.counts(self, parity), c->n,
                                                       L.rows_word(self, parity, c->peer_rank), (unsigned int)d.n_rows);
    c->launches++;
    c->peer_cnt_stamp[parity] = d.upload_gen;
  }
  return cudaGetLastError();
}

// the exchange reads every rank's state buffer `cur` and leaves the result in the buffers `cur ^ 1`
static void peer_swap(fmb200_ctx* c) {
  c->peer_cur ^= 1;
  c->p32.base = c->comm.buf(c->comm_base.get(), c->peer_cur);
}

cudaError_t launch_peer_meanfield(fmb200_ctx* c) {
  const CommLayout& L = c->comm;
  unsigned char* self = c->comm_base.get();
  MeanFieldArgs a;
  const int cur = c->peer_cur;
  for (int q = 0; q < c->peer_world; q++) {
    a.p.flags[q] = CommLayout::words(c->peer_base[q]);
    a.p.cur[q] = reinterpret_cast<const float4*>(L.buf(c->peer_base[q], cur));
    a.cnt[q] = L.counts(c->peer_base[q], (c->peer_seq + 1u) & 1u);
  }
  a.p.next_local = reinterpret_cast<float4*>(L.buf(self, cur ^ 1));
  a.p.world = c->peer_world;
  a.p.rank = c->peer_rank;
  a.p.seq = ++c->peer_seq;
  a.p.n_vec = (c->p32.n_floats + 3) / 4;
  a.p.inv_world = 1.f / (float)c->peer_world;
  a.base_local = reinterpret_cast<float4*>(L.theta0(self));
  a.cntm = L.mean_counts(self);
  a.part_in = L.partials(self, c->peer_part_cur);
  a.part_out = L.partials(self, c->peer_part_cur ^ 1);
  a.n_part = c->peer_n_part;
  a.off_w = c->p32.off_w;
  a.off_v = c->p32.off_v;
  a.ws = c->p32.ws;
  a.kp = c->kp;
  a.n = c->n;
  a.lr = (float)c->hp.lr;
  a.reg0 = (float)c->hp.reg0;
  a.regw = (float)c->hp.regw;
  a.regv = (float)c->hp.regv;
  {  // the barrier + the local table of mean counts
    const int grid = (int)std::max<uint32_t>(1, std::min<uint32_t>((c->n + 255) / 256, (uint32_t)c->sm_count));
    fm_peer_counts_mean_kernel<<<grid, 256, 0, c->stream>>>(a);
    c->launches++;
  }
  // small state: one-shot; large state: sliced (1/G of the reads; + a trailing barrier)
  bool sliced = a.p.n_vec * 16ull >= (8ull << 20);
  if (c->tune_variant == 8) sliced = true;
  if (c->tune_variant == 9) sliced = false;
  if (sliced) {
    MeanFieldPush t;
    for (int q = 0; q < c->peer_world; q++) {
      t.next[q] = reinterpret_cast<float4*>(L.buf(c->peer_base[q], cur ^ 1));
      t.base[q] = reinterpret_cast<float4*>(L.theta0(c->peer_base[q]));
      t.part[q] = L.partials(c->peer_base[q], c->peer_part_cur ^ 1);
    }
    const uint64_t per = (a.p.n_vec + c->peer_world - 1) / c->peer_world;
    const int grid = std::min(peer_grid(c, per), FMB_PEER_PART / c->peer_world);
    fm_peer_meanfield_sliced_kernel<<<grid, 256, 0, c->stream>>>(a, t);
    c->launches++;
    c->peer_n_part = grid * c->peer_world;
    cudaError_t e = launch_peer_barrier(c);
    if (e != cudaSuccess) return e;
  } else {
    const int grid = peer_grid(c, a.p.n_vec);
    fm_peer_meanfield_kernel<<<grid, 256, 0, c->stream>>>(a);
    c->launches++;
    c->peer_n_part = grid;
  }
  c->peer_part_cur ^= 1;
  peer_swap(c);
  return cudaGetLastError();
}

cudaError_t launch_peer_mean(fmb200_ctx* c) {
  const CommLayout& L = c->comm;
  PeerArgs a;
  const int cur = c->peer_cur;
  for (int q = 0; q < c->peer_world; q++) {
    a.flags[q] = CommLayout::words(c->peer_base[q]);
    a.cur[q] = reinterpret_cast<const float4*>(L.buf(c->peer_base[q], cur));
  }
  a.next_local = reinterpret_cast<float4*>(L.buf(c->comm_base.get(), cur ^ 1));
  a.world = c->peer_world;
  a.rank = c->peer_rank;
  a.seq = ++c->peer_seq;
  a.n_vec = (c->p32.n_floats + 3) / 4;
  a.inv_world = 1.f / (float)c->peer_world;
  const int grid = peer_grid(c, a.n_vec);
  fm_peer_mean_kernel<<<grid, 256, 0, c->stream>>>(a);
  c->launches++;
  peer_swap(c);
  c->peer_base_valid = false;  // theta0 of the mean-field combine no longer matches
  return cudaGetLastError();
}

}  // namespace fmb
