// fmb200_internal.h -- context layout and kernel launch entry points shared by
// the translation units of libfmb200.so.  Not part of the public ABI.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/fmb200.h"
#include "fm_sgda_plan.h"

namespace fmb {

// Owning handles: every device buffer, pinned host buffer and event of a context is released by
// its owner's destructor.  Kernel argument structs keep raw pointers (they are copied to the device).
struct CudaFree {
  void operator()(void* p) const { cudaFree(p); }
};
struct CudaFreeHost {
  void operator()(void* p) const { cudaFreeHost(p); }
};
struct CudaEventDestroy {
  void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
};
template <class T>
using DevPtr = std::unique_ptr<T, CudaFree>;
template <class T>
using HostPtr = std::unique_ptr<T, CudaFreeHost>;
using EventPtr = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, CudaEventDestroy>;

// p := a fresh device buffer of n elements (at least one); what p held is released first
template <class T>
cudaError_t alloc(DevPtr<T>& p, uint64_t n) {
  p.reset();
  T* raw = nullptr;
  const cudaError_t e = cudaMalloc(&raw, (n ? n : 1) * sizeof(T));
  p.reset(raw);
  return e;
}

// p := a fresh pinned host buffer of n elements
template <class T>
cudaError_t host_alloc(HostPtr<T>& p, size_t n) {
  p.reset();
  T* raw = nullptr;
  const cudaError_t e = cudaHostAlloc((void**)&raw, n * sizeof(T), cudaHostAllocDefault);
  p.reset(raw);
  return e;
}

inline cudaError_t event_create(EventPtr& p, unsigned int flags) {
  cudaEvent_t raw = nullptr;
  const cudaError_t e = cudaEventCreateWithFlags(&raw, flags);
  p.reset(raw);
  return e;
}

// Grow-on-demand scratch: make p hold at least n elements, cap = what it holds.  Contents are not kept.
template <class T, class Cap>
cudaError_t grow(DevPtr<T>& p, Cap& cap, uint64_t n) {
  if (p && cap >= n) return cudaSuccess;
  cap = 0;
  const cudaError_t e = alloc(p, n);
  if (e == cudaSuccess) cap = (Cap)n;
  return e;
}

// slack (in elements) behind every per-row and per-entry array of a slot (the CSR arrays and the
// ORDERED index) so that whole-tile TMA bulk copies of the last tile stay inside the allocation
constexpr uint64_t kRowSlack = 512 + 8;
constexpr uint64_t kEntrySlack = 16;

// The dealt copy of a data set for the row-lane epoch's dealt schedule (fm_deal.cu): the rows of every
// window of grid x tr rows stably sorted by the id of their last entry; pos[i] = dealt row i's position
// inside its window in file order.  Built for upload generation `gen`.
struct RowlaneDeal {
  DevPtr<uint64_t> row_ptr;  // [rows_cap + 1]
  DevPtr<uint32_t> col, pos;
  DevPtr<float> val, target;
  uint64_t rows_cap = 0, nnz_cap = 0;
  uint64_t gen = 0;
  int tr = 0;
  uint32_t grid = 0;
  DevPtr<unsigned char> scratch;  // the sort's keys, values and temporary storage
  size_t scratch_bytes = 0;
  bool matches(uint64_t g, int t, uint32_t G) const { return gen == g && tr == t && grid == G; }
};

// One uploaded data set, SoA CSR in HBM.  Arrays are over-allocated so that
// 16-byte-granular TMA bulk copies may read past the logical end.
struct DataSlot {
  bool present = false;
  uint64_t n_rows = 0;
  uint64_t nnz = 0;
  DevPtr<uint64_t> row_ptr;  // [cap_rows + 1 + kRowSlack]
  DevPtr<uint32_t> col;      // [cap_nnz + kEntrySlack]
  DevPtr<float> val;         // [cap_nnz + kEntrySlack]
  DevPtr<float> target;      // [cap_rows + kRowSlack]
  uint32_t max_row_nnz = 0;
  uint64_t cap_rows = 0, cap_nnz = 0;  // allocated capacity (re-uploads reuse the buffers)
  DevPtr<float> feat_cnt;    // [n_attr] occurrences of each feature in this data set
  DevPtr<unsigned int> d_flag;   // 16 words: inspection results of the last upload
  HostPtr<unsigned int> h_flag;  // pinned mirror
  EventPtr ready;                // recorded behind the upload's last operation
  bool pending = false;            // an upload is enqueued and not yet collected
  uint64_t upload_gen = 0;         // unique per upload of a context (fmb200_ctx::upload_counter)
  uint32_t max_feat_cnt = 0;
  // worst-case 4-element-aligned nnz span of any tile of 2^(5+i) rows
  // (i = 0..4 -> 32, 64, 128, 256, 512 rows); sizes the smem staging buffers
  uint32_t tile_span[5] = {0, 0, 0, 0, 0};
  // ORDERED mode (fm_ordered.cu): per-entry distance to the previous entry of the same
  // feature, per-row distance to the nearest earlier row sharing a feature; built lazily
  DevPtr<uint32_t> link;
  DevPtr<uint32_t> rowdep;
  uint64_t link_cap = 0, rowdep_cap = 0;
  uint32_t* ord_shape = nullptr;  // behind rowdep: bit 0 = all values 1, bit 1 = all rows max_row_nnz long
  bool links_ready = false;
  DevPtr<unsigned char> ord_scratch;  // scratch of the index build (kept for re-uploads of moderate size)
  size_t ord_scratch_bytes = 0;
  // fmb200_upload_xblock: the block as the file stores it, the rows' sizes and the offset scan's tile sums
  // (kept with the slot: an asynchronous upload reads them after the call returns)
  DevPtr<unsigned int> x_words, x_row_size;
  DevPtr<unsigned long long> x_scan;
  uint64_t x_words_cap = 0, x_row_size_cap = 0, x_scan_cap = 0;
  RowlaneDeal deal;  // built by a synchronous upload, else at the second HOGWILD epoch (fm_hogwild.cu)
  uint32_t hogwild_epochs = 0;  // HOGWILD epochs run on this upload
};

// Layout of the peer comm block (fm_peer.cu), one per context, mapped by its peers:
//   header | state buffer 0 | state buffer 1 | theta0 | counts, parity 0 | |V|^2 partials x 2 |
//   mean counts | counts, parity 1
// The published counts and row-count words are double-buffered by the parity of the exchange that
// will read them: a slow peer may still be reading exchange e's table while this rank prepares e+1.
// Header words (u32):
constexpr int COMM_SEQ_WORD = 0;                 // [rank]: sequence number of the averaging kernels
constexpr int COMM_BAR_WORD = FMB200_MAX_PEERS;  // [rank]: sequence number of the barrier kernel
constexpr int COMM_ROWS_WORD = 64;               // [COMM_ROWS_PARITY_STRIDE parity + rank]: rows of a shard
constexpr int COMM_ROWS_PARITY_STRIDE = 16;
constexpr int COMM_MEAN_ROWS_WORD = 100;         // [parity]: mean rows per shard, as a float

// per-block |V|^2 partials of the mean-field exchange: two tables of this many floats in the comm block
// (the sliced exchange needs world x grid entries)
constexpr int FMB_PEER_PART = 4096;

struct CommLayout {
  static constexpr size_t hdr_bytes = 1024;
  size_t buf_bytes = 0;   // one state buffer (the packed fp32 state, rounded up to 256 bytes)
  size_t cnt_floats = 0;  // one count table (n_attr, rounded up to 64)
  CommLayout() = default;
  CommLayout(uint64_t n_floats, uint32_t n_attr)
      : buf_bytes((n_floats * sizeof(float) + 255) & ~(size_t)255), cnt_floats(((size_t)n_attr + 63) & ~(size_t)63) {}
  size_t total_bytes() const { return hdr_bytes + 3 * buf_bytes + (3 * cnt_floats + 2 * (size_t)FMB_PEER_PART) * sizeof(float); }
  static unsigned int* words(unsigned char* b) { return reinterpret_cast<unsigned int*>(b); }
  unsigned int* rows_word(unsigned char* b, unsigned parity, int rank) const {
    return words(b) + COMM_ROWS_WORD + COMM_ROWS_PARITY_STRIDE * parity + rank;
  }
  float* buf(unsigned char* b, int i) const { return reinterpret_cast<float*>(b + hdr_bytes + (size_t)i * buf_bytes); }
  float* theta0(unsigned char* b) const { return buf(b, 2); }
  float* counts(unsigned char* b, unsigned parity) const {
    float* cnt0 = buf(b, 3);
    return parity ? cnt0 + 2 * cnt_floats + 2 * (size_t)FMB_PEER_PART : cnt0;
  }
  float* partials(unsigned char* b, int j) const { return counts(b, 0) + cnt_floats + (size_t)j * FMB_PEER_PART; }
  float* mean_counts(unsigned char* b) const { return partials(b, 2); }
};

// Packed fp32 state: [w0, 0 ... | w[n*ws], 0 ... | V[n][kp]].  base is 256-byte aligned and w and V start
// on multiples of `align` floats (one 128-byte line), so a factor row of kp = 8 floats is one 32-byte
// sector and a longer row touches no sector or line it does not fill; the same holds for the records of the
// row-lane epoch's accumulator, which mirrors the state element for element.  The padding words are zero
// and stay zero: the kernels that walk the whole state (fold, scale, peer exchange) rely on it.
// ws = stride of the linear weights in floats: 8 (one w per 32-byte sector) for small
// tables, whose few lines otherwise serialise at L2 under load+reduction traffic, else 1.
struct Params32 {
  static constexpr uint64_t align = 32;  // floats
  float* base = nullptr;
  uint64_t n_floats = 0;
  uint64_t off_w = align;
  uint64_t off_v = 0;
  int ws = 1;
  __host__ __device__ float* w0() const { return base; }
  __host__ __device__ float* w() const { return base + off_w; }
  __host__ __device__ float* v() const { return base + off_v; }
};

// fp64 state: [w0, pad | w[n] (+pad to even) | V[n][k] | 2 pad] attribute-major; w and V start
// on 16-byte boundaries (the ORDERED epoch fetches them with 16-byte cp.async)
struct Params64 {
  double* base = nullptr;
  uint64_t n_doubles = 0;
  uint64_t off_v = 0;
  static constexpr uint64_t off_w = 2;
  __host__ __device__ double* w0() const { return base; }
  __host__ __device__ double* w() const { return base + off_w; }
  __host__ __device__ double* v() const { return base + off_v; }
};

struct HParams {
  int task = 0;
  double lr = 0, reg0 = 0, regw = 0, regv = 0;
  double min_target = 0, max_target = 0;
};

struct McmcState;  // fm_mcmc.cu
struct RelView;    // fm_mcmc.cu
struct McmcDelete {
  void operator()(McmcState* s) const;
};

// One relation block as fmb200_mcmc_set_relations was given it, copied and checked
struct RelationHost {
  uint32_t num_cases = 0, num_feature = 0, attr_offset = 0;
  std::vector<uint64_t> col_ptr;  // [num_feature + 1]
  std::vector<uint32_t> row;
  std::vector<float> val;
  std::vector<uint32_t> join[2];  // train, test
};

struct EpochConfig {
  int lanes_per_row = 0, slots = 0, rows_per_tile = 0, grid = 0, block = 0, smem = 0, damp = 0;
  int dealt = 0;  // the row-lane epoch ran the dealt schedule
};

// The reproducible HOGWILD SGD epoch (fm_sgd_window.cu): tiles of kWindowTileRows rows, windows of kWindowTiles
// tiles (W = 16 384 rows; scripts/sgd_window_study.py, DESIGN.md section 3.3) unless fmb200_set_reproducible sets
// them, within the limits below; the first
// kWindowRampTiles windows of the bias ramp are one tile each
constexpr uint64_t kWindowTileRows = 256, kWindowTiles = 64, kWindowRampTiles = 4;
constexpr int kWindowMaxTileRows = 1024, kWindowMaxTiles = 65536;

// The bookkeeping of the windowed epochs (fm_window.cuh): the stamps for the reproducible SGD and the HOGWILD SGDA
// epoch, the list and count words for the SGD epoch.
// A window's stamp comes from `next`, which only grows, and stamps are only compared for equality with the current
// window's, so no epoch needs the table reset.
struct WindowBook {
  DevPtr<uint32_t> stamp;          // [n]: the stamp of the last window that touched each feature (zero at first)
  DevPtr<uint32_t> list;           // [n]: the features the running window touched, in no particular order
  DevPtr<unsigned long long> aux;  // by window parity: [0, 1] the SGD epoch's bias steps, [2, 3] the list's length
  uint32_t next = 1;               // the stamp of the next launch's window 0
};

}  // namespace fmb

struct fmb200_ctx {
  int device = 0;
  int sm_count = 0;
  int max_smem_optin = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;  // asynchronous uploads (fmb200_upload_data_async)
  fmb::EventPtr ev0, ev1;
  uint32_t n = 0;
  int k = 0, kp = 0;
  bool k0 = true, k1 = true;
  int mode = FMB200_MODE_HOGWILD;
  fmb::HParams hp;
  fmb::Params32 p32;  // base points into the comm block
  fmb::Params64 p64;  // base = p64_buf
  fmb::DevPtr<double> p64_buf;
  fmb::DataSlot slots[FMB200_MAX_SLOTS];
  // scratch
  fmb::DevPtr<double> d_partials;  // evaluate: per-block partial sums (3 per block)
  uint64_t n_partials = 0;
  fmb::DevPtr<double> d_pred;  // predict output staging
  uint64_t pred_cap = 0;
  fmb::DevPtr<unsigned int> d_sched;   // hogwild tile scheduler: [next tile, CTAs run dry]
  fmb::DevPtr<unsigned long long> d_acc;  // the reproducible epochs' fixed-point accumulator (acc_ready)
  fmb::WindowBook window;                 // the windowed SGD and SGDA epochs' stamps, the SGD epoch's list
  // its dealt schedule: the bias step of a window by window parity [2], then the rows' (mult, hjoint) pairs
  fmb::DevPtr<unsigned long long> d_deal_bias;
  uint64_t deal_bias_cap = 0;  // u64 words
  fmb::DevPtr<unsigned int> d_gbar;    // row-lane epoch: arrival counter of its grid barriers (never reset) ...
  uint32_t gbar_count = 0;             // ... and its value once every launch enqueued so far has run
  fmb::DevPtr<unsigned int> d_flag;    // 16 device words: upload-time inspection results
  fmb::HostPtr<unsigned int> h_flag;   // pinned host mirror of d_flag
  fmb::HostPtr<unsigned char> h_stage;  // pinned staging for set/get_params (small models)
  uint64_t launches = 0;
  fmb::EpochConfig last_cfg;
  int tune_ctas_per_sm = 0, tune_rows_per_tile = 0, tune_threads = 0;
  // peer-memory parameter averaging (fm_peer.cu)
  fmb::DevPtr<unsigned char> comm_base;
  fmb::CommLayout comm;
  bool peer_base_valid = false;  // theta0 holds the state the running epoch started from
  bool hogwild_fresh = true;     // no HOGWILD epoch has run since the state was last set (bias ramp)
  int peer_part_cur = 0, peer_n_part = 0;
  unsigned char* peer_base[FMB200_MAX_PEERS] = {nullptr};
  bool peer_ipc[FMB200_MAX_PEERS] = {false};
  int peer_world = 1, peer_rank = 0, peer_cur = 0;
  unsigned int peer_seq = 0, peer_bar_seq = 0;
  // which counts the comm block currently publishes (fm_peer.cu::peer_before_epoch)
  uint64_t peer_cnt_stamp[2] = {0, 0};  // upload generation held by the table of each parity (0 = none)
  uint64_t upload_counter = 0;          // generations handed out to uploads
  // SGDA state (fm_learn_sgd_element_adapt_reg.h): stored gradients, per-group regularisation
  fmb::DevPtr<double> sgda_grad_w, sgda_grad_v, sgda_reg_w, sgda_reg_v;
  fmb::DevPtr<double> sgda_moments;  // var_w | var_v[k] of the last epoch's last update_means
  bool sgda_moments_ready = false;   // an epoch has run since fmb200_sgda_begin
  fmb::DevPtr<uint32_t> sgda_group;
  uint32_t sgda_groups = 0;
  // HOGWILD SGDA (fm_sgda_hogwild.cu): fp32 stored gradients and their window sums, beside the packed state
  // element for element; the lambda-steps' per-group terms of a window [W][groups * (k + 1)]
  fmb::DevPtr<float> sgda_grad32;
  fmb::DevPtr<unsigned long long> sgda_gacc;
  fmb::DevPtr<double> sgda_part;
  uint64_t sgda_part_cap = 0;
  int tune_damp = 0;  // 0 auto, 1 force on, -1 force off
  int tune_variant = 0;  // 0 auto, 1 row-group kernel, 2 row-lane kernel when eligible
  // the reproducible HOGWILD SGD epoch (fmb200_set_reproducible, fm_sgd_window.cu): on, its tile and window
  // geometry, a window's rows' (mult, h_joint)
  bool win_on = false;
  int win_tile_rows = (int)fmb::kWindowTileRows, win_tiles = (int)fmb::kWindowTiles;
  fmb::DevPtr<float2> win_rows;
  uint64_t win_rows_cap = 0;
  std::unique_ptr<fmb::McmcState, fmb::McmcDelete> mcmc;  // MCMC / ALS learner state (fm_mcmc.cu)
  // relation blocks for the next fmb200_mcmc_begin on these slots (fmb200_mcmc_set_relations), consumed by it
  std::vector<fmb::RelationHost> mcmc_rel;
  int mcmc_rel_slot[2] = {-1, -1};
  uint64_t mcmc_rel_gen[2] = {0, 0};  // the two slots' upload generations when the relations were set
};

namespace fmb {

// launch size of the grid-stride helper kernels: blocks of 256 threads, at least 1, at most 8 per SM
inline int grid_for(const fmb200_ctx* c, uint64_t work) {
  const uint64_t blocks = (work + 255) / 256, cap = (uint64_t)c->sm_count * 8;
  return (int)(blocks < 1 ? 1 : (blocks < cap ? blocks : cap));
}

#ifdef __CUDACC__
// One grid-stride helper kernel on c->stream, grid_for(c, work) blocks; counts the launch
template <class... P, class... A>
cudaError_t launch_for(fmb200_ctx* c, uint64_t work, void (*kernel)(P...), A... args) {
  kernel<<<grid_for(c, work), 256, 0, c->stream>>>(args...);
  c->launches++;
  return cudaGetLastError();
}
#endif

// fm_inorder.cu: sequential-equivalent fp64 epoch (one warp, rows in order)
cudaError_t launch_sgd_inorder(fmb200_ctx* c, const DataSlot& d);
// fm_inorder.cu: exact fp64 scores, one warp per row.  out_pred may be null;
// partials (3 doubles per block: sq, abs, correct) may be null.
cudaError_t launch_predict64(fmb200_ctx* c, const DataSlot& d, int transform, double* out_pred,
                             double* partials, int n_blocks);
// fm_ordered.cu: sequentially consistent fp64 epoch (runs of independent rows in parallel, bias by
// affine scan).  *handled = false: shape not eligible, nothing launched (caller uses launch_sgd_inorder)
cudaError_t launch_sgd_ordered(fmb200_ctx* c, DataSlot& d, bool* handled);
// The training entries stably sorted by feature id (each feature's occurrences in file order):
// ids[i] = the id, ent[i] = the entry's position in col[] / val[]
struct SortedEntries {
  const uint32_t* ids = nullptr;
  const uint32_t* ent = nullptr;
};
// Build link[] / rowdep[] of a data set on c->stream (no host sync).  sorted != null: also keep the
// (id, entry) sort behind the index whatever the data set's size, and return a view of it.
cudaError_t build_ordered_links(fmb200_ctx* c, DataSlot& d, SortedEntries* sorted = nullptr);
// fm_mcmc.cu: the MCMC / ALS e-term pass (fm_learn_mcmc.h:148-378), bit-identical accumulation; with relations, the
// n_rel blocks rel (device memory) add their terms through join `side`
cudaError_t launch_mcmc_eterms(fmb200_ctx* c, const DataSlot& d, double* e_out, const RelView* rel = nullptr,
                               uint32_t n_rel = 0, int side = 0);
// fm_mcmc.cu: MCMC / ALS learning (fm_learn_mcmc_simultaneous); "" on success, else the error
std::string mcmc_begin(fmb200_ctx* c, int train, int test, int do_sample, int do_multilevel, uint32_t n_groups,
                       const uint32_t* attr_group, const uint32_t* attr_per_group, double reg0,
                       const double* w_lambda0, const double* v_lambda0, const fmb200_xt_blocks* train_xt = nullptr,
                       const fmb200_xt_blocks* test_xt = nullptr);
std::string mcmc_iteration(fmb200_ctx* c, double* train_metric, uint32_t* counters);
// fm_mcmc.cu: the checks of fmb200_mcmc_set_relations and the host copy; "" on success
std::string mcmc_check_relations(const fmb200_ctx* c, int train, int test, uint32_t n_rel, const fmb200_relation* rel,
                                 std::vector<RelationHost>* out);
bool mcmc_get(const fmb200_ctx* c, double* alpha, double* w_mu, double* w_lambda, double* v_mu, double* v_lambda,
              double* pred_this, double* pred_sum_all, double* pred_sum_all_but5, uint32_t* n_runs);
// fm_inorder.cu: one SGDA epoch (theta-step per training row, lambda-step per validation row).  Its
// per-group state lives in dynamic shared memory: reg_w[G] | reg_v[G][k] | sum_f[G][k] | sum_f_dash_f[G][k] | lwg[G]
inline size_t sgda_smem_bytes(uint32_t n_groups, int k) {
  return sizeof(double) * ((size_t)n_groups * (2 + 3 * (size_t)k));
}
// One launch of an SGDA epoch (fm_sgda_plan.h), after the moments kernel when l.moments.  tr holds training rows
// [tr_row0, tr_row0 + tr.n_rows) of n_train, va validation rows [va_row0, ...) of n_val.
cudaError_t launch_sgda(fmb200_ctx* c, const SgdaLaunch& l, int lambda_steps, const DataSlot& tr, uint64_t tr_row0,
                        uint64_t n_train, const DataSlot& va, uint64_t va_row0, uint64_t n_val);
// fm_sgda_hogwild.cu: the windowed SGDA epoch of HOGWILD mode.  Its windows are kSgdaWindowRows training rows, or
// fmb200_set_tuning's rows_per_tile when that is set; a window's lambda-steps keep groups * (k + 1) doubles each,
// at most kSgdaMaxTerms.
constexpr uint64_t kSgdaWindowRows = 4096;
constexpr uint64_t kSgdaMaxTerms = 8192;
uint64_t sgda_hogwild_window(const fmb200_ctx* c);
cudaError_t launch_sgda_hogwild(fmb200_ctx* c, const DataSlot& tr, const DataSlot& va, int lambda_steps);
// fm_hogwild.cu: throughput epoch
cudaError_t launch_sgd_hogwild(fmb200_ctx* c, DataSlot& d);
// fm_sgd_window.cu: the reproducible HOGWILD SGD epoch, windows of win_tiles tiles of win_tile_rows rows
cudaError_t launch_sgd_window(fmb200_ctx* c, DataSlot& d);
// fm_hogwild.cu: the fixed-point accumulator of the reproducible epochs (row-lane, windowed SGD, SGDA), zeroed on
// first use: *steps := its n_floats step words, *flag (when not null) := the divergence flag behind them
cudaError_t acc_ready(fmb200_ctx* c, unsigned long long** steps, unsigned long long** flag);
// fm_hogwild.cu: a fresh state clears the accumulator's divergence flag
cudaError_t clear_acc_flag(fmb200_ctx* c);
// fm_hogwild.cu: build the dealt copy the row-lane epoch would run on this data set, if it would deal
cudaError_t prepare_rowlane_deal(fmb200_ctx* c, DataSlot& d);
// fm_deal.cu: d.deal := the dealt copy of d for windows of G tiles of TR rows (kept while it matches)
cudaError_t build_rowlane_deal(fmb200_ctx* c, DataSlot& d, int TR, uint32_t G);
// fm_predict.cu: fp32 scores / metrics with sub-warp row groups
cudaError_t launch_predict32(fmb200_ctx* c, const DataSlot& d, int transform, double* out_pred,
                             double* partials, int n_blocks);
// fm_predict.cu: state conversion and scaling
cudaError_t launch_p64_to_p32(fmb200_ctx* c);
cudaError_t launch_p32_to_p64(fmb200_ctx* c);
cudaError_t launch_scale_p32(fmb200_ctx* c, float factor);
// fm_peer.cu: one-shot all-reduce (mean) of the packed fp32 state over peer memory
cudaError_t launch_peer_mean(fmb200_ctx* c);
cudaError_t launch_peer_barrier(fmb200_ctx* c);
cudaError_t peer_preload_kernels();  // defeat lazy loading before any exchange kernel can spin
// mean-field combine theta = theta0 + gamma_i * sum_g (theta_g - theta0) (see fm_peer.cu)
cudaError_t launch_peer_meanfield(fmb200_ctx* c);
cudaError_t peer_before_epoch(fmb200_ctx* c, const DataSlot& d);
// device-side structural check of row offsets (see fm_predict.cu)
cudaError_t launch_csr_inspect(fmb200_ctx* c, cudaStream_t st, const uint64_t* rp, uint64_t n_rows, uint64_t nnz,
                               unsigned int* out8);
// histogram of column ids -> float counts in cnt[n]; *out_max = largest count
cudaError_t launch_feature_counts(fmb200_ctx* c, cudaStream_t st, const uint32_t* col, uint64_t nnz, float* cnt,
                                  unsigned int* out_max_id, unsigned int* out_max);

// fm_upload.cu: the reference's AoS containers -> SoA CSR on the device; one-hot materialisation
cudaError_t launch_aos_to_csr(fmb200_ctx* c, cudaStream_t st, const void* d_rows, const void* d_entries, uint64_t n_rows,
                              uint64_t nnz, unsigned long long host_base_ptr, unsigned long long* scratch,
                              uint64_t* row_ptr, uint32_t* col, float* val, unsigned int* flag);
cudaError_t launch_aos_split(fmb200_ctx* c, cudaStream_t st, const void* d_entries, uint64_t nnz, uint32_t* col, float* val);
uint64_t aos_scan_tiles(uint64_t n_rows);
// d_words: a .x block of n_rows rows and nnz entries (n_rows + 2 nnz words); d_row_size: the rows' sizes.
// Writes row_ptr[0..n_rows], col and val; *flag := n_rows - (first row whose header word is not its size), or 0.
cudaError_t launch_xblock_to_csr(fmb200_ctx* c, cudaStream_t st, const unsigned int* d_words, const unsigned int* d_row_size,
                                 uint64_t n_rows, uint64_t nnz, unsigned long long* scratch, uint64_t* row_ptr,
                                 uint32_t* col, float* val, unsigned int* flag);
cudaError_t launch_onehot_fill(fmb200_ctx* c, cudaStream_t st, uint64_t n_rows, uint32_t z, uint64_t* row_ptr, float* val);
// *out := max(*out, the largest id in col[0..nnz))
cudaError_t launch_max_id(fmb200_ctx* c, cudaStream_t st, const uint32_t* col, uint64_t nnz, unsigned int* out);

// fm_context.cu: a block of a .xt file (rows = features, ids = cases, the .x layout) into `slot`, decoded on
// the device like a .x block; no targets.  _enqueue puts the copies and the decode on `st`; _finish waits for
// them and fails (fmb200_last_error) naming column first_col + r when a header word disagrees with its size,
// or when a case id is not below n_cases.
int upload_xt_enqueue(fmb200_ctx* c, int slot, uint64_t n_cols, uint64_t nnz, const void* words,
                      const uint32_t* col_size, cudaStream_t st);
int upload_xt_finish(fmb200_ctx* c, int slot, uint64_t first_col, uint64_t n_cases);

// pick the sub-warp geometry for a data set: G lanes per V row (power of two
// covering kp/4 float4 chunks), S entry slots per row group, and the row-group
// register-cache class (row_class: -1 .. 3 from short to long rows)
void pick_geometry(int kp, uint64_t n_rows, uint64_t nnz, int* G, int* S, int* cls);

// The register-cache classes of the row-group kernels (fm_rowgroup.cuh): R factor chunks and RW linear
// weights cached per lane, U row sets in flight per warp.
//   class -1: rows of <= S entries            -> R=1,  RW=1, U=4
//   class 0: rows of <= 2*S entries           -> R=2,  RW=1, U=2
//   class 1: medium rows (<= 8*S entries)     -> R=8,  RW=2, U=1
//   class 2: long rows (Criteo-like, 39/row)  -> R=20, RW=2, U=1  (no re-gather up to 20*S)
//   class 3: k = 128 (G = 32, S = 1): a lane walks every entry of the row; 40 cached chunks (160 registers,
//            one CTA per SM) keep a 39-entry row entirely in registers.  Narrower groups stay at class 2.
// U sets the rows a CTA has in flight, and with them the damping's concurrency.
struct RowClass {
  int R, RW, U;
};
constexpr RowClass row_class(int cls, int G) {
  return cls < 0                 ? RowClass{1, 1, 4}
         : cls == 0              ? RowClass{2, 1, 2}
         : cls == 1              ? RowClass{8, 2, 1}
         : (cls == 2 || G < 32) ? RowClass{20, 2, 1}
                                 : RowClass{40, 2, 1};
}
// CTAs per SM the training kernel of (R, U) is built for (its __launch_bounds__); the launcher sizes the
// tiles to that share of the SM's shared memory
constexpr int row_class_ctas(int R, int U) { return R * U <= 4 ? 3 : (R > 20 ? 1 : 2); }

// f(Int<G>{}, Int<S>{}) for the (G, S) of pick_geometry as compile-time constants.  The row-group kernels
// exist for every G of pick_geometry and every power of two S <= 8 with G * S <= 32.
template <int V>
using Int = std::integral_constant<int, V>;

// Factors per lane of a warp whose lane l owns factors l, l + 32, ...: body(Int<KF>{}) for the smallest KF in
// {1, 2, 4, 8} with 32 * KF >= k, up to MAX_KF (4 or 8); cudaErrorInvalidValue when k > 32 * MAX_KF
template <int MAX_KF, class Body>
cudaError_t with_kf(int k, Body&& body) {
  static_assert(MAX_KF == 4 || MAX_KF == 8, "KF is 1, 2, 4 or 8");
  if (k > 32 * MAX_KF) return cudaErrorInvalidValue;
  if (k <= 32) return body(Int<1>{});
  if (k <= 64) return body(Int<2>{});
  if constexpr (MAX_KF == 8) {
    if (k > 128) return body(Int<8>{});
  }
  return body(Int<4>{});
}
template <int G, class F>
auto dispatch_s(int S, F& f) {
  if constexpr (G <= 4) {
    if (S >= 8) return f(Int<G>{}, Int<8>{});
  }
  if constexpr (G <= 8) {
    if (S >= 4) return f(Int<G>{}, Int<4>{});
  }
  if constexpr (G <= 16) {
    if (S >= 2) return f(Int<G>{}, Int<2>{});
  }
  return f(Int<G>{}, Int<1>{});
}
template <class F>
auto dispatch_gs(int G, int S, F f) {
  switch (G) {
    case 1: return dispatch_s<1>(S, f);
    case 2: return dispatch_s<2>(S, f);
    case 4: return dispatch_s<4>(S, f);
    case 8: return dispatch_s<8>(S, f);
    case 16: return dispatch_s<16>(S, f);
    default: return dispatch_s<32>(S, f);
  }
}

// Phase timers, a development aid (fmb200_set_tuning variant 132): a kernel adds the cycles of each of its
// phases to one slot of `slots` (null when the timers are off).  fm_context.cu.
struct PhaseTimers {
  DevPtr<unsigned long long> slots;
  int n = 0;
  // n_slots zeroed slots, on stream st
  cudaError_t start(int n_slots, cudaStream_t st);
  // after the stream's work: one line to stderr, the printf `head` then " name=<slot / per>" for each slot
  // with `decimals` digits; slots that stayed zero are left out when skip_zero
  cudaError_t print(cudaStream_t st, const char* const* names, double per, int decimals, bool skip_zero,
                    const char* head, ...);
};

}  // namespace fmb
