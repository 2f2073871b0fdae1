// fmb200_internal.h -- context layout and kernel launch entry points shared by
// the translation units of libfmb200.so.  Not part of the public ABI.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/fmb200.h"

namespace fmb {

// One uploaded data set, SoA CSR in HBM.  Arrays are over-allocated so that
// 16-byte-granular TMA bulk copies may read past the logical end.
struct DataSlot {
  bool present = false;
  uint64_t n_rows = 0;
  uint64_t nnz = 0;
  uint64_t* row_ptr = nullptr;  // [n_rows + 1] (+ padding)
  uint32_t* col = nullptr;      // [nnz] (+ padding)
  float* val = nullptr;         // [nnz] (+ padding)
  float* target = nullptr;      // [n_rows] (+ padding)
  uint32_t max_row_nnz = 0;
  uint64_t cap_rows = 0, cap_nnz = 0;  // allocated capacity (re-uploads reuse the buffers)
  float* feat_cnt = nullptr;    // [n_attr] occurrences of each feature in this data set
  unsigned int* d_flag = nullptr;  // 16 words: inspection results of the last upload
  unsigned int* h_flag = nullptr;  // pinned mirror
  cudaEvent_t ready = nullptr;     // recorded behind the upload's last operation
  bool pending = false;            // an upload is enqueued and not yet collected
  uint64_t upload_gen = 0;         // unique per upload of a context (fmb200_ctx::upload_counter)
  uint32_t max_feat_cnt = 0;
  // worst-case 4-element-aligned nnz span of any tile of 2^(5+i) rows
  // (i = 0..4 -> 32, 64, 128, 256, 512 rows); sizes the smem staging buffers
  uint32_t tile_span[5] = {0, 0, 0, 0, 0};
  // ORDERED mode (fm_ordered.cu): per-entry distance to the previous entry of the same
  // feature, per-row distance to the nearest earlier row sharing a feature; built lazily
  uint32_t* link = nullptr;
  uint32_t* rowdep = nullptr;
  uint32_t* ord_shape = nullptr;  // behind rowdep: bit 0 = all values 1, bit 1 = all rows max_row_nnz long
  bool links_ready = false;
  void* ord_scratch = nullptr;  // scratch of the index build (kept for re-uploads of moderate size)
  size_t ord_scratch_bytes = 0;
};

// Packed fp32 state: [w0, 0, 0, 0 | w[n*ws] padded to a multiple of 4 | V[n][kp]].
// ws = stride of the linear weights in floats: 8 (one w per 32-byte sector) for small
// tables, whose few lines otherwise serialise at L2 under load+reduction traffic, else 1.
struct Params32 {
  float* base = nullptr;
  uint64_t n_floats = 0;
  uint64_t off_w = 4;
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

// per-block |V|^2 partials of the mean-field exchange: two tables of this many floats in the comm block
// (the sliced exchange needs world x grid entries)
constexpr int FMB_PEER_PART = 4096;

struct McmcState;  // fm_mcmc.cu

struct EpochConfig {
  int lanes_per_row = 0, slots = 0, rows_per_tile = 0, grid = 0, block = 0, smem = 0, damp = 0;
};

}  // namespace fmb

struct fmb200_ctx {
  int device = 0;
  int sm_count = 0;
  int max_smem_optin = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;  // asynchronous uploads (fmb200_upload_data_async)
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  uint32_t n = 0;
  int k = 0, kp = 0;
  bool k0 = true, k1 = true;
  int mode = FMB200_MODE_HOGWILD;
  fmb::HParams hp;
  fmb::Params32 p32;
  fmb::Params64 p64;
  fmb::DataSlot slots[FMB200_MAX_SLOTS];
  // scratch
  double* d_partials = nullptr;  // evaluate: per-block partial sums
  int n_partials = 0;
  double* d_pred = nullptr;  // predict output staging
  uint64_t pred_cap = 0;
  unsigned int* d_sched = nullptr;   // hogwild tile scheduler: [next tile, CTAs run dry]
  unsigned long long* d_acc = nullptr;  // fixed-point steps of one row-lane launch, beside p32 (zero between launches)
  unsigned int* d_flag = nullptr;    // 16 device words: upload-time inspection results
  unsigned int* h_flag = nullptr;    // pinned host mirror of d_flag
  void* h_stage = nullptr;           // pinned staging for set/get_params (small models)
  size_t h_stage_bytes = 0;
  uint64_t launches = 0;
  fmb::EpochConfig last_cfg;
  int tune_ctas_per_sm = 0, tune_rows_per_tile = 0, tune_threads = 0;
  // peer-memory parameter averaging (fm_peer.cu).  comm block = [flags | buf0 | buf1]
  unsigned char* comm_base = nullptr;
  size_t comm_hdr = 1024, comm_buf_bytes = 0;
  // behind the two state buffers: theta0 (comm_buf_bytes) | counts (comm_cnt_floats) | |V|^2 partials (2 x FMB_PEER_PART) | mean counts | counts of the other parity
  size_t comm_cnt_floats = 0;
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
  double *sgda_grad_w = nullptr, *sgda_grad_v = nullptr, *sgda_reg_w = nullptr, *sgda_reg_v = nullptr;
  uint32_t* sgda_group = nullptr;
  uint32_t sgda_groups = 0;
  int tune_damp = 0;  // 0 auto, 1 force on, -1 force off
  int tune_variant = 0;  // 0 auto, 1 row-group kernel, 2 row-lane kernel when eligible
  fmb::McmcState* mcmc = nullptr;  // MCMC / ALS learner state (fm_mcmc.cu)
};

namespace fmb {

// fm_inorder.cu: sequential-equivalent fp64 epoch (one warp, rows in order)
cudaError_t launch_sgd_inorder(fmb200_ctx* c, const DataSlot& d);
// fm_inorder.cu: exact fp64 scores, one warp per row.  out_pred may be null;
// partials (3 doubles per block: sq, abs, correct) may be null.
cudaError_t launch_predict64(fmb200_ctx* c, const DataSlot& d, int transform, double* out_pred,
                             double* partials, int n_blocks);
// fm_ordered.cu: sequentially consistent fp64 epoch (runs of independent rows in parallel, bias by
// affine scan).  *handled = false: shape not eligible, nothing launched (caller uses launch_sgd_inorder)
cudaError_t launch_sgd_ordered(fmb200_ctx* c, DataSlot& d, bool* handled);
// keep_scratch: keep the (id, entry) sort in d.ord_scratch whatever the data set's size
cudaError_t build_ordered_links(fmb200_ctx* c, DataSlot& d, bool keep_scratch = false);
// fm_inorder.cu: the MCMC / ALS e-term pass (fm_learn_mcmc.h:148-378), bit-identical accumulation
cudaError_t launch_mcmc_eterms(fmb200_ctx* c, const DataSlot& d, double* e_out);
// fm_mcmc.cu: MCMC / ALS learning (fm_learn_mcmc_simultaneous); "" on success, else the error
std::string mcmc_begin(fmb200_ctx* c, int train, int test, int do_sample, int do_multilevel, uint32_t n_groups,
                       const uint32_t* attr_group, const uint32_t* attr_per_group, double reg0,
                       const double* w_lambda0, const double* v_lambda0);
std::string mcmc_iteration(fmb200_ctx* c, double* train_metric, uint32_t* counters);
bool mcmc_get(const fmb200_ctx* c, double* alpha, double* w_mu, double* w_lambda, double* v_mu, double* v_lambda,
              double* pred_this, double* pred_sum_all, double* pred_sum_all_but5, uint32_t* n_runs);
void mcmc_free(fmb200_ctx* c);
// fm_inorder.cu: one SGDA epoch (theta-step per training row, lambda-step per validation row)
cudaError_t launch_sgda_epoch(fmb200_ctx* c, const DataSlot& tr, const DataSlot& va, int lambda_steps);
// fm_hogwild.cu: throughput epoch
cudaError_t launch_sgd_hogwild(fmb200_ctx* c, const DataSlot& d);
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
cudaError_t launch_csr_inspect(fmb200_ctx* c, const uint64_t* rp, uint64_t n_rows, uint64_t nnz,
                               unsigned int* out8);
// histogram of column ids -> float counts in cnt[n]; *out_max = largest count
cudaError_t launch_feature_counts(fmb200_ctx* c, const uint32_t* col, uint64_t nnz, float* cnt,
                                  unsigned int* out_max_id, unsigned int* out_max);

// fm_upload.cu: the reference's AoS containers -> SoA CSR on the device; one-hot materialisation
cudaError_t launch_aos_to_csr(fmb200_ctx* c, const void* d_rows, const void* d_entries, uint64_t n_rows,
                              uint64_t nnz, unsigned long long host_base_ptr, unsigned long long* scratch,
                              uint64_t* row_ptr, uint32_t* col, float* val, unsigned int* flag);
cudaError_t launch_aos_split(fmb200_ctx* c, const void* d_entries, uint64_t nnz, uint32_t* col, float* val);
uint64_t aos_scan_tiles(uint64_t n_rows);
cudaError_t launch_onehot_fill(fmb200_ctx* c, uint64_t n_rows, uint32_t z, uint64_t* row_ptr, float* val);

// pick the sub-warp geometry for a data set: G lanes per V row (power of two
// covering kp/4 float4 chunks), S entry slots per row group, and the row-group
// register-cache class (fm_hogwild.cu, pick_r: -1 .. 3 from short to long rows)
void pick_geometry(int kp, uint64_t n_rows, uint64_t nnz, int* G, int* S, int* cls);

}  // namespace fmb
