/* fmb200.h -- C ABI of the H100-native libFM SGD hot path.
 *
 * The reference (srendle/libfm) has no plugin/FFI interface; its de-facto seam is
 * the fm_learn vtable (src/libfm/src/fm_learn.h:31-60) and the per-row calls
 * fm->predict / fm_SGD (src/libfm/src/fm_learn_sgd_element.h:57,66).  A per-row
 * seam is useless for a GPU, so this ABI replaces the BODY OF THE EPOCH LOOP
 * (fm_learn_sgd_element.h:56-67) and the evaluate / predict passes
 * (fm_learn.h:93-153, fm_learn_sgd.h:76-90) at per-epoch granularity.
 *
 * Conventions
 *  - every function returns 0 on success, non-zero on error; the message is
 *    available from fmb200_last_error() (thread-local static string).  Nothing
 *    throws across the boundary (the reference throws std::string / const char*,
 *    caught at libfm.cpp:436-440; the host learner converts codes back to that).
 *  - plain pointers and sizes only.  Host pointers unless the name says device.
 *  - one context == one GPU.  Not re-entrant per context (same as the reference,
 *    whose fm_model carries mutable scratch, fm_model.h:65); distinct contexts
 *    may be driven from distinct threads/processes.
 *  - the library is CUDA-only: there is no CPU fallback.  fmb200_create fails
 *    loudly when no sm_90 device is usable.
 */
#ifndef FMB200_H_
#define FMB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct fmb200_ctx fmb200_ctx;

#define FMB200_TASK_REGRESSION 0     /* fm_learn.h:47 */
#define FMB200_TASK_CLASSIFICATION 1 /* fm_learn.h:48 */

/* execution modes of fmb200_sgd_epoch */
#define FMB200_MODE_INORDER 0 /* sequential-equivalent: rows strictly in file order, fp64
                                 state; bit-compatible with fm_learn_sgd_element::learn */
#define FMB200_MODE_HOGWILD 1 /* throughput: rows in parallel, fp32 state, damped per-tile bias
                                 step; rows of at most 4 entries with k <= 8 give the same
                                 result on every run */

#define FMB200_MODE_ORDERED 2 /* sequentially consistent: every example reads all parameters as
                                 the examples before it left them (the reference's order), fp64
                                 state; conflict-free runs of rows execute in parallel and the bias
                                 chain is solved by an affine prefix scan, so sums associate
                                 differently: deterministic, within ~1e-12 of the reference (not
                                 bit-exact; the <=1e-5 RMSE gate with margin), and fast */

#define FMB200_MAX_SLOTS 8
#define FMB200_MAX_PEERS 16
#define FMB200_IPC_HANDLE_BYTES 64

/* Replaces: fm_model construction, libfm.cpp:245-256 (num_attribute, k0, k1, num_factor).
 * `device` is the CUDA ordinal. */
int fmb200_create(fmb200_ctx** out, int device, uint32_t n_attr, int num_factor, int use_w0,
                  int use_w);
void fmb200_destroy(fmb200_ctx* ctx);
const char* fmb200_last_error(void);

/* Replaces: the learner fields set at libfm.cpp:294-309,366-404:
 * task, learn_rate (scalar; fm_learn_sgd.h:67-69), reg0/regw/regv, min/max_target. */
int fmb200_set_hparams(fmb200_ctx* ctx, int task, double learn_rate, double reg0, double regw,
                       double regv, double min_target, double max_target);
int fmb200_set_mode(fmb200_ctx* ctx, int mode);

/* Replaces: the in-memory matrix Data::load builds (Data.h:180-290): upload a CSR
 * copy of a data set into `slot` (0 = train, 1 = test, ...).  The context copies;
 * the caller may free afterwards.  row_ptr has n_rows+1 entries, row_ptr[0]==0.
 * Fails if any col >= n_attr (the reference's live assert, fm_model.h:112). */
int fmb200_upload_data(fmb200_ctx* ctx, int slot, uint64_t n_rows, uint64_t nnz,
                       const uint64_t* row_ptr, const uint32_t* col, const float* val,
                       const float* target);
/* Asynchronous variant: enqueues the copy (and the device-side validation) on the
 * context's copy stream and returns.  The slot must not be in use by a running epoch.
 * The next call that touches the slot (epoch / evaluate / predict) waits for the copy
 * and reports a validation failure; this lets the upload of the NEXT batch overlap the
 * epoch on the current one (two slots, ping-pong).  Host buffers must stay valid and
 * should be page-locked (fmb200_host_alloc) for the copy to be truly asynchronous. */
int fmb200_upload_data_async(fmb200_ctx* ctx, int slot, uint64_t n_rows, uint64_t nnz,
                             const uint64_t* row_ptr, const uint32_t* col, const float* val,
                             const float* target);
/* Same, straight from the reference's AoS layout (util/fmatrix.h:34-42):
 * `rows` points at n_rows sparse_row{sparse_entry* data; uint size;} records (16 B
 * each on LP64), each entry {uint id; float value} (8 B).  When the rows lie back to back in one
 * block -- as Data::load allocates them (Data.h:238,260) -- the row array and the block are
 * copied as they are and converted on the device (offset scan + AoS->SoA split); rows scattered
 * over the heap are gathered on the host first. */
int fmb200_upload_data_aos(fmb200_ctx* ctx, int slot, uint64_t n_rows, const void* rows,
                           const float* target);
/* One-hot rows of a fixed width (every value 1.0, e.g. (user, item) pairs -- what Data::load
 * produces for `y u:1 i:1` files): only ids[n_rows * nnz_per_row] and the targets cross PCIe
 * (4*z + 4 bytes per row instead of 12*z + 12); row offsets and values are materialised on the
 * device.  The _async form behaves like fmb200_upload_data_async. */
int fmb200_upload_onehot(fmb200_ctx* ctx, int slot, uint64_t n_rows, uint32_t nnz_per_row,
                         const uint32_t* ids, const float* target);
int fmb200_upload_onehot_async(fmb200_ctx* ctx, int slot, uint64_t n_rows, uint32_t nnz_per_row,
                               const uint32_t* ids, const float* target);
/* Same, from n_rows consecutive rows of a binary .x file exactly as the file stores them (util/fmatrix.h:
 * per row {uint size; size x {uint id; float value}}, 4 n_rows + 8 nnz bytes at `words`), with the rows'
 * sizes row_size[n_rows] (what the caller read from the headers) and their targets.  Row offsets, the
 * id / value split and the check that every row's header word equals its row_size run on the device; a
 * mismatch fails the upload and names the row (0-based within the block).  The _async form behaves
 * like fmb200_upload_data_async.  This is how the command line streams a data set larger than
 * -cache_size through the GPU, one block at a time. */
int fmb200_upload_xblock(fmb200_ctx* ctx, int slot, uint64_t n_rows, uint64_t nnz, const void* words,
                         const uint32_t* row_size, const float* target);
int fmb200_upload_xblock_async(fmb200_ctx* ctx, int slot, uint64_t n_rows, uint64_t nnz, const void* words,
                               const uint32_t* row_size, const float* target);
int fmb200_free_data(fmb200_ctx* ctx, int slot);

/* Page-locked host memory for the arrays handed to fmb200_upload_data: uploads from it
 * run at full PCIe rate and asynchronously (pageable memory is staged by the driver).
 * The reference allocates its CSR with plain new[] (Data.h:238); a loader that wants
 * the fast path allocates here instead.  Any host memory is accepted by the upload. */
int fmb200_host_alloc(void** out, uint64_t bytes);
int fmb200_host_free(void* p);

/* Replaces: reading / writing fm_model::w0, w, v (fm_model.h:46-48).  v is the
 * reference's FACTOR-MAJOR double [num_factor][n_attr] (util/matrix.h:152-175). */
int fmb200_set_params(fmb200_ctx* ctx, double w0, const double* w, const double* v_factor_major);
int fmb200_get_params(fmb200_ctx* ctx, double* w0, double* w, double* v_factor_major);

/* Replaces: the row loop of fm_learn_sgd_element::learn (fm_learn_sgd_element.h:56-67):
 * predict + loss multiplier + fm_SGD over every row of `slot`.  Blocking; if
 * device_seconds != NULL it receives the CUDA-event time of the epoch. */
int fmb200_sgd_epoch(fmb200_ctx* ctx, int slot, double* device_seconds);
/* enqueue only (no host sync); pair with fmb200_sync */
int fmb200_sgd_epoch_async(fmb200_ctx* ctx, int slot);
int fmb200_sync(fmb200_ctx* ctx);

/* Replaces: fm_learn::evaluate_regression / evaluate_classification
 * (fm_learn.h:113-153).  Regression fills sum_sq_err and sum_abs_err of
 * clamp(p)-y; classification fills n_correct (sign agreement). */
int fmb200_evaluate(fmb200_ctx* ctx, int slot, double* sum_sq_err, double* sum_abs_err,
                    uint64_t* n_correct);

/* Replaces: fm_learn_sgd::predict (fm_learn_sgd.h:76-90).  transform=1 applies
 * the task transform (clamp / sigmoid) exactly as -out writes it; transform=0
 * returns the raw score of fm_model::predict (fm_model.h:105-127). */
int fmb200_predict(fmb200_ctx* ctx, int slot, int transform, double* out);

/* Replaces: fm_learn_mcmc::predict_data_and_write_to_eterms (fm_learn_mcmc.h:148-378, data sets
 * without relations) -- the full re-prediction of a data set the MCMC / ALS learner runs on train
 * and test once per iteration (fm_learn_mcmc_simultaneous.h:69,122).  e_out[c] receives the e-term
 * of case c, accumulated in the learner's own order (feature-major through the transposed data),
 * bit-identical to the reference; the caller subtracts the targets and keeps the Gibbs draws.
 * Uses the fp64 state (INORDER / ORDERED mode): fmb200_set_params after every draw_all(). */
int fmb200_mcmc_eterms(fmb200_ctx* ctx, int slot, double* e_out);

/* Replaces: fm_learn_mcmc_simultaneous (fm_learn_mcmc.h, fm_learn_mcmc_simultaneous.h) on data sets without
 * relations: -method mcmc (do_sample = do_multilevel = 1) and -method als (both 0).  The parameters, the
 * hyperparameters, the NaN/Inf counters and the test predictions after every iteration are bit-identical to
 * the reference's.  Uses the fp64 state (INORDER / ORDERED mode).
 *  _begin:     fm_learn_mcmc::init + the prologue of _learn (:56-86).  The caller has set the model as
 *              libfm.cpp:245-283 leaves it (fm.init(), then w ~ N(init_mean, init_stdev)), the task and
 *              min/max_target (fmb200_set_hparams).  attr_group[n] (NULL: one group) and
 *              attr_per_group[n_groups] (NULL: counted from attr_group) are DataMetaInfo's; reg0,
 *              w_lambda[n_groups] and v_lambda[n_groups][num_factor] are what -regular sets
 *              (libfm.cpp:326-364).  Builds the transposed training set and its feature runs.
 *  _iteration: one pass of the iteration loop (:88-200): draw_all, re-prediction of train and test, the
 *              test prediction sums and the target step.  The draws take libc rand() of the calling
 *              process in the reference's order, so the caller seeds it with srand (libfm.cpp:115-116)
 *              before initialising the model.  train_metric receives the RMSE (regression) or accuracy
 *              (classification) the #Iter line prints as Train; counters[16] the NaN and Inf counts of
 *              alpha, w0, w, v, w_mu, w_lambda, v_mu, v_lambda in that order.  One deviation: a sampled draw
 *              the reference would skip without consuming a random number (posterior variance not finite
 *              or zero, which only a diverged state gives) fails the call, naming the parameter and the
 *              iteration, instead of desynchronising the random stream.
 *  _get_hyper: alpha, w_mu[n_groups], w_lambda[n_groups], v_mu[n_groups][num_factor], v_lambda (any NULL).
 *  _get_pred:  pred_this, pred_sum_all, pred_sum_all_but5 over the test set (any NULL).
 *  _runs:      how many runs of conflict-free feature ids the sweep walks. */
int fmb200_mcmc_begin(fmb200_ctx* ctx, int train_slot, int test_slot, int do_sample, int do_multilevel,
                      uint32_t n_groups, const uint32_t* attr_group, const uint32_t* attr_per_group, double reg0,
                      const double* w_lambda, const double* v_lambda);
/* Out-of-core form of _begin (the reference's Data with has_xt and -cache_size: LargeSparseMatrixHD over
 * <file>.xt, Data.h:120-176).  A data set given as fmb200_xt_blocks (non-NULL) is not held on the device: every
 * pass of every iteration (the sweeps, the q rebuilds, the e-terms) streams its .xt blocks in file order
 * through the two slots it names, decoding each on the device like fmb200_upload_xblock; the copy of block b+1
 * overlaps the work on block b.  A NULL blocks pointer takes that data set from its slot as _begin does; train
 * and test decide independently.  Results are bit-identical to _begin's.  fmb200_mcmc_iteration, _get_hyper,
 * _get_pred and _runs serve both.  _runs counts the runs the streamed sweep walks: the resident cut plus a
 * cut at every block start (a run never spans two blocks).
 * The .xt layout is the .x layout with rows = features and ids = cases: per column {uint size; size x
 * {uint case; float value}}, a column's cases ascending, a case named twice by a column adjacent in entry order.
 * Limits: fewer than 2^32 cases and fewer than 2^32 entries per block; the total entry count is not bounded. */
typedef struct fmb200_xt_blocks {
  uint64_t n_cases;        /* the .xt header's num_cols; equals the number of targets */
  const float* target;     /* [n_cases], read during the call */
  uint64_t n_blocks;       /* >= 1 */
  const uint32_t* col_lo;  /* [n_blocks + 1]: block b holds columns (feature ids) [col_lo[b], col_lo[b+1]);
                              col_lo[0] = 0, col_lo[n_blocks] = the .xt's num_rows <= num_attribute */
  const uint64_t* nnz;     /* [n_blocks] entries of each block */
  int slot[2];             /* the two slots the blocks pass through (distinct, and not the other set's slot) */
  void* user;
  /* Block b as the file stores it (col_lo[b+1] - col_lo[b] columns, 4 per column + 8 per entry bytes at *words)
   * and its columns' sizes; page-locked memory makes the copy asynchronous.  The memory must stay valid until
   * release(user, b).  Blocks are fetched in order, from 0, once per pass; non-zero fails the call. */
  int (*fetch)(void* user, uint64_t block, const void** words, const uint32_t** col_size);
  void (*release)(void* user, uint64_t block);
} fmb200_xt_blocks;
int fmb200_mcmc_begin_xt(fmb200_ctx* ctx, int train_slot, const fmb200_xt_blocks* train_xt, int test_slot,
                         const fmb200_xt_blocks* test_xt, int do_sample, int do_multilevel, uint32_t n_groups,
                         const uint32_t* attr_group, const uint32_t* attr_per_group, double reg0,
                         const double* w_lambda, const double* v_lambda);
/* Relational data (block structure, BS): the reference's RelationData / RelationJoin (relation.h) and the
 * relational parts of fm_learn_mcmc (fm_learn_mcmc.h:148-378, 430-641, 734-790, 849-935, 1183-1188).  Each case
 * of train and test joins one row of each relation block; the block's attributes are the model's ids
 * attr_offset .. attr_offset + num_feature - 1.  Called after the train and test uploads and before
 * fmb200_mcmc_begin with the same two slots, it makes that _begin, and the _iteration, _get_hyper and _get_pred
 * calls after it, run the relational learner; the next _begin without a new call runs without relations.  A
 * _begin consumes them whether it succeeds or fails, and refuses them when either slot was re-uploaded.  The
 * call copies everything it is given.  n_rel = 0 withdraws relations set before.  attr_group / attr_per_group of
 * _begin are the joined meta table of libfm.cpp:213-240 over all n attributes.  Checks (a named error, nothing is
 * kept): join lengths equal to the slots' case counts, join and row ids below num_cases, a .xt whose column
 * starts ascend from 0, and offsets that follow one another and end at num_attribute.  _begin then checks that
 * neither main data set names an id at or above the first attr_offset.  fmb200_mcmc_begin_xt refuses relations;
 * fmb200_mcmc_eterms ignores them. */
typedef struct fmb200_relation {
  uint32_t num_cases;          /* rows of the block (RelationData::num_cases, the .xt's num_cols) */
  uint32_t num_feature;        /* its attributes (the .xt's num_rows) */
  uint32_t attr_offset;        /* model id of its attribute 0 */
  const uint64_t* col_ptr;     /* [num_feature + 1]: the block's .xt, column j at [col_ptr[j], col_ptr[j + 1]) */
  const uint32_t* row;         /* [col_ptr[num_feature]]: relation row of every entry, in file order */
  const float* val;            /* [col_ptr[num_feature]] */
  uint64_t n_train, n_test;    /* lengths of the two joins */
  const uint32_t* train_join;  /* [n_train]: train case -> relation row (<rel>.train) */
  const uint32_t* test_join;   /* [n_test]: test case -> relation row (<rel>.test) */
} fmb200_relation;
int fmb200_mcmc_set_relations(fmb200_ctx* ctx, int train_slot, int test_slot, uint32_t n_rel,
                              const fmb200_relation* rel);
int fmb200_mcmc_iteration(fmb200_ctx* ctx, double* train_metric, uint32_t* counters);
int fmb200_mcmc_get_hyper(fmb200_ctx* ctx, double* alpha, double* w_mu, double* w_lambda, double* v_mu,
                          double* v_lambda);
int fmb200_mcmc_get_pred(fmb200_ctx* ctx, double* pred_this, double* pred_sum_all, double* pred_sum_all_but5);
int fmb200_mcmc_runs(fmb200_ctx* ctx, uint32_t* n_runs);

/* Replaces: fm_learn_sgd_element_adapt_reg (SGDA, fm_learn_sgd_element_adapt_reg.h).
 *  _begin: init() + the prologue of learn() (:60-90, :281-292): stored gradients and the per-group
 *          regularisation values start at 0, fm->w is zeroed; attr_group[n] = DataMetaInfo::attr_group
 *          (NULL = one group).
 *  _epoch: one pass of :295-311 -- a theta-step (:136-169) per training row, each followed, when
 *          lambda_steps != 0 (the reference skips them in its first epoch, :301), by a lambda-step
 *          (:201-248) on the next validation row, the cursor restarting per epoch and wrapping.
 *          Sequential semantics, fp64, bit-identical to the reference (one warp; for num_factor <= 8
 *          and rows of at most 4 entries a wavefront of conflict-free steps, fmb200_set_tuning
 *          variant 1 forcing the one-warp kernel).
 *  _epoch_x: the out-of-core form of _epoch (the reference's -cache_size over binary .x data).  A set given
 *          as fmb200_xt_blocks (non-NULL) is not held on the device: its .x blocks are fetched in file order
 *          through its two slots and decoded on the device like fmb200_upload_xblock, the copy of the next block
 *          overlapping the work on the current one; a NULL blocks pointer takes the set from its slot as _epoch
 *          does.  The struct describes a .x exactly as it describes a .xt, with rows in place of columns: n_cases
 *          = the rows (= targets), col_lo[b] = the first row of block b, col_lo[n_blocks] = n_cases, fetch hands
 *          out block b's words and its rows' sizes.  The training set is passed once per epoch.  The validation
 *          set is read only by lambda-steps, from the cursor's row: a pass over it starts at block 0 once every
 *          block fetched before has been released (the cursor restarts), and may end early (the epoch ends).
 *          Parameters, regularisation values and moments after every epoch are bit-identical to _epoch on the
 *          same data resident.  Limits: one GPU, the fp64 modes, fewer than 2^32 rows and fewer than 2^32
 *          entries per block.
 *  _get_reg: reg_w[n_groups], reg_v[n_groups][num_factor].
 *  _get_moments: var_w and var_v[num_factor] of the last epoch's last update_means (:250-274), taken
 *          at the epoch's start or, when the validation cursor restarts, before the last restart's
 *          lambda-step; the means the reference logs with them are always 0 (:270-273).
 *  _get_reg and _get_moments serve _epoch and _epoch_x alike.
 *
 * In HOGWILD mode the same entry points run SGDA as a windowed fp32 epoch (fm_sgda_hogwild.cu), for
 * throughput.  The epoch is cut into windows of W consecutive training rows, the first at row 0 (W = 4096; for
 * tests fmb200_set_tuning's rows_per_tile overrides it).  In each window every training row is scored from the
 * state as the window found it and takes the reference's theta-step with reg as the previous window left it, its
 * steps damped by the mean-field scale of the HOGWILD epoch (damp = -1 turns that off), rounded to 2^-32 and
 * summed exactly; the window's stored gradient of every feature it names becomes the sum of its rows' gradients.
 * Then, with lambda_steps, one lambda-step per theta-step reads the folded state, those gradients and the same
 * reg, and reg <- max(0, reg + the window's summed lambda terms).  With W = 1 and no damping this is the
 * reference's SGDA.  The moments are those of the state the lambda-steps read in the window holding the last
 * cursor restart (the epoch's start without one).  Every sum is exact or in a fixed order, so an epoch computes
 * the same bits on every run and at every grid size.  _begin also zeroes the fp32 w.  Limits: num_factor <= 128,
 * n_groups * (num_factor + 1) <= 8192, one GPU, resident data sets (_epoch_x with blocks is refused); a step or
 * gradient that is not finite or not below 2^11 turns the state into NaN. */
int fmb200_sgda_begin(fmb200_ctx* ctx, uint32_t n_groups, const uint32_t* attr_group);
int fmb200_sgda_epoch(fmb200_ctx* ctx, int train_slot, int val_slot, int lambda_steps, double* device_seconds);
int fmb200_sgda_epoch_x(fmb200_ctx* ctx, int train_slot, const fmb200_xt_blocks* train, int val_slot,
                        const fmb200_xt_blocks* val, int lambda_steps, double* device_seconds);
int fmb200_sgda_get_reg(fmb200_ctx* ctx, double* reg_w, double* reg_v);
int fmb200_sgda_get_moments(fmb200_ctx* ctx, double* var_w, double* var_v);

/* Multi-GPU plumbing (row sharding + one all-reduce of w0|w|V per epoch; the
 * reference has no equivalent).  The HOGWILD state is one packed fp32 device
 * buffer [w0, pad | w (strided), pad | V[n][kp]], the pads zero; the caller all-reduces it
 * (NCCL) and calls fmb200_scale_params(1/G).  Both run on fmb200_stream(). */
int fmb200_params_device(fmb200_ctx* ctx, void** device_ptr, uint64_t* n_floats);
int fmb200_scale_params(fmb200_ctx* ctx, double factor);
/* geometry of the packed fp32 state: w0 at [0], w[i] at [off_w + i*ws], V[i][f] at [off_v + i*kp + f];
 * off_w and off_v are multiples of 32 floats and the buffer is 256-byte aligned, so w and V start on
 * 128-byte lines */
int fmb200_params_layout(fmb200_ctx* ctx, uint64_t* off_w, int* ws, uint64_t* off_v, int* kp);
int fmb200_stream(fmb200_ctx* ctx, void** cuda_stream);

/* The same exchange without NCCL, over NVLink peer memory: every rank maps the
 * peers' state (CUDA IPC between processes: export -> exchange the 64-byte handles by
 * any means -> attach; or attach_local for contexts of one process) and
 * fmb200_allreduce_mean() launches ONE kernel per rank that barriers through peer
 * flags and averages all replicas into a second local buffer (double-buffered, so
 * fmb200_params_device() changes after every call).  Attach once, before training. */
int fmb200_peer_export(fmb200_ctx* ctx, void* handle /* FMB200_IPC_HANDLE_BYTES */);
int fmb200_peer_attach_ipc(fmb200_ctx* ctx, int world, int rank, const void* handles /* world x 64 B */);
int fmb200_peer_attach_local(fmb200_ctx* ctx, int world, int rank, fmb200_ctx* const* contexts);
int fmb200_allreduce_mean(fmb200_ctx* ctx);
/* Same exchange, but instead of the plain mean the replicas' epoch steps are combined as
 * theta = theta0 + gamma_i * sum_g (theta_g - theta0), gamma_i = (1-(1-s_i)^G)/(G s_i) with s_i the
 * relative size of one shard-epoch's step on parameter i (from the per-feature counts every upload
 * builds): parameters a shard-epoch already converges (the bias, hot features) are averaged, barely
 * touched ones are summed.  8 shards then follow the single-stream trajectory instead of advancing
 * 1/8 epoch per epoch (DESIGN.md section 4).  Call after every epoch, like fmb200_allreduce_mean.
 * State of 8 MB and more takes the SLICED form: rank r combines slice r (read from all replicas) and pushes
 * it into every rank's buffers -- 2(G-1)/G x state bytes over NVLink per rank instead of (G-1) x -- followed
 * by a peer barrier (fmb200_set_tuning variant 8 forces it, 9 forces the one-shot kernel). */
int fmb200_allreduce_meanfield(fmb200_ctx* ctx);
/* stream-ordered barrier across the attached peers (no data); used to align ranks */
int fmb200_peer_barrier(fmb200_ctx* ctx);

/* Introspection for tests / bench */
/* the device CSR of a slot, copied back (any pointer may be NULL): lets the tests check the
 * layout conversions of the upload paths bit for bit */
int fmb200_download_data(fmb200_ctx* ctx, int slot, uint64_t* n_rows, uint64_t* nnz, uint64_t* row_ptr,
                         uint32_t* col, float* val, float* target);
int fmb200_kernel_launches(fmb200_ctx* ctx, uint64_t* count); /* kernels launched so far */
int fmb200_last_epoch_config(fmb200_ctx* ctx, int* lanes_per_row, int* slots, int* rows_per_tile,
                             int* grid, int* block, int* smem_bytes, int* damp);
/* 1 when the last epoch was the row-lane epoch's dealt schedule: each window's rows dealt to the CTAs
 * sorted by the id of their last entry (bit-identical to the file-order schedule, fewer L2 requests) */
int fmb200_last_epoch_dealt(fmb200_ctx* ctx, int* dealt);
/* hogwild tuning knobs; 0 keeps the default.  ctas_per_sm bounds the number of
 * rows in flight (the Hogwild staleness window).  damp: 0 = automatic hot-feature
 * damping (on when the hottest feature's expected concurrency matters), 1 = force
 * on, -1 = force off (plain summed Hogwild on w/V).  variant: 0 = automatic choice
 * of the epoch kernel, 1 = sub-warp row-group kernel, 2 = one-lane-per-row kernel
 * (k <= 8, rows of <= 4 entries; ignored when not applicable), 3 = its warp-specialised
 * form (producer warp + mbarrier hand-offs; bias read three tiles ahead), 5 = the one-lane-per-row
 * kernel on rows in file order (no deal; see fmb200_last_epoch_dealt).  rows_per_tile (1 .. 2^20): the SGD epochs
 * take the tile of 32 .. 512 rows nearest below it; HOGWILD SGDA (fmb200_sgda_epoch) takes it as its window W,
 * for tests, and damps unless damp = -1.
 * INORDER mode runs the wavefront schedule of the sequential epoch for k <= 8 and rows of <= 4
 * entries (conflict-free runs of examples gather and scatter in parallel, only the bias chain
 * stays serial; bit-identical to the row-at-a-time kernel, verified on the device); variant 1
 * forces the row-at-a-time kernel.
 * MCMC / ALS, read by fmb200_mcmc_begin: the sweeps over segments (relation blocks, streamed .xt blocks) sweep each
 * stretch of narrow feature runs (no more features than the CTA has warps) with one CTA of `threads` threads
 * (0: 256) and a CTA barrier between runs, and wide runs with the cooperative grid; variant 1 sweeps every run
 * with the grid.  The results are the same bits either way. */
int fmb200_set_tuning(fmb200_ctx* ctx, int ctas_per_sm, int rows_per_tile, int threads, int damp,
                      int variant);
/* Reproducible HOGWILD SGD (on != 0): every fmb200_sgd_epoch[_async] in HOGWILD mode runs the windowed epoch
 * (fm_sgd_window.cu), whatever k (<= 128) and row length.  Tiles are tile_rows consecutive rows in file order,
 * windows window_tiles tiles, the first at row 0, the last tile and window what is left; 0 takes the default
 * (256 rows, 64 tiles: windows of 16 384 rows).  Limits: tile_rows 1 .. 1024, window_tiles 1 .. 65 536.  In the
 * first epoch after fmb200_set_params, with a bias, unless damp = -1, on more than 32 tiles, the first 4 windows
 * are one tile each (the bias ramp).  Every row of a window is scored from the state as the window found it and
 * takes the reference's SGD step (fm_sgd.h:38-50) -- a feature the row names twice takes two steps from that
 * state --, damped by gamma(c_i, lr (h_joint + reg)) with c_i = count_i * min(N, flight) / N (flight = the window's
 * rows, one tile in a ramp window), rounded to 2^-32 and summed exactly; the bias takes one damped step per tile
 * from the tile's summed loss multipliers and curvatures, added in a fixed order; the sums are folded into the fp32
 * state after the window.  Damping is on when the hottest feature's concurrency over a window matters
 * (fmb200_set_tuning's damp forces it on or off).  The parameters after an epoch are a function of the state, the
 * data, the hyperparameters and (tile_rows, window_tiles, damping) only: the same bits on every run, for every
 * grid size, CTAs per SM, threads per CTA and SM count.  fmb200_set_tuning's ctas_per_sm and threads still pick
 * the launch and change no result; its rows_per_tile and variant are ignored (variant 132
 * prints the kernel's phase timers, a development aid).  fmb200_last_epoch_config reports
 * the launch's grid and block and tile_rows as rows_per_tile.  Limits of exactness: a window adds at most
 * S = min(window rows * longest row, nnz) steps to an element, and a step that is not finite or not below
 * min(2^11, 2^31 / S) (so every sum stays below 2^63) turns the state into NaN.  A data set streamed in blocks
 * (fmb200_upload_xblock) runs one epoch call per block, so windows restart at every block; with several GPUs each
 * shard's epoch is reproducible, the exchange is not part of the claim.  INORDER and ORDERED epochs are
 * deterministic already and HOGWILD SGDA is windowed already: the switch leaves them alone.  on = 0 restores
 * the default dispatch. */
int fmb200_set_reproducible(fmb200_ctx* ctx, int on, int tile_rows, int window_tiles);
/* The dependency index ORDERED mode builds per data set (bit-exact index work, tested against a
 * host restatement): link[e] = e - (previous entry naming the same feature), rowdep[r] = r -
 * (nearest earlier row sharing a feature; 0 = the row names a feature twice); 0xffffffff = none.
 * Builds the index if the slot does not have it yet.  Either pointer may be NULL. */
int fmb200_ordered_index(fmb200_ctx* ctx, int slot, uint32_t* link /* [nnz] */,
                         uint32_t* rowdep /* [n_rows] */);

#ifdef __cplusplus
}
#endif
#endif /* FMB200_H_ */
